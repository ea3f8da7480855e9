"""Every (C, k, dilation) link of the generator's space-to-depth stages (csrc/amp_s2d.cu), whose edge taps
multiply only the output columns they reach: each link against the oracle, with and without the Snake output
and the residual, and bitwise identical across reruns."""
import pytest
import torch
import torch.nn.functional as F

from oracle import svc_oracle as O
from tests.util import max_abs

pytestmark = pytest.mark.gpu

# configs/base.yaml, stages 2-4: C = 40, 20, 10; resblock kernels 3, 7, 11; c1 dilations 1, 3, 5 (c2: 1)
LINKS = [(C, k, d) for C in (40, 20, 10) for k in (3, 7, 11) for d in (1, 3, 5)]


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    from whisper_vits_svc_b200 import ops as o
    return o


@pytest.mark.parametrize("snake_res", [True, False])
@pytest.mark.parametrize("C,K,dil", LINKS)
def test_link_with_trimmed_taps(ops, sd, C, K, dil, snake_res):
    r = 160 // C
    S = 128 - 2 * (1 if r >= 8 else 2)
    B, L = 2, r * (2 * S + 38)                     # two whole tiles and a partial one per item; L % 8 == 0
    g = torch.Generator().manual_seed(C * 31 + K * 7 + dil + snake_res)
    x = torch.randn(B, C, L, generator=g) * 1.5
    w = torch.randn(C, C, K, generator=g) / (C * K) ** 0.5
    b = torch.randn(C, generator=g) * 0.1
    res = torch.randn(B, C, L, generator=g) if snake_res else None
    filt = {"upsample.filter": sd["dec.activation_post.upsample.filter"],
            "downsample.lowpass.filter": sd["dec.activation_post.downsample.lowpass.filter"]}
    fa = {"a.act.alpha": torch.randn(C, generator=g) * 0.4, "a.act.beta": torch.randn(C, generator=g) * 0.4,
          **{"a." + k: v for k, v in filt.items()}}
    fb = {"b.act.alpha": torch.randn(C, generator=g) * 0.4, "b.act.beta": torch.randn(C, generator=g) * 0.4,
          **{"b." + k: v for k, v in filt.items()}}

    def run():
        return ops.amp_s2d_link(x.cuda(), fa["a.act.alpha"], fa["a.act.beta"], filt["upsample.filter"],
                                filt["downsample.lowpass.filter"], w, b.cuda(), dilation=dil,
                                res=res.cuda() if snake_res else None,
                                alpha_out=fb["b.act.alpha"] if snake_res else None,
                                beta_out=fb["b.act.beta"] if snake_res else None)

    got, got_act = run()
    again, again_act = run()
    torch.cuda.synchronize()
    assert torch.equal(got, again)
    ref = F.conv1d(O.snake_alias(fa, "a", x), w, b, dilation=dil, padding=dil * (K - 1) // 2)
    if snake_res:
        ref = ref + res
        assert torch.equal(got_act, again_act)
    e1 = max_abs(got, ref)
    e2 = max_abs(got_act, O.snake_alias(fb, "b", ref)) if snake_res else 0.0
    assert e1 <= 2e-4 and e2 <= 3e-4, (e1, e2)
