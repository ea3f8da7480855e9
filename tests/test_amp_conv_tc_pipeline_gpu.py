"""The AMP-link convolution of generator stages 0-1 (csrc/amp_conv_tc.cu) where each persistent CTA walks several
tiles: C = 80 runs the ping-pong schedule (the two consumer warpgroups take the even and the odd tiles of the CTA's
walk, one's epilogue under the other's MMAs), C = 160 the cooperative one (both warpgroups on one tile).  Every
(C, k, dilation) link of the two stages, with and without the residual, the stage accumulation and the division,
at a length that is not a multiple of the 128-row tile and gives every CTA an odd number of tiles.  Results are
checked against the oracle at the gate of test_ops_gpu.py and must be bitwise identical across reruns."""
import pytest
import torch
import torch.nn.functional as F

from oracle import svc_oracle as O
from tests.util import max_abs

pytestmark = pytest.mark.gpu

# (dilation, residual, accumulate, divide): the c1 links, a plain c2 link, and the two last links of a stage
MODES = [(1, False, False, False), (3, False, False, False), (5, False, False, False),
         (1, True, False, False), (1, True, True, False), (1, True, True, True)]


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    from whisper_vits_svc_b200 import ops as o
    return o


@pytest.fixture(scope="module")
def inputs(sd):
    """Per C: B = 3 items of L = 128 n_sm - 37 samples, so 3 n_sm tiles and 3 per CTA (two for warpgroup 0, one for
    warpgroup 1), the last tile of each item partly past its end; plus SnakeAlias(x) from the oracle."""
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    B, L = 3, 128 * n_sm - 37
    out = {}
    for C in (160, 80):
        g = torch.Generator().manual_seed(C)
        x = torch.randn(B, C, L, generator=g) * 1.5
        fa = {"a.act.alpha": torch.randn(C, generator=g) * 0.4, "a.act.beta": torch.randn(C, generator=g) * 0.4,
              "a.upsample.filter": sd["dec.activation_post.upsample.filter"],
              "a.downsample.lowpass.filter": sd["dec.activation_post.downsample.lowpass.filter"]}
        res = torch.randn(B, C, L, generator=g)
        acc = torch.randn(B, C, L, generator=g)
        out[C] = (x, fa, O.snake_alias(fa, "a", x), res, acc)
    return out


@pytest.mark.parametrize("mode", MODES, ids=lambda m: "d{}{}{}{}".format(m[0], "_res" * m[1], "_acc" * m[2], "_div" * m[3]))
@pytest.mark.parametrize("K", [3, 7, 11])
@pytest.mark.parametrize("C", [160, 80])
def test_link_many_tiles_per_cta(ops, inputs, C, K, mode):
    dil, with_res, accum, div = mode
    x, fa, xs, res, acc = inputs[C]
    g = torch.Generator().manual_seed(C * 7 + K + dil)
    w = torch.randn(C, C, K, generator=g) / (C * K) ** 0.5
    b = torch.randn(C, generator=g) * 0.1
    out_div = 3.0 if div else 0.0

    def run():
        return ops.amp_conv_tc(x.cuda(), fa["a.act.alpha"], fa["a.act.beta"], fa["a.upsample.filter"],
                               fa["a.downsample.lowpass.filter"], w, b.cuda(), dilation=dil,
                               res=res.cuda() if with_res else None, acc=acc.cuda() if accum else None, out_div=out_div)

    got = run()
    again = run()
    torch.cuda.synchronize()
    assert torch.equal(got, again)
    ref = F.conv1d(xs, w, b, dilation=dil, padding=dil * (K - 1) // 2)
    if with_res:
        ref = ref + res
    if accum:
        ref = ref + acc
    if div:
        ref = ref / out_div
    err = max_abs(got, ref)
    print(f"C={C} K={K} d={dil} res={with_res} acc={accum} div={div}: max-abs {err:.3e}")
    assert err <= 2e-4


def test_ragged_stages_0_1_equal_lone_calls(hp, sd):
    """A ragged batch whose items end inside stage-0 and stage-1 tiles (5 n and 20 n samples, none a multiple of 128):
    each item is bitwise what a lone call of its own length gives."""
    from whisper_vits_svc_b200 import models
    m = models.SynthesizerInfer(513, 25, hp, precision=3)
    m.load_state_dict(sd)
    m.to("cuda")
    lens, T = [611, 433, 97, 250], 611
    g = torch.Generator().manual_seed(5)
    B, hop = len(lens), 320
    d = {"ppg": torch.randn(B, T, hp.vits.ppg_dim, generator=g), "vec": torch.randn(B, T, hp.vits.vec_dim, generator=g),
         "pit": torch.randint(100, 501, (B, T), generator=g).float(), "spk": torch.randn(B, hp.vits.spk_dim, generator=g) * 0.05,
         "source": torch.randn(B, 1, T * hop, generator=g) * 0.1, "eps": torch.randn(B, hp.vits.inter_channels, T, generator=g)}
    d = {k: v.cuda() for k, v in d.items()}
    w = m.inference_ragged(d["ppg"], d["vec"], d["pit"], d["spk"], lens, d["source"], eps=d["eps"])
    torch.cuda.synchronize()
    for b, n in enumerate(lens):
        lone = m.inference(d["ppg"][b:b + 1, :n], d["vec"][b:b + 1, :n], d["pit"][b:b + 1, :n], d["spk"][b:b + 1],
                           torch.tensor([n]), d["source"][b:b + 1, :, :n * hop], eps=d["eps"][b:b + 1, :, :n])
        assert torch.isfinite(lone).all()
        assert torch.equal(w[b, 0, :n * hop], lone[0, 0]), n
