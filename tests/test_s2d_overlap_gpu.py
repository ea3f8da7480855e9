"""The space-to-depth AMP link (csrc/amp_s2d.cu) with its Snake epilogue running under the next tile's MMAs: every
(C, k, dilation) link of the generator's stages 2-4, with and without the Snake output and the residual, over a
ragged batch long enough that every persistent CTA walks more than four tiles.  Each item is checked against the
oracle run on that item alone, two runs must be bitwise equal, and nothing may be written past an item's end: y,
the decoded next-link image and the raw output-image rows outside each item stay zero."""
import pytest
import torch
import torch.nn.functional as F

from oracle import svc_oracle as O
from tests.util import max_abs

pytestmark = pytest.mark.gpu

# configs/base.yaml, stages 2-4: C = 40, 20, 10; resblock kernels 3, 7, 11; c1 dilations 1, 3, 5 (c2: 1)
LINKS = [(C, k, d) for C in (40, 20, 10) for k in (3, 7, 11) for d in (1, 3, 5)]
PADR = 16          # zero rows in front of every (item, octet) of an S2D image


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    from whisper_vits_svc_b200 import ops as o
    return o


_BATCH = {}


def batch(C, n_sm, filt):
    """Input, residual and item lengths of one stage, and the oracle SnakeAlias of every item's input (one per C)."""
    if C in _BATCH:
        return _BATCH[C]
    r = 160 // C
    S = 128 - 2 * (1 if r >= 8 else 2)                       # useful rows per tile
    B = 3
    tpi = (4 * n_sm) // B + 2                                # tiles per item: > 4 tiles per CTA
    L = r * (S * tpi - 8)                                    # the longest item's last tile is partly empty
    lens = [L, L - 37 * 8 * r, 8 * r * (L // (16 * r)) + 24 * r]   # the others end inside a tile
    g = torch.Generator().manual_seed(C)
    x = torch.randn(B, C, L, generator=g) * 1.5
    res = torch.randn(B, C, L, generator=g)
    fa = {"a.act.alpha": torch.randn(C, generator=g) * 0.4, "a.act.beta": torch.randn(C, generator=g) * 0.4,
          "a.upsample.filter": filt[0], "a.downsample.lowpass.filter": filt[1]}
    xa = [O.snake_alias(fa, "a", x[b:b + 1, :, :n]) for b, n in enumerate(lens)]
    _BATCH[C] = x, res, lens, fa, xa
    return _BATCH[C]


@pytest.mark.parametrize("snake_res", [True, False])
@pytest.mark.parametrize("C,K,dil", LINKS)
def test_link_overlap_ragged(ops, sd, C, K, dil, snake_res):
    filt = (sd["dec.activation_post.upsample.filter"], sd["dec.activation_post.downsample.lowpass.filter"])
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    x, res, lens, fa, xa = batch(C, n_sm, filt)
    r = 160 // C
    g = torch.Generator().manual_seed(C * 31 + K * 7 + dil + snake_res)
    w = torch.randn(C, C, K, generator=g) / (C * K) ** 0.5
    b = torch.randn(C, generator=g) * 0.1
    fb = {"b.act.alpha": torch.randn(C, generator=g) * 0.4, "b.act.beta": torch.randn(C, generator=g) * 0.4,
          "b.upsample.filter": filt[0], "b.downsample.lowpass.filter": filt[1]}
    xd, rd = x.cuda(), res.cuda()

    def run():
        return ops.amp_s2d_link_ragged(xd, lens, fa["a.act.alpha"], fa["a.act.beta"], filt[0], filt[1], w, b.cuda(),
                                       dilation=dil, res=rd if snake_res else None,
                                       alpha_out=fb["b.act.alpha"] if snake_res else None,
                                       beta_out=fb["b.act.beta"] if snake_res else None)

    first, second = run(), run()
    torch.cuda.synchronize()
    assert all((a is None) == (not snake_res) for a in first[1:])
    for a, c in zip(first, second):
        assert (a is None and c is None) or torch.equal(a, c)
    y, y_act, o_hi, o_lo = (t.cpu() if t is not None else None for t in first)
    e1 = e2 = 0.0
    for i, n in enumerate(lens):
        ref = F.conv1d(xa[i], w, b, dilation=dil, padding=dil * (K - 1) // 2)
        if snake_res:
            ref = ref + res[i:i + 1, :, :n]
            e2 = max(e2, max_abs(y_act[i:i + 1, :, :n], O.snake_alias(fb, "b", ref)))
            assert not y_act[i, :, n:].any()
            nrows = n // r
            assert not o_hi[i, :, :PADR].any() and not o_lo[i, :, :PADR].any()
            assert not o_hi[i, :, PADR + nrows:].any() and not o_lo[i, :, PADR + nrows:].any()
        e1 = max(e1, max_abs(y[i:i + 1, :, :n], ref))
        assert not y[i, :, n:].any()
    print(f"C={C} K={K} d={dil} lens={lens}: conv max-abs {e1:.3e}, next-snake max-abs {e2:.3e}")
    assert e1 <= 2e-4 and e2 <= 3e-4, (e1, e2)
