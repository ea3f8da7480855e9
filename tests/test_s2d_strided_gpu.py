"""Folded space-to-depth links (csrc/amp_s2d.cu): every c1 link of generator stages 2-4 on the fold pack.s2d_fold
picks, dense and ragged, at lengths that end inside a block and inside a tile, against the oracle; and every c2 link
writing the next c1 link's folded image, which must hold, position by position, the bits of the standard image the
same link writes, and zeros at every position past an item's end."""
import pytest
import torch
import torch.nn.functional as F

from oracle import svc_oracle as O
from tests.util import max_abs
from whisper_vits_svc_b200 import pack

pytestmark = pytest.mark.gpu

PADR = 16          # zero rows in front of every (item, octet) of an S2D image
C1_LINKS = [(C, k, d) for C in (40, 20, 10) for k in (3, 7, 11) for d in (3, 5)
            if pack.s2d_fold(k, d, pack.s2d_factor(C)) > 1]
C2_OUT = [(C, k, f) for C in (40, 20, 10) for k in (3, 7, 11) for f in (3, 5)]


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    from whisper_vits_svc_b200 import ops as o
    return o


def snake_params(C, g, filt, name):
    return {f"{name}.act.alpha": torch.randn(C, generator=g) * 0.4, f"{name}.act.beta": torch.randn(C, generator=g) * 0.4,
            f"{name}.upsample.filter": filt[0], f"{name}.downsample.lowpass.filter": filt[1]}


def lengths(C, n_sm):
    """A length that ends inside a block of folds 3 and 5 and inside a tile, long enough for > 2 tiles per CTA,
    and ragged item lengths that end inside blocks too."""
    r = 160 // C
    nrows = 120 * ((3 * n_sm) // 2) + 112                  # 112: not a multiple of 3 or 5
    lens = [nrows * r, (nrows - 166) * r, 607 * r]
    return nrows * r, [n - n % 8 for n in lens]


@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("C,K,dil", C1_LINKS)
def test_folded_c1_link(ops, sd, C, K, dil, ragged):
    filt = (sd["dec.activation_post.upsample.filter"], sd["dec.activation_post.downsample.lowpass.filter"])
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    L, lens = lengths(C, n_sm)
    if not ragged:
        lens = [L, L]
    B = len(lens)
    g = torch.Generator().manual_seed(C * 131 + K * 17 + dil)
    x = torch.randn(B, C, L, generator=g) * 1.5
    res = torch.randn(B, C, L, generator=g)
    w = torch.randn(C, C, K, generator=g) / (C * K) ** 0.5
    b = torch.randn(C, generator=g) * 0.1
    fa, fb = snake_params(C, g, filt, "a"), snake_params(C, g, filt, "b")
    kw = dict(dilation=dil, res=res.cuda(), alpha_out=fb["b.act.alpha"], beta_out=fb["b.act.beta"])

    def run():
        if ragged:
            return ops.amp_s2d_link_ragged(x.cuda(), lens, fa["a.act.alpha"], fa["a.act.beta"], filt[0], filt[1], w,
                                           b.cuda(), **kw)[:2]
        return ops.amp_s2d_link(x.cuda(), fa["a.act.alpha"], fa["a.act.beta"], filt[0], filt[1], w, b.cuda(), **kw)

    first, second = run(), run()
    torch.cuda.synchronize()
    assert torch.equal(first[0], second[0]) and torch.equal(first[1], second[1])
    y, y_act = first[0].cpu(), first[1].cpu()
    e1 = e2 = 0.0
    for i, n in enumerate(lens):
        xa = O.snake_alias(fa, "a", x[i:i + 1, :, :n])
        ref = F.conv1d(xa, w, b, dilation=dil, padding=dil * (K - 1) // 2) + res[i:i + 1, :, :n]
        e1 = max(e1, max_abs(y[i:i + 1, :, :n], ref))
        e2 = max(e2, max_abs(y_act[i:i + 1, :, :n], O.snake_alias(fb, "b", ref)))
        if ragged:
            assert not y[i, :, n:].any() and not y_act[i, :, n:].any()
    print(f"C={C} K={K} d={dil} fold={pack.s2d_fold(K, dil, 160 // C)} lens={lens}: {e1:.3e} {e2:.3e}")
    assert e1 <= 2e-4 and e2 <= 3e-4, (e1, e2)


def image_samples(img, C, f, n):
    """(values [C, n] of the samples < n, values at positions holding a sample >= n) of one item's raw image
    [20, Rp, 8] of fold f."""
    r = 160 // C
    Rp = img.shape[1]
    rows = (Rp - PADR) // f * f
    v = img[:, PADR:PADR + rows].permute(1, 0, 2).reshape(rows, C, r)           # [row][c][p]
    row = torch.arange(rows)[:, None]
    p = torch.arange(r)[None, :]
    s = (row // f) * r * f + row % f + p * f                                     # [row][p]
    out = torch.empty(C, n, dtype=v.dtype)
    inside = s < n
    out[:, s[inside]] = v.permute(1, 0, 2)[:, inside]
    return out, v.permute(1, 0, 2)[:, ~inside]


@pytest.mark.parametrize("C,K,fold", C2_OUT)
def test_c2_writes_folded_image(ops, sd, C, K, fold):
    filt = (sd["dec.activation_post.upsample.filter"], sd["dec.activation_post.downsample.lowpass.filter"])
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    L, lens = lengths(C, n_sm)
    B = len(lens)
    g = torch.Generator().manual_seed(C * 7 + K * 3 + fold)
    x = torch.randn(B, C, L, generator=g) * 1.5
    res = torch.randn(B, C, L, generator=g)
    w = torch.randn(C, C, K, generator=g) / (C * K) ** 0.5
    b = torch.randn(C, generator=g) * 0.1
    fa, fb = snake_params(C, g, filt, "a"), snake_params(C, g, filt, "b")

    def run(od):
        out = ops.amp_s2d_link_ragged(x.cuda(), lens, fa["a.act.alpha"], fa["a.act.beta"], filt[0], filt[1], w,
                                      b.cuda(), dilation=1, res=res.cuda(), alpha_out=fb["b.act.alpha"],
                                      beta_out=fb["b.act.beta"], out_dilation=od)
        return [t.cpu() for t in out]

    std, fol, again = run(1), run(fold), run(fold)
    assert all(torch.equal(a, c) for a, c in zip(fol, again))
    assert torch.equal(std[0], fol[0]) and torch.equal(std[1], fol[1])          # y, decoded next image
    for i, n in enumerate(lens):
        for part in (2, 3):                                                      # hi, lo
            s_std, _ = image_samples(std[part][i].view(torch.int16), C, 1, n)
            s_fol, outside = image_samples(fol[part][i].view(torch.int16), C, fold, n)
            assert torch.equal(s_std, s_fol), (C, K, fold, i)
            assert not outside.any()
