"""Folded space-to-depth images (csrc/amp_s2d.cu): a conv of dilation d run as the undilated conv's block-Toeplitz
matrices over an image whose row b*d + q holds the samples b*r*d + q + j*d, tap m shifted by m*d rows, equals the
dilated conv; and pack.py's plan folds the c1 links of generator stages 2-4 where that lowers their column work."""
import pytest
import torch
import torch.nn.functional as F

from whisper_vits_svc_b200 import pack

# configs/base.yaml, stages 2-4: C = 40, 20, 10; resblock kernels 3, 7, 11; c1 dilations 1, 3, 5 (c2: 1)
LINKS = [(C, k, d) for C in (40, 20, 10) for k in (3, 7, 11) for d in (1, 3, 5)]


def fold_perm(nrows, r, f):
    """Sample held by element (row, p) of a fold-f image, flattened row-major over whole blocks of rows."""
    rows = -(-nrows // f) * f
    row, p = torch.arange(rows).repeat_interleave(r), torch.arange(r).repeat(rows)
    return (row // f) * r * f + row % f + p * f


@pytest.mark.parametrize("C,k,d", LINKS)
def test_folded_conv_matches_dilated_conv(C, k, d):
    r = pack.s2d_factor(C)
    f = pack.s2d_fold(k, d, r)
    L = r * (3 * 5 * 7 + 2)                       # ends inside a block of every fold
    g = torch.Generator().manual_seed(C * 100 + k * 10 + d)
    x = torch.randn(C, L, generator=g, dtype=torch.float64)
    w = torch.randn(C, C, k, generator=g, dtype=torch.float64)
    ref = F.conv1d(x[None], w, dilation=d, padding=d * (k - 1) // 2)[0]

    perm = fold_perm(L // r, r, f)
    rows = perm.numel() // r
    inside = perm < L
    img = torch.zeros(rows * r, C, dtype=torch.float64)        # [(row, p)][c]
    img[inside] = x[:, perm[inside]].T
    img = img.view(rows, r, C).permute(0, 2, 1).reshape(rows, C * r)   # K' index c * r + p
    mats = pack.conv_s2d_matrices(w.float(), 1 if f > 1 else d, r).double()
    mlo, mhi = pack.s2d_taps(k, 1 if f > 1 else d, r)
    pad = (mlo + mhi) * f
    src = torch.zeros(rows + 2 * pad, C * r, dtype=torch.float64)
    src[pad:pad + rows] = img
    out = torch.zeros(rows, C * r, dtype=torch.float64)
    for m in range(-mlo, mhi + 1):
        out += src[pad + m * f:pad + m * f + rows] @ mats[m + mlo].T
    y = torch.zeros(C, L, dtype=torch.float64)
    y[:, perm[inside]] = out.view(rows, C, r).permute(0, 2, 1).reshape(rows * r, C)[inside].T   # un-permute
    # the fp32 matrices carry fp32 rounding of w
    assert torch.allclose(y, ref, atol=1e-4 * k * C ** 0.5, rtol=0), (y - ref).abs().max()


def test_plan_folds_and_taps():
    taps, folds = {}, {}
    for C, k, d in LINKS:
        r = pack.s2d_factor(C)
        f = pack.s2d_fold(k, d, r)
        folds[C, k, d] = f
        taps[C, k, d] = sum(pack.s2d_taps(k, 1 if f > 1 else d, r)) + 1
    # folded: the links of more than 3 full taps of column work whose undilated conv needs less per useful row
    folded = {(40, 3, 5), (40, 7, 3), (40, 7, 5), (40, 11, 3), (40, 11, 5), (20, 7, 3), (20, 7, 5), (20, 11, 3),
              (20, 11, 5), (10, 11, 5)}
    for C, k, d in LINKS:
        assert folds[C, k, d] == (d if (C, k, d) in folded else 1), (C, k, d, folds[C, k, d])
    # every link has at most 5 taps; stage 2's fold the issue's 5, 7, 9, 9, 15 taps to 3, 3, 3, 5, 5
    assert max(taps.values()) == 5
    assert [taps[40, k, d] for k, d in ((3, 5), (7, 3), (7, 5), (11, 3), (11, 5))] == [3, 3, 3, 5, 5]
    assert all(taps[C, k, d] == 3 for C in (20, 10) for k in (3, 7, 11) for d in (3, 5))


def test_column_work_of_a_step():
    """Column work (in 160-column taps) of the 54 links of a step: 165 unfolded, 125 with the plan's folds."""
    def work(k, d, r):
        return sum(n1 - n0 for n0, n1 in pack.s2d_tap_cols(k, d, r)) / 160

    before = after = 0.0
    for C, k, d in LINKS:
        r = pack.s2d_factor(C)
        c2 = work(k, 1, r)
        before += work(k, d, r) + c2
        after += work(k, 1 if pack.s2d_fold(k, d, r) > 1 else d, r) + c2
    assert (before, after) == (165.0, 125.0)


def test_tile_geometry():
    # folded inputs: tiles of whole blocks inside the 144-row A panel with the taps' reach, a halo of one block
    assert pack.s2d_tile(4, 5, 1, 2, 2) == (5, 110, 10)        # C = 40, k = 11, d = 5: +-10 rows, 120-row tiles
    assert pack.s2d_tile(4, 3, 1, 2, 2) == (3, 120, 6)
    assert pack.s2d_tile(8, 5, 1, 1, 1) == (5, 115, 5)
    assert pack.s2d_tile(16, 3, 1, 1, 1) == (3, 120, 3)
    # folded outputs: whole output blocks of useful rows
    assert pack.s2d_tile(4, 1, 3, 1, 1) == (2, 123, 8)
    assert pack.s2d_tile(4, 1, 5, 1, 1) == (2, 120, 8)
    assert pack.s2d_tile(8, 1, 5, 1, 1) == (1, 125, 8)
    assert pack.s2d_tile(16, 1, 1, 1, 1) == (1, 126, 8)


def test_blob_holds_undilated_matrices_for_folded_links():
    w = torch.randn(40, 40, 11, generator=torch.Generator().manual_seed(3))
    assert torch.equal(pack.pack_conv_s2d_link(w, 5, 4), pack.pack_conv_s2d_slots(w, 1, 4))
    assert torch.equal(pack.pack_conv_s2d_link(w, 1, 4), pack.pack_conv_s2d_slots(w, 1, 4))
    w3 = torch.randn(10, 10, 3, generator=torch.Generator().manual_seed(4))
    assert torch.equal(pack.pack_conv_s2d_link(w3, 3, 16), pack.pack_conv_s2d_slots(w3, 3, 16))
