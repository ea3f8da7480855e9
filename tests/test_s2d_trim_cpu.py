"""Output-column order and per-tap column ranges of the space-to-depth AMP links (csrc/amp_s2d.cu): the kernel's
weight image is a column permutation of pack_conv_s2d's, and every weight outside a tap's declared column range
is exactly zero, hi and lo, so the kernel may skip those columns without changing any result bit."""
import itertools

import pytest
import torch

from whisper_vits_svc_b200 import pack

# every link of configs/base.yaml's stages 2-4 (C = 40, 20, 10; k in 3, 7, 11; c1 with dilation 1, 3, 5, c2
# with 1) and the shapes of test_pack_cpu
BASE_LINKS = sorted({(C, k, d) for C in (40, 20, 10) for k in (3, 7, 11) for d in (1, 3, 5)})
PACK_LINKS = [(20, 3, 1), (20, 7, 3), (20, 11, 5), (10, 11, 5), (10, 3, 3), (40, 7, 5), (40, 11, 5)]


def _image(w, dil, r, packer):
    T = sum(pack.s2d_taps(w.shape[-1], dil, r)) + 1
    return packer(w, dil, r).view(torch.bfloat16).view(T, 2, 20, 160, 8)


@pytest.mark.parametrize("r", [4, 8, 16])
def test_column_order_is_a_permutation(r):
    order = pack.s2d_column_order(r)
    assert sorted(order.tolist()) == list(range(160))
    C, g = 160 // r, r // 4
    for n in range(160):   # slot n // 40 holds phase group S2D_SLOT_GROUPS[n // 40], channel by channel
        c, p = divmod(int(order[n]), r)
        assert p // g == pack.S2D_SLOT_GROUPS[n // 40] and c == (n % 40) // g


@pytest.mark.parametrize("C,k,dil", PACK_LINKS)
def test_slot_image_is_a_column_permutation(C, k, dil):
    r = pack.s2d_factor(C)
    g = torch.Generator().manual_seed(C * 13 + k + dil)
    w = torch.randn(C, C, k, generator=g)
    ref = _image(w, dil, r, pack.pack_conv_s2d)
    got = _image(w, dil, r, pack.pack_conv_s2d_slots)
    assert torch.equal(got.view(torch.int16), ref[:, :, :, pack.s2d_column_order(r)].view(torch.int16))


@pytest.mark.parametrize("C,k,dil", sorted(set(BASE_LINKS + PACK_LINKS)))
def test_weights_outside_a_taps_columns_are_zero(C, k, dil):
    r = pack.s2d_factor(C)
    g = torch.Generator().manual_seed(C * 17 + k + dil)
    w = torch.randn(C, C, k, generator=g) + 1.0      # no exact zeros inside the reach
    img = _image(w, dil, r, pack.pack_conv_s2d_slots).view(torch.int16)
    cols = pack.s2d_tap_cols(k, dil, r)
    assert len(cols) == img.shape[0]
    for t, (n0, n1) in enumerate(cols):
        assert (n0, n1) in ((0, 40), (0, 80), (80, 120), (80, 160), (0, 160))
        outside = torch.ones(160, dtype=torch.bool)
        outside[n0:n1] = False
        assert torch.count_nonzero(img[t][:, :, outside]) == 0, (t, n0, n1)     # hi and lo, all bits
        # a trimmed range is tight at 40-column granularity: its outermost slot holds a nonzero weight
        if n1 - n0 < 160:
            assert torch.count_nonzero(img[t][0, :, n1 - 40:n1]) > 0


@pytest.mark.parametrize("C,k,dil", sorted(set(BASE_LINKS + PACK_LINKS)))
def test_tap_phase_range_closed_form_matches_enumeration(C, k, dil):
    """Tap m reaches output phase p when some conv tap j maps p to input row offset m:
    r*m + pi = p + j*dil - P for a pi in [0, r).  The closed form [max(0, r m - P), min(r-1, r m + r-1 + P)]
    must contain every such phase (so skipping the rest is exact) and be tight wherever it is not clamped to
    [0, r-1] (at a clamped end a dilation larger than r can leave phases unreached); the declared columns
    must cover every reached phase."""
    r = pack.s2d_factor(C)
    P = dil * (k - 1) // 2
    mlo, mhi = pack.s2d_taps(k, dil, r)
    reached = {m: set() for m in range(-mlo, mhi + 1)}
    for p, j in itertools.product(range(r), range(k)):
        m, _ = divmod(p + j * dil - P, r)
        reached[m].add(p)
    order = pack.s2d_column_order(r)
    for t, (n0, n1) in enumerate(pack.s2d_tap_cols(k, dil, r)):
        m = t - mlo
        lo, hi = max(0, r * m - P), min(r - 1, r * m + r - 1 + P)
        assert reached[m] and lo <= min(reached[m]) and max(reached[m]) <= hi
        if r * m - P > 0:
            assert min(reached[m]) == lo
        if r * m + r - 1 + P < r - 1:
            assert max(reached[m]) == hi
        phases = {int(order[n]) % r for n in range(n0, n1)}
        assert reached[m] <= phases
