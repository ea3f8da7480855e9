"""The AMP-link convolution of generator stages 0-1 (csrc/amp_conv_tc.cu) at a length that is a multiple of 4, where
the residual and the stage sum are bulk-copied into shared memory by channel row, with a partial last tile.  Every
(C, k, dilation) link of the two stages, with and without the residual, the stage accumulation and the division, as
in test_amp_conv_tc_pipeline_gpu.py (whose length is not a multiple of 4, so it runs the generic-load epilogue), plus
channel counts that are not a multiple of 8, whose last octet stages fewer than 8 rows per array.
The result must match the oracle and be bitwise what the generic-load epilogue gives: a residual that starts 4 bytes
off a 16-byte boundary cannot be bulk-copied, so the same call with such a copy of it takes that path."""
import pytest
import torch
import torch.nn.functional as F

from oracle import svc_oracle as O
from tests.test_amp_conv_tc_pipeline_gpu import MODES, ops  # noqa: F401  (ops: fixture)
from tests.util import max_abs

pytestmark = pytest.mark.gpu


def _link_inputs(sd, C, B, L, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, C, L, generator=g) * 1.5
    fa = {"a.act.alpha": torch.randn(C, generator=g) * 0.4, "a.act.beta": torch.randn(C, generator=g) * 0.4,
          "a.upsample.filter": sd["dec.activation_post.upsample.filter"],
          "a.downsample.lowpass.filter": sd["dec.activation_post.downsample.lowpass.filter"]}
    res = torch.randn(B, C, L, generator=g)
    acc = torch.randn(B, C, L, generator=g)
    return x, fa, O.snake_alias(fa, "a", x), res, acc


@pytest.fixture(scope="module")
def inputs(sd):
    """Per C: B = 3 items of L = 128 n_sm - 36 samples (a multiple of 4), so 3 n_sm tiles and 3 per CTA, the last
    tile of each item 92 rows long; plus SnakeAlias(x) from the oracle.  C = 20 and 12: B = 2, L = 1020."""
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    out = {C: _link_inputs(sd, C, 3, 128 * n_sm - 36, C + 1) for C in (160, 80)}
    out.update({C: _link_inputs(sd, C, 2, 1020, C + 1) for C in (20, 12)})
    return out


def _unaligned(t):
    """A copy of t on the GPU whose data starts 4 bytes past a 16-byte boundary."""
    buf = torch.empty(t.numel() + 1, device="cuda")
    v = buf[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 == 4
    return v


@pytest.mark.parametrize("mode", MODES, ids=lambda m: "d{}{}{}{}".format(m[0], "_res" * m[1], "_acc" * m[2], "_div" * m[3]))
@pytest.mark.parametrize("K", [3, 7, 11])
@pytest.mark.parametrize("C", [160, 80])
def test_link_staged_residual(ops, inputs, C, K, mode):
    _check_link(ops, inputs, C, K, mode)


@pytest.mark.parametrize("mode", MODES[3:], ids=lambda m: "d{}{}{}{}".format(m[0], "_res" * m[1], "_acc" * m[2], "_div" * m[3]))
@pytest.mark.parametrize("C", [20, 12])
def test_link_staged_residual_partial_octet(ops, inputs, C, mode):
    _check_link(ops, inputs, C, 3, mode)


def _check_link(ops, inputs, C, K, mode):
    dil, with_res, accum, div = mode
    x, fa, xs, res, acc = inputs[C]
    g = torch.Generator().manual_seed(C * 7 + K + dil)
    w = torch.randn(C, C, K, generator=g) / (C * K) ** 0.5
    b = torch.randn(C, generator=g) * 0.1
    out_div = 3.0 if div else 0.0
    xg, rg, ag = x.cuda(), res.cuda(), acc.cuda()

    def run(r):
        return ops.amp_conv_tc(xg, fa["a.act.alpha"], fa["a.act.beta"], fa["a.upsample.filter"],
                               fa["a.downsample.lowpass.filter"], w, b.cuda(), dilation=dil,
                               res=r if with_res else None, acc=ag if accum else None, out_div=out_div)

    got = run(rg)
    again = run(rg)
    generic = run(_unaligned(rg))
    torch.cuda.synchronize()
    assert torch.equal(got, again)
    assert torch.equal(got, generic)
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
