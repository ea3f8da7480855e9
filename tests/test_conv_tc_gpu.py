"""The persistent conv_tc kernel's scheduling paths against F.conv1d (fp32 CPU): a batch whose tiles wrap the
grid several times, ragged last tiles of both tile heights (256 rows for N tiles up to 192 wide, 128 rows above),
three N tiles per t-tile, and precision 1."""
import pytest
import torch
import torch.nn.functional as F

from tests.util import max_abs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    from whisper_vits_svc_b200 import ops as o
    return o


@pytest.mark.parametrize("B,Cin,Cout,T,K,dil,nsplit,tol", [
    (32, 192, 384, 1000, 5, 1, 3, 2e-4),    # 256 tiles of 256 x 192: every CTA walks about two
    (3, 192, 192, 300, 3, 1, 3, 2e-4),      # ragged last 256-row tile
    (2, 192, 640, 700, 3, 1, 3, 2e-4),      # three 224-wide N tiles of 128 rows, ragged
    (5, 160, 160, 1000, 11, 5, 3, 2e-4),    # wide dilated reach
    (32, 192, 384, 333, 5, 1, 1, 5e-2)])
def test_conv_tc_schedule(ops, B, Cin, Cout, T, K, dil, nsplit, tol):
    g = torch.Generator().manual_seed(B + Cin + Cout + T + K)
    x = torch.randn(B, Cin, T, generator=g)
    w = torch.randn(Cout, Cin, K, generator=g) / (Cin * K) ** 0.5
    b = torch.randn(Cout, generator=g) * 0.1
    ref = F.conv1d(x, w, b, dilation=dil, padding=dil * (K - 1) // 2)
    got = ops.conv_tc(x.cuda(), w, b.cuda(), dilation=dil, nsplit=nsplit)
    err = max_abs(got, ref)
    print(f"conv_tc B={B} {Cin}->{Cout} T={T} K={K} d={dil} nsplit={nsplit}: max-abs {err:.3e}")
    assert err <= tol
