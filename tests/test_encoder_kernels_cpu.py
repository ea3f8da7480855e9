"""The gates of tests/test_encoder_kernels_gpu.py can tell a wrong kernel from fp32 rounding: on the same inputs, at the
smallest shapes and at the largest K, each named near-miss reference (what a subtly wrong kernel would store) fails its
gate by 10x or more on some element.  fp64 on the host, no GPU."""
import math

import pytest
import torch

from tests import test_encoder_kernels_gpu as E

MISS = 10.0


def worst_f32(v_miss, v, gate):
    return float(E.ratio_gate(v_miss.float(), v, gate).max())


def worst_bf16(v_miss, v, e):
    return float(E.ratio_bf16(v_miss.bfloat16(), v, e).max())


@pytest.mark.parametrize("M,N,K", [(1, 256, 64), (129, 256, 5120)])
def test_gate_catches_a_dropped_ktile(M, N, K):
    A, W, b = E.gemm_operands(M, N, K, seed=M + N + K)
    acc, S = E.gemm64(A, W, b, "cpu")
    miss, _ = E.gemm64(A, W, b, "cpu", drop_ktile=K // 64 - 1)
    assert worst_f32(miss, acc, E.TAU * S) >= MISS                       # epilogue 2
    v, vm = E.gelu64(acc), E.gelu64(miss)
    assert worst_bf16(vm, v, E.gelu_gate(S, v)) >= MISS                  # epilogue 1
    assert worst_bf16(miss, acc, E.TAU * S) >= MISS                      # epilogue 4


@pytest.mark.parametrize("M,N,K", [(1, 256, 64), (129, 256, 5120)])
def test_gate_catches_a_shifted_bias(M, N, K):
    A, W, b = E.gemm_operands(M, N, K, seed=M + N + K)
    acc, S = E.gemm64(A, W, b, "cpu")
    miss, _ = E.gemm64(A, W, b, "cpu", bias_shift=1)
    assert worst_f32(miss, acc, E.TAU * S) >= MISS
    v, vm = E.gelu64(acc), E.gelu64(miss)
    assert worst_bf16(vm, v, E.gelu_gate(S, v)) >= MISS


@pytest.mark.parametrize("n2,B,D", [(1, 3, 256), (127, 1, 1280)])
def test_gate_catches_res_mod_off_by_one(n2, B, D):
    """Epilogue 3 reading res[(m mod n2) + 1]: the next row of the table (NaN past n2)."""
    M, N, K = B * n2, D, 3 * D
    A, W, b = E.gemm_operands(M, N, K, seed=n2 + B + D)
    tab = torch.randn(n2 + 5, N, generator=torch.Generator().manual_seed(n2)).double()
    tab[n2:] = math.nan
    acc, S = E.gemm64(A, W, b, "cpu")
    m = torch.arange(M)
    g = E.gelu64(acc)
    v, rr = g + tab[m % n2], tab[m % n2].abs()
    assert worst_f32(g + tab[m % n2 + 1], v, E.gelu_gate(S, v, rr)) >= MISS


@pytest.mark.parametrize("n", [3, 255])
def test_gate_catches_conv2_last_position_reading_gelu_bias(n):
    """Epilogue 5 with odd item lengths F_b < n: conv2's last position (t = F_b tap) holding GELU(bias) instead of 0."""
    lens = E.conv2_lens(n)
    assert any(f % 2 == 1 and f < n for f in lens)
    M, N, K = len(lens) * n, 256, 256
    A, W, b = E.gemm_operands(M, N, K, seed=n + N)
    acc, S = E.gemm64(A, W, b, "cpu")
    idx, v, e = E.conv2_image_ref(acc, S, n, lens, N, "cpu")
    idx_m, v_m, _ = E.conv2_image_ref(acc, S, n, lens, N, "cpu", last_reads_bias=b)
    assert torch.equal(idx, idx_m)
    assert worst_bf16(v_m, v, e) >= MISS


ATT_CASES = [(2, 1, [1, 2]), (65, 1, [64, 65]), (1500, 1, [1499, 1500])]


@pytest.mark.parametrize("T,H,lens", ATT_CASES)
def test_gate_catches_key_tb_unmasked(T, H, lens):
    q, k, v = E.attn_inputs(len(lens), T, H, lens, seed=T)
    refs = E.attn_ref(q, k, v, lens, "cpu")
    miss = E.attn_ref(q, k, v, lens, "cpu", nkeys=lambda tb: min(tb + 1, T))
    worst = max(float(E.ratio_gate(m.float(), r, g).max()) for (r, g), (m, _), tb in zip(refs, miss, lens) if tb < T)
    assert worst >= MISS


@pytest.mark.parametrize("T,H,lens", ATT_CASES)
def test_gate_catches_key_tb_minus_1_masked(T, H, lens):
    q, k, v = E.attn_inputs(len(lens), T, H, lens, seed=T)
    refs = E.attn_ref(q, k, v, lens, "cpu")
    miss = E.attn_ref(q, k, v, lens, "cpu", nkeys=lambda tb: tb - 1)
    for (r, g), (m, _) in zip(refs, miss):
        assert float(E.ratio_gate(m.float(), r, g).max()) >= MISS


@pytest.mark.parametrize("M,D", [(1, 256), (9, 2048)])
def test_gate_catches_layernorm_without_eps(M, D):
    x, gamma, beta = E.ln_inputs(M, D, seed=M + D)
    ref, gate = E.ln_ref(x, gamma, beta)
    miss, _ = E.ln_ref(x, gamma, beta, eps=0.0)
    assert float(E.ratio_gate(miss.float(), ref, gate).max()) >= MISS


def test_gates_pass_the_reference_rounded_once():
    """The other side: the fp64 value rounded once to the output type passes every gate."""
    A, W, b = E.gemm_operands(129, 256, 5120, seed=3)
    acc, S = E.gemm64(A, W, b, "cpu")
    v = E.gelu64(acc)
    assert float(E.ratio_gate(acc.float(), acc, E.TAU * S).max()) <= 1.0
    assert bool(E.ok_bf16(v.bfloat16(), v, E.gelu_gate(S, v)).all())
    assert float(E.ratio_bf16(v.bfloat16(), v, E.gelu_gate(S, v)).max()) <= 1.0
    x, gamma, beta = E.ln_inputs(9, 2048, seed=1)
    ref, gate = E.ln_ref(x, gamma, beta)
    assert float(E.ratio_gate(ref.float(), ref, gate).max()) <= 1.0
