"""The encoders' bf16 tensor-core layer on its own, against fp64 (csrc/whisper_gemm.cu, csrc/whisper_attn_tc.cu).

These kernels have a near-exact contract: operands are bf16, so every product is exact in fp32; sums are fp32; each
store rounds once.  An fp64 evaluation of the same bf16 values is therefore a reference against which the gates can
be tight:
  * S = sum_k |a_k w_k| + |bias| (+ |res|) per output; tau = 2^-17.
  * fp32 outputs: |got - ref| <= tau S; after GELU, tau (1.13 S + |res|) + 2^-21 |ref| (1.13 bounds |GELU'|, the
    2^-21 term covers erff).
  * bf16 outputs: got is the round-to-nearest-even of the fp64 value; where that value lies within the fp32 bound of
    a rounding midpoint, either neighbour passes (got in [bf16(ref - e), bf16(ref + e)]).
  * attention: |got - ref| <= 2^-8 (sum_k p_k |v_kd| + |ref_d|), the bf16 rounding of P and of the output, 2x margin.
  * ln_rows: |got - ref| <= 2^-18 (|gamma| (1 + (|mu| + |x - mu|) / s) + |beta|), s = sqrt(var + 1e-5).
Every output lives in a guarded allocation filled with a NaN sentinel bit pattern: entries the contract writes must
hold their values, every other entry (guard bands included) must still hold the sentinel, so a stray store shows up
as a value.  Each case prints its worst err / gate ratio.  tests/test_encoder_kernels_cpu.py shows, without a GPU,
that named near-miss references fail these gates by 10x or more."""
import ctypes
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

TAU = 2.0 ** -17
GELU_SLOPE = 1.13
ERF_REL = 2.0 ** -21
ATT_REL = 2.0 ** -8
LN_REL = 2.0 ** -18
LN_EPS = 1e-5
SENT = {torch.bfloat16: 0x7FA5, torch.float32: 0x7FA5A5A5}   # quiet-NaN payloads no kernel produces
BITS = {torch.bfloat16: torch.int16, torch.float32: torch.int32}
GUARD = 8192   # guard elements before and after every output


# ----------------------------------------------------------------------------- layouts, restated from the kernels
def img_off(m, k, KT):
    """Element offset of (row m, column k) in a tile image with KT 64-wide k-tiles per 128-row tile
    (csrc/whisper_gemm.cu:49-51, img_off)."""
    return ((m >> 7) * KT + (k >> 6)) * (128 * 64) + ((k & 63) >> 3) * (128 * 8) + (m & 127) * 8 + (k & 7)


def qkv_heads_off(b, w, h, t, d, heads, Tp):
    """Element offset of (item b, q|k|v w, head h, position t, dim d) in the attention kernel's head-major QKV
    (csrc/common.cuh:374-378, qkv_heads_off): q blocks [Tp/128][8][128][8], k and v blocks [Tp/64][8][64][8]."""
    base = ((b * 3 + w) * heads + h) * Tp * 64
    q = base + (t >> 7) * 8192 + (d >> 3) * 1024 + (t & 127) * 8 + (d & 7)
    kv = base + (t >> 6) * 4096 + (d >> 3) * 512 + (t & 63) * 8 + (d & 7)
    return torch.where(w == 0, q, kv)


def tiles(M):
    return (M + 127) // 128 * 128


def ref_device(flops):
    """fp64 references on the host; the largest ones as a device fp64 matmul."""
    return "cuda" if flops > 2 ** 29 and torch.cuda.is_available() else "cpu"


# ----------------------------------------------------------------------------- inputs and fp64 references
def gemm_operands(M, N, K, seed, bias=True):
    """A [M, K], W [N, K] drawn in fp32 and rounded to bf16 (both sides use those values); bias fp32 [N] or None."""
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(M, K, generator=g).bfloat16()
    W = (torch.randn(N, K, generator=g) / math.sqrt(K)).bfloat16()
    b = 0.5 * torch.randn(N, generator=g) if bias else None
    return A, W, b


def gemm64(A, W, bias, dev, drop_ktile=None, bias_shift=0):
    """(acc + bias, S = sum |a w| + |bias|) in fp64 on dev.  Near misses: drop_ktile leaves out the products of one
    64-wide k-tile, bias_shift reads bias[n - bias_shift]; S is always that of the true operation."""
    A64, W64 = A.to(dev, torch.float64), W.to(dev, torch.float64)
    acc = A64 @ W64.T
    S = A64.abs() @ W64.abs().T
    if drop_ktile is not None:
        ks = slice(64 * drop_ktile, 64 * drop_ktile + 64)
        acc = acc - A64[:, ks] @ W64[:, ks].T
    if bias is not None:
        b64 = bias.to(dev, torch.float64)
        acc = acc + torch.roll(b64, bias_shift)
        S = S + b64.abs()
    return acc, S


def gelu64(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def gelu_gate(S, v, res_abs=0.0):
    return TAU * (GELU_SLOPE * S + res_abs) + ERF_REL * v.abs()


def half_ulp_bf16(v):
    _, e = torch.frexp(v)
    return torch.ldexp(torch.ones_like(v), (e - 9).to(torch.int32))


def ratio_bf16(got, v, e):
    """|got - v| / (half a bf16 ulp + e): <= 1 for a correctly rounded store."""
    g = got.to(v.device, torch.float64)
    r = (g - v).abs() / (half_ulp_bf16(v) + e)
    return torch.where(torch.isfinite(g), r, torch.full_like(r, math.inf))


def ok_bf16(got, v, e):
    g = got.to(v.device, torch.float64)
    lo, hi = (v - e).bfloat16().double(), (v + e).bfloat16().double()
    return (g >= lo) & (g <= hi)


def ratio_gate(got, v, gate):
    """|got - v| / gate; an exact reference (gate 0) must be met exactly; a non-finite got never passes."""
    g = got.to(v.device, torch.float64)
    err = (g - v).abs()
    r = torch.where(gate > 0, err / torch.where(gate > 0, gate, torch.ones_like(gate)),
                    torch.where(err == 0, torch.zeros_like(err), torch.full_like(err, math.inf)))
    return torch.where(torch.isfinite(g), r, torch.full_like(r, math.inf))


# epilogue 5: conv1's frames (b, t) land in conv2's im2col image at (b n2 + t2, j N + co) with t = 2 t2 + j - 1
def conv2_taps(n, n2):
    """(frame t, position t2, tap j) for every entry the scatter writes (csrc/whisper_gemm.cu epilogue 5)."""
    t = torch.arange(n)
    ev, od = t[t % 2 == 0], t[t % 2 == 1]
    a = od[(od + 1) // 2 < n2]
    ts = torch.cat([ev, a, od])
    t2 = torch.cat([ev // 2, (a + 1) // 2, (od - 1) // 2])
    j = torch.cat([torch.ones_like(ev), torch.zeros_like(a), torch.full_like(od, 2)])
    return ts, t2, j


def conv2_image_ref(acc, S, n, lens, N, dev, last_reads_bias=None):
    """Flat image offsets, fp64 values and gates of the entries epilogue 5 writes.  Frames t >= lens[b] are zeros
    (exact).  Near miss last_reads_bias (a bias [N]): for items with odd lens[b] < n, the last position's t = lens[b]
    tap holds GELU(bias) instead of 0."""
    B, n2 = len(lens), (n - 1) // 2 + 1
    ts, t2, j = [x.to(dev) for x in conv2_taps(n, n2)]
    co = torch.arange(N, device=dev)
    idx, vals, gates = [], [], []
    for b in range(B):
        rows = b * n + ts
        v = gelu64(acc[rows])
        e = gelu_gate(S[rows], v)
        past = (ts >= lens[b])[:, None]
        v = torch.where(past, torch.zeros_like(v), v)
        e = torch.where(past, torch.zeros_like(e), e)
        if last_reads_bias is not None and lens[b] % 2 == 1 and lens[b] < n:
            sel = (ts == lens[b]) & (j == 2)
            v[sel] = gelu64(last_reads_bias.to(dev, torch.float64))[None, :]
        idx.append(img_off((b * n2 + t2)[:, None], (j * N)[:, None] + co[None, :], 3 * N // 64))
        vals.append(v)
        gates.append(e)
    return torch.cat(idx).flatten(), torch.cat(vals).flatten(), torch.cat(gates).flatten()


def attn_inputs(B, T, heads, lens, seed, junk=0):
    """q, k, v [B, heads, T, 64] bf16 that make a mask error large: keys [T_b, T) score at least 30 above every valid
    score (k[0] = 512 against q[0] = 1) and carry v = +-300; in the even query rows the last valid key has the
    largest score (q[1] = k[1] = 8: +8).  junk = 1 fills rows [T_b, T) of k and v with other values."""
    g = torch.Generator().manual_seed(seed)
    q = 0.5 * torch.randn(B, heads, T, 64, generator=g)
    k = 0.5 * torch.randn(B, heads, T, 64, generator=g)
    v = torch.randn(B, heads, T, 64, generator=g)
    q[..., 0] = 1.0
    q[..., 1] = 0.0
    q[:, :, ::2, 1] = 8.0
    k[..., 1] = 0.0
    for b, tb in enumerate(lens):
        k[b, :, tb - 1, 1] = 8.0
        if tb < T:
            if junk == 0:
                k[b, :, tb:] = 0.0
                k[b, :, tb:, 0] = 512.0
                v[b, :, tb:] = 300.0 * torch.where(torch.rand(heads, T - tb, 64, generator=g) < 0.5, -1.0, 1.0)
            else:
                k[b, :, tb:] = 4.0 * torch.randn(heads, T - tb, 64, generator=g)
                v[b, :, tb:] = 1000.0 * torch.randn(heads, T - tb, 64, generator=g)
    return q.bfloat16(), k.bfloat16(), v.bfloat16()


def attn_ref(q, k, v, lens, dev, nkeys=None):
    """Per item: fp64 softmax(q k^T / 8) v of query rows [0, T_b) over the first nkeys(T_b) keys (default T_b), and
    the gate 2^-8 (sum_k p_k |v_kd| + |ref_d|) of the true operation."""
    out = []
    for b, tb in enumerate(lens):
        qb, kb, vb = (x[b].to(dev, torch.float64) for x in (q, k, v))
        p = torch.softmax(qb[:, :tb] @ kb[:, :tb].transpose(-1, -2) / 8.0, dim=-1)
        ref = p @ vb[:, :tb]
        gate = ATT_REL * (p @ vb[:, :tb].abs() + ref.abs())
        nk = tb if nkeys is None else nkeys(tb)
        if nk != tb:
            if nk <= 0:
                ref = torch.full_like(ref, math.nan)
            else:
                pm = torch.softmax(qb[:, :tb] @ kb[:, :nk].transpose(-1, -2) / 8.0, dim=-1)
                ref = pm @ vb[:, :nk]
        out.append((ref, gate))
    return out


def ln_inputs(M, D, seed):
    """Rows by kind (row i is kind i % 4): constant, N(0, 1), mean 1e3 with sigma 0.1, N(0, 1) with one 1e4 outlier.
    The constants are multiples of 1/16, so that their fp32 sums are exact and the mean is within an ulp."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, D, generator=g)
    kind = torch.arange(M) % 4
    x[kind == 0] = (torch.round(48.0 * torch.randn(M, 1, generator=g)) / 16.0).expand(M, D)[kind == 0]
    x[kind == 2] = 1e3 + 0.1 * x[kind == 2]
    rows = torch.nonzero(kind == 3).flatten()
    x[rows, (rows * 37) % D] = 1e4
    gamma = 1.0 + 0.5 * torch.randn(D, generator=g)
    beta = 0.5 * torch.randn(D, generator=g)
    return x, gamma, beta


def ln_ref(x, gamma, beta, eps=LN_EPS):
    """fp64 LayerNorm and the gate 2^-18 (|gamma| (1 + (|mu| + |x - mu|) / s) + |beta|) with the true eps."""
    x64, g64, b64 = x.double(), gamma.double(), beta.double()
    mu = x64.mean(1, keepdim=True)
    var = ((x64 - mu) ** 2).mean(1, keepdim=True)
    y = (x64 - mu) / torch.sqrt(var + eps) * g64 + b64
    s = torch.sqrt(var + LN_EPS)
    gate = LN_REL * (g64.abs() * (1.0 + (mu.abs() + (x64 - mu).abs()) / s) + b64.abs())
    return y, gate


# ----------------------------------------------------------------------------- device side
def _lib():
    from whisper_vits_svc_b200 import _lib as L
    return L


def guarded(n, dtype):
    """A device buffer of GUARD + n + GUARD elements, all holding the sentinel; the contract's region starts at GUARD."""
    buf = torch.empty(n + 2 * GUARD, dtype=dtype, device="cuda")
    buf.view(BITS[dtype]).fill_(SENT[dtype])
    return buf


def inner_ptr(buf, off=0):
    return buf.data_ptr() + (GUARD + off) * buf.element_size()


def check_store(buf, idx, v, gate, bf16, what):
    """The entries idx (offsets from the region's start) of a guarded buffer hold v within gate (bf16: correctly
    rounded), every other entry of the allocation holds the sentinel.  Prints and returns the worst ratio."""
    dev = v.device
    flat = buf.to(dev)
    idx = idx.to(dev) + GUARD
    got = flat[idx]
    if bf16:
        ratio = ratio_bf16(got, v, gate)
        bad = ~ok_bf16(got, v, gate) | ~torch.isfinite(got.double())
    else:
        ratio = ratio_gate(got, v, gate)
        bad = ratio > 1
    keep = torch.ones(flat.numel(), dtype=torch.bool, device=dev)
    keep[idx] = False
    stray = int((flat.view(BITS[buf.dtype])[keep] != SENT[buf.dtype]).sum())
    worst = float(ratio.max()) if ratio.numel() else 0.0
    print(f"{what}: worst err/gate {worst:.3f} over {idx.numel()} entries")
    assert int(bad.sum()) == 0, f"{what}: {int(bad.sum())} entries outside the gate (worst ratio {worst:.3g})"
    assert stray == 0, f"{what}: {stray} entries outside the contract were written"
    assert int(torch.unique(idx).numel()) == idx.numel(), f"{what}: the expected stores overlap"
    return worst


def run_gemm(A, W, bias, out_ptr, res_ptr, epi, res_mod=0, aux=0, lens=None):
    L = _lib()
    lib = L.load()
    M, K = A.shape
    N = W.shape[0]
    Ad, Wd = A.cuda(), W.cuda()
    bd = bias.cuda() if bias is not None else None
    scratch = torch.empty(int(lib.svcb_op_gemm_bf16_scratch_bytes(M, N, K)), dtype=torch.uint8, device="cuda")
    lens_c = (ctypes.c_int32 * len(lens))(*lens) if lens is not None else None
    st = lib.svcb_op_gemm_bf16(Ad.data_ptr(), Wd.data_ptr(), bd.data_ptr() if bd is not None else None, out_ptr, res_ptr,
                               M, N, K, epi, res_mod, aux, lens_c, scratch.data_ptr(), scratch.numel(), L.stream())
    L.check(st, "svcb_op_gemm_bf16")
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------- GEMM epilogues
@pytest.mark.parametrize("M,N,K", [(1, 1024, 256), (129, 3072, 768), (3000, 5120, 1280), (129, 5120, 256),
                                   (3000, 1024, 768), (1, 3072, 1280)])
def test_epi1_gelu_bf16_image(M, N, K):
    """GELU -> the bf16 tile image of the next GEMM's A; image rows >= M (pad rows of the last tile) are not written."""
    A, W, b = gemm_operands(M, N, K, seed=M + N + K)
    buf = guarded(tiles(M) * N, torch.bfloat16)
    run_gemm(A, W, b, inner_ptr(buf), None, 1)
    dev = ref_device(M * N * K)
    acc, S = gemm64(A, W, b, dev)
    v = gelu64(acc)
    m, n = torch.arange(M, device=dev), torch.arange(N, device=dev)
    check_store(buf, img_off(m[:, None], n[None, :], N // 64).flatten(), v.flatten(), gelu_gate(S, v).flatten(), True,
                f"epi 1 M={M} N={N} K={K}")


@pytest.mark.parametrize("M,N,K,res", [(1, 256, 64, "res"), (127, 1280, 128, "none"), (128, 256, 320, "alias"),
                                       (129, 1280, 5120, "res"), (129, 256, 5120, "alias"), (24000, 1280, 64, "alias"),
                                       (24000, 256, 128, "res"), (24000, 1280, 320, "none")])
def test_epi2_fp32_residual(M, N, K, res):
    """fp32 acc + bias (+ res): res null, a separate res, and res == out as the encoders' residual GEMMs call it.  The
    24000-row cases have more tiles than SMs at K / 64 = 1, 2 and 5 k-tiles, so the producer's ring phase carries
    across tiles."""
    A, W, b = gemm_operands(M, N, K, seed=7 * M + N + K)
    r = torch.randn(M, N, generator=torch.Generator().manual_seed(M + K))
    buf = guarded(M * N, torch.float32)
    rd = None
    if res == "alias":
        buf[GUARD:GUARD + M * N] = r.flatten().cuda()
        res_ptr = inner_ptr(buf)
    elif res == "res":
        rd = r.cuda()
        res_ptr = rd.data_ptr()
    else:
        res_ptr = None
    run_gemm(A, W, b, inner_ptr(buf), res_ptr, 2)
    dev = ref_device(M * N * K)
    acc, S = gemm64(A, W, b, dev)
    if res != "none":
        r64 = r.to(dev, torch.float64)
        acc, S = acc + r64, S + r64.abs()
    check_store(buf, torch.arange(M * N, device=dev), acc.flatten(), (TAU * S).flatten(), False,
                f"epi 2 M={M} N={N} K={K} res={res}")


@pytest.mark.parametrize("n2,B,D,res", [(1, 3, 256, True), (64, 3, 256, True), (127, 1, 1280, True), (750, 3, 256, True),
                                        (1500, 1, 1280, True), (1500, 3, 256, True), (127, 3, 256, False),
                                        (750, 1, 1280, False)])
def test_epi3_gelu_add_rows_mod(n2, B, D, res):
    """fp32 GELU(acc + bias) + res[m mod n2]: the stem's conv2 with the positional table (K = 3 D).  Table rows >= n2
    are NaN, so a wrong row index shows as a non-finite output.  res null: the plain GELU rows HuBERT's conv6 writes."""
    M, N, K = B * n2, D, 3 * D
    A, W, b = gemm_operands(M, N, K, seed=n2 + B + D)
    buf = guarded(M * N, torch.float32)
    tab = torch.randn(n2 + 5, N, generator=torch.Generator().manual_seed(n2))
    tab[n2:] = math.nan
    td = tab.cuda()
    run_gemm(A, W, b, inner_ptr(buf), td.data_ptr() if res else None, 3, res_mod=n2 if res else 0)
    dev = ref_device(M * N * K)
    acc, S = gemm64(A, W, b, dev)
    v = gelu64(acc)
    if res:
        rr = tab.to(dev, torch.float64)[torch.arange(M, device=dev) % n2]
        v, gate = v + rr, gelu_gate(S, v + rr, rr.abs())
    else:
        gate = gelu_gate(S, v)
    check_store(buf, torch.arange(M * N, device=dev), v.flatten(), gate.flatten(), False,
                f"epi 3 n2={n2} B={B} D={D} res={res}")


@pytest.mark.parametrize("T,D,B", [(1, 256, 3), (63, 768, 2), (64, 1280, 2), (65, 256, 3), (128, 768, 2), (129, 1280, 2),
                                   (1500, 768, 2), (1500, 256, 1)])
def test_epi4_qkv_heads(T, D, B):
    """bf16 acc + bias in the head-major QKV layout: q panels of 128 positions, k and v panels of 64; positions
    [T, Tp) of every panel are not written."""
    M, N, K, heads, Tp = B * T, 3 * D, D, D // 64, tiles(T)
    A, W, b = gemm_operands(M, N, K, seed=T + D + B)
    buf = guarded(B * Tp * 3 * D, torch.bfloat16)
    run_gemm(A, W, b, inner_ptr(buf), None, 4, res_mod=T)
    dev = ref_device(M * N * K)
    acc, S = gemm64(A, W, b, dev)
    m, n = torch.arange(M, device=dev)[:, None], torch.arange(N, device=dev)[None, :]
    idx = qkv_heads_off(m // T, n // D, (n % D) // 64, m % T, n % 64, heads, Tp)
    check_store(buf, idx.flatten(), acc.flatten(), (TAU * S).flatten(), True, f"epi 4 T={T} D={D} B={B}")


def conv2_lens(n):
    """Item lengths with 1, 2, odd, even and n frames."""
    out = []
    for x in (n, 1, 2, 3, 2 * (n // 4) + 1, max(2, 2 * (n // 4))):
        x = min(max(x, 1), n)
        if x not in out:
            out.append(x)
    return out


@pytest.mark.parametrize("n,D", [(1, 256), (2, 256), (3, 256), (255, 1280), (256, 256), (3000, 256)])
@pytest.mark.parametrize("init", ["zero", "sentinel"])
def test_epi5_conv1_into_conv2_image(n, D, init):
    """conv1's GELU scattered into conv2's im2col image, lens ragged (items of 1, 2, odd, even and n frames).
    zero: the image zeroed first, as the encoder does, must equal bf16(GELU(h1)) im2col with zeros at t = -1,
    t >= lens, t >= n.  sentinel: exactly the t = -1 taps, the t = n tap of odd n and the pad rows stay unwritten, and
    frames [lens, n) are written as exact zeros."""
    lens = conv2_lens(n)
    B, n2, K = len(lens), (n - 1) // 2 + 1, 256
    M, N = B * n, D
    A, W, b = gemm_operands(M, N, K, seed=n + D)
    size = tiles(B * n2) * 3 * N
    buf = guarded(size, torch.bfloat16)
    if init == "zero":
        buf[GUARD:GUARD + size] = 0
    run_gemm(A, W, b, inner_ptr(buf), None, 5, res_mod=n, lens=lens)
    dev = ref_device(M * N * K)
    acc, S = gemm64(A, W, b, dev)
    idx, v, e = conv2_image_ref(acc, S, n, lens, N, dev)
    if init == "zero":   # every other entry of the image is a zero
        full_v = torch.zeros(size, dtype=torch.float64, device=dev)
        full_e = torch.zeros(size, dtype=torch.float64, device=dev)
        full_v[idx], full_e[idx] = v, e
        idx, v, e = torch.arange(size, device=dev), full_v, full_e
    check_store(buf, idx, v, e, True, f"epi 5 n={n} D={D} lens={lens} init={init}")


@pytest.mark.parametrize("aux", [2, 3])
@pytest.mark.parametrize("frames_of", ["aux", "aux+1", "64", "257", "1000"])
def test_epi6_valid_stride2_scatter(aux, frames_of):
    """GELU scattered into the next stride-2 valid conv's im2col image (HuBERT's stem, bias null as there): every
    entry of rows < B Tn is written, the image's later rows are not."""
    nfr = {"aux": aux, "aux+1": aux + 1}.get(frames_of) or int(frames_of)
    B, N, K = 2, 512, 1536
    M, Tn = B * nfr, (nfr - aux) // 2 + 1
    A, W, _ = gemm_operands(M, N, K, seed=nfr + aux, bias=False)
    buf = guarded(tiles(B * Tn) * aux * N, torch.bfloat16)
    run_gemm(A, W, None, inner_ptr(buf), None, 6, res_mod=nfr, aux=aux)
    dev = ref_device(M * N * K)
    acc, S = gemm64(A, W, None, dev)
    r = torch.arange(B * Tn, device=dev)
    bi, t2 = r // Tn, r % Tn
    j = torch.arange(aux, device=dev)
    co = torch.arange(N, device=dev)
    src = (bi * nfr + 2 * t2)[:, None] + j[None, :]          # [rows, aux] source rows of the GEMM
    v = gelu64(acc[src])                                     # [rows, aux, N]
    e = gelu_gate(S[src], v)
    idx = img_off(r[:, None, None], (j * N)[None, :, None] + co[None, None, :], aux * N // 64)
    check_store(buf, idx.flatten(), v.flatten(), e.flatten(), True, f"epi 6 aux={aux} frames={nfr}")


@pytest.mark.parametrize("c0,M", [(0, 300), (336, 129), (720, 1)])
def test_epi7_grouped_conv_stripe(c0, M):
    """fp32 GELU(acc + bias) + res over the first 48 of 256 columns, rows 768 apart (one group of HuBERT's positional
    conv, called with out = y + c0 and res = x + c0): columns outside [c0, c0 + 48) of every row are not written."""
    N, K, cg, ld = 256, 6144, 48, 768
    A, W, b = gemm_operands(M, N, K, seed=c0 + M)
    x = torch.randn(M, ld, generator=torch.Generator().manual_seed(c0))
    xd = x.cuda()
    buf = guarded(M * ld, torch.float32)
    run_gemm(A, W, b, inner_ptr(buf, c0), xd.data_ptr() + 4 * c0, 7, res_mod=cg, aux=ld)
    dev = ref_device(M * N * K)
    acc, S = gemm64(A, W, b, dev)
    rr = x.to(dev, torch.float64)[:, c0:c0 + cg]
    v = gelu64(acc[:, :cg]) + rr
    gate = gelu_gate(S[:, :cg], v, rr.abs())
    m, c = torch.arange(M, device=dev)[:, None], torch.arange(cg, device=dev)[None, :]
    check_store(buf, (m * ld + c0 + c).flatten(), v.flatten(), gate.flatten(), False, f"epi 7 c0={c0} M={M}")


def test_gemm_rejects_epilogue_0_and_8():
    L = _lib()
    lib = L.load()
    A, W, b = gemm_operands(1, 256, 64, seed=1)
    buf = guarded(128 * 256, torch.float32)
    for epi in (0, 8):
        with pytest.raises(L.SvcbError):
            run_gemm(A, W, b, inner_ptr(buf), None, epi)
        assert (buf.view(torch.int32) == SENT[torch.float32]).all()
    assert "epilogue must be 1..7" in lib.svcb_last_error().decode()


# ----------------------------------------------------------------------------- attention
def run_attention(q, k, v, lens, v_layout=0):
    L = _lib()
    lib = L.load()
    B, H, T, _ = q.shape
    D = 64 * H
    qkv = torch.stack([q, k, v]).permute(1, 3, 0, 2, 4).reshape(B * T, 3 * D).cuda()
    buf = guarded(B * T * D, torch.bfloat16)
    scratch = torch.empty(int(lib.svcb_op_attention_tc_bf16_scratch_bytes(B, T, D)), dtype=torch.uint8, device="cuda")
    lens_c = (ctypes.c_int32 * B)(*lens) if lens is not None else None
    st = lib.svcb_op_attention_tc_bf16(qkv.data_ptr(), inner_ptr(buf), B, T, D, H, v_layout, lens_c, scratch.data_ptr(),
                                       scratch.numel(), L.stream())
    L.check(st, "svcb_op_attention_tc_bf16")
    torch.cuda.synchronize()
    return buf


def attn_worst(buf, refs, lens, T, H, what):
    """Rows < T_b of each item within the gate; rows of query tiles wholly past T_b exact zeros; rows [T_b, T) of a
    partly valid tile finite; the guard bands untouched."""
    D = 64 * H
    out = buf[GUARD:GUARD + len(lens) * T * D].view(len(lens), T, H, 64).permute(0, 2, 1, 3)
    worst = 0.0
    for b, (tb, (ref, gate)) in enumerate(zip(lens, refs)):
        got = out[b, :, :tb].to(ref.device)
        r = ratio_gate(got, ref, gate)
        worst = max(worst, float(r.max()))
        assert float(r.max()) <= 1.0, f"{what} item {b} (T_b={tb}): worst ratio {float(r.max()):.3g}"
        live = tiles(tb)
        assert torch.isfinite(out[b, :, tb:min(live, T)].float()).all(), f"{what} item {b}: non-finite rows in [T_b, tile end)"
        assert (out[b, :, live:].float() == 0).all(), f"{what} item {b}: query tiles past T_b are not zeros"
    bits = buf.view(torch.int16)
    assert (bits[:GUARD] == SENT[torch.bfloat16]).all() and (bits[-GUARD:] == SENT[torch.bfloat16]).all()
    print(f"{what}: worst err/gate {worst:.3f}")
    return worst


@pytest.mark.parametrize("heads", [1, 4, 20])
@pytest.mark.parametrize("T", [1, 2, 63, 64, 65, 127, 128, 129, 191, 1500])
def test_attention_lens_vs_fp64(T, heads):
    """One item per T_b in {1, 63, 64, 65, T} (those <= T) with lens, then two dense items without.  Rows < T_b are
    bitwise the same whatever rows [T_b, T) of k and v hold."""
    lens = sorted({x for x in (1, 63, 64, 65, T) if x <= T})
    dev = ref_device(len(lens) * heads * T * T * 128)
    q, k, v = attn_inputs(len(lens), T, heads, lens, seed=T + heads)
    for b, tb in enumerate(lens):   # the inputs make a mask error large
        if tb < T:
            sc = (q[b].to(dev, torch.float64) @ k[b].to(dev, torch.float64).transpose(-1, -2)) / 8.0
            assert float(sc[:, :, tb:].min() - sc[:, :, :tb].max()) >= 30.0
    buf = run_attention(q, k, v, lens)
    attn_worst(buf, attn_ref(q, k, v, lens, dev), lens, T, heads, f"attention T={T} heads={heads} lens={lens}")
    q2, k2, v2 = attn_inputs(len(lens), T, heads, lens, seed=T + heads, junk=1)
    assert torch.equal(q2, q)
    buf2 = run_attention(q2, k2, v2, lens)
    D = 64 * heads
    a = buf[GUARD:GUARD + len(lens) * T * D].view(len(lens), T, D)
    a2 = buf2[GUARD:GUARD + len(lens) * T * D].view(len(lens), T, D)
    for b, tb in enumerate(lens):
        assert torch.equal(a[b, :tb].view(torch.int16), a2[b, :tb].view(torch.int16)), f"item {b}: rows < T_b depend on rows past T_b"
    dense = [T, T]
    qd, kd, vd = attn_inputs(2, T, heads, dense, seed=3 * T + heads)
    buf = run_attention(qd, kd, vd, None)
    attn_worst(buf, attn_ref(qd, kd, vd, dense, dev), dense, T, heads, f"attention T={T} heads={heads} dense")


def test_attention_v_descriptor_layout():
    """v_layout 1 exchanges LBO / SBO of the V descriptor: it must NOT match (pins the descriptor semantics the kernel
    relies on)."""
    B, T, H = 2, 100, 2
    lens = [T] * B
    q, k, v = attn_inputs(B, T, H, lens, seed=5)
    refs = attn_ref(q, k, v, lens, "cpu")
    good = run_attention(q, k, v, None, v_layout=0)
    attn_worst(good, refs, lens, T, H, "attention v_layout=0")
    bad = run_attention(q, k, v, None, v_layout=1)
    out = bad[GUARD:GUARD + B * T * H * 64].view(B, T, H, 64).permute(0, 2, 1, 3)
    worst = max(float(ratio_gate(out[b].cpu(), r, g).max()) for b, (r, g) in enumerate(refs))
    print(f"attention v_layout=1: worst err/gate {worst:.3g} (must fail)")
    assert worst > 10.0


# ----------------------------------------------------------------------------- ln_rows
@pytest.mark.parametrize("M", [1, 7, 8, 9, 129, 3000])
@pytest.mark.parametrize("D", [256, 512, 768, 1280, 2048])
def test_ln_rows_vs_fp64(D, M):
    """The bf16 tile image with fp32 rows (y32), and the fp32 mode (ln_post): y32 and the fp32 rows within the gate,
    the image bitwise y32.bfloat16(); rows >= M of every output (image pad rows included) are never written."""
    L = _lib()
    lib = L.load()
    x, gamma, beta = ln_inputs(M, D, seed=M + D)
    xd, gd, bd = x.cuda(), gamma.cuda(), beta.cuda()
    img = guarded(tiles(M) * D, torch.bfloat16)
    y32 = guarded(M * D, torch.float32)
    L.check(lib.svcb_op_ln_rows(xd.data_ptr(), gd.data_ptr(), bd.data_ptr(), inner_ptr(img), inner_ptr(y32), M, D, 1,
                                L.stream()), "svcb_op_ln_rows")
    rows = guarded(M * D, torch.float32)
    L.check(lib.svcb_op_ln_rows(xd.data_ptr(), gd.data_ptr(), bd.data_ptr(), inner_ptr(rows), None, M, D, 0, L.stream()),
            "svcb_op_ln_rows")
    torch.cuda.synchronize()
    ref, gate = ln_ref(x, gamma, beta)
    allidx = torch.arange(M * D)
    w1 = check_store(y32, allidx, ref.flatten(), gate.flatten(), False, f"ln_rows y32 D={D} M={M}")
    w2 = check_store(rows, allidx, ref.flatten(), gate.flatten(), False, f"ln_rows fp32 D={D} M={M}")
    got32 = y32[GUARD:GUARD + M * D].cpu()
    m, n = torch.arange(M)[:, None], torch.arange(D)[None, :]
    ioff = img_off(m, n, D // 64).flatten()
    check_store(img, ioff, got32.bfloat16().double(), torch.zeros(M * D, dtype=torch.float64), True,
                f"ln_rows image D={D} M={M}")
    assert max(w1, w2) <= 1.0


# ----------------------------------------------------------------------------- im2col writers
def im2col_s1_ref(mel, KT):
    B, nm, n = mel.shape
    Mp = tiles(B * n)
    A = torch.zeros(Mp, KT * 64)
    pad = torch.nn.functional.pad(mel, (1, 1))
    for j in range(3):
        A[:B * n, j * nm:(j + 1) * nm] = pad[:, :, j:j + n].permute(0, 2, 1).reshape(B * n, nm)
    return A.bfloat16()


def to_image(A, KT):
    """row-major [Mp, KT * 64] -> tile image, through the restated img_off"""
    Mp = A.shape[0]
    m, k = torch.arange(Mp)[:, None], torch.arange(KT * 64)[None, :]
    img = torch.empty(Mp * KT * 64, dtype=A.dtype)
    img[img_off(m, k, KT).flatten()] = A.flatten()
    return img


@pytest.mark.parametrize("B,n", [(1, 1), (2, 3), (3, 200), (2, 3000)])
def test_im2col_s1_image(B, n):
    """Whisper's conv1 im2col image of the log-mel: K = 240 padded to 256 with zeros, zero taps outside the item,
    the pad rows of the last tile zero."""
    L = _lib()
    lib = L.load()
    nm, KT = 80, 4
    mel = torch.randn(B, nm, n, generator=torch.Generator().manual_seed(n))
    size = tiles(B * n) * KT * 64
    buf = guarded(size, torch.bfloat16)
    L.check(lib.svcb_op_im2col_s1_image(mel.cuda().data_ptr(), inner_ptr(buf), B, nm, n, L.stream()), "svcb_op_im2col_s1_image")
    torch.cuda.synchronize()
    want = to_image(im2col_s1_ref(mel, KT), KT)
    got = buf.cpu()
    assert torch.equal(got[GUARD:GUARD + size].view(torch.int16), want.view(torch.int16))
    assert (got[:GUARD].view(torch.int16) == SENT[torch.bfloat16]).all()
    assert (got[GUARD + size:].view(torch.int16) == SENT[torch.bfloat16]).all()


@pytest.mark.parametrize("B,T,ld,c0,cg,taps,pad,lens", [(2, 100, 768, 336, 48, 128, 64, [100, 37]),
                                                         (2, 100, 768, 720, 48, 128, 64, None),
                                                         (3, 129, 64, 8, 16, 4, 2, [1, 129, 64]),
                                                         (1, 1, 768, 0, 48, 128, 64, [1])])
def test_im2col_rows_image(B, T, ld, c0, cg, taps, pad, lens):
    """One channel group of a 'same' conv over time-major rows [B T, ld]: offsets c0 and ld, zero taps outside
    [0, lens[b]), the pad rows of the last tile zero."""
    L = _lib()
    lib = L.load()
    x = torch.randn(B * T, ld, generator=torch.Generator().manual_seed(T + c0))
    K = taps * cg
    KT = K // 64
    size = tiles(B * T) * K
    buf = guarded(size, torch.bfloat16)
    scratch = torch.empty(4 * B, dtype=torch.uint8, device="cuda")
    lens_c = (ctypes.c_int32 * B)(*lens) if lens is not None else None
    L.check(lib.svcb_op_im2col_rows_image(x.cuda().data_ptr(), inner_ptr(buf), lens_c, B, T, ld, c0, cg, taps, pad,
                                          scratch.data_ptr(), scratch.numel(), L.stream()), "svcb_op_im2col_rows_image")
    torch.cuda.synchronize()
    A = torch.zeros(tiles(B * T), K)
    xs = x.view(B, T, ld)[:, :, c0:c0 + cg]
    for b in range(B):
        tb = T if lens is None else lens[b]
        for j in range(taps):
            t = torch.arange(T) + j - pad
            ok = (t >= 0) & (t < tb)
            A[b * T + torch.nonzero(ok).flatten(), j * cg:(j + 1) * cg] = xs[b, t[ok]]
    want = to_image(A.bfloat16(), KT)
    got = buf.cpu()
    assert torch.equal(got[GUARD:GUARD + size].view(torch.int16), want.view(torch.int16))
    assert (got[:GUARD].view(torch.int16) == SENT[torch.bfloat16]).all()
    assert (got[GUARD + size:].view(torch.int16) == SENT[torch.bfloat16]).all()
