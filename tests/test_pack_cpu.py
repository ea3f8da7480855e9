"""Host packer: the re-laid-out weights mean what the kernels assume (checked with torch on CPU)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from whisper_vits_svc_b200 import pack


def unpack_conv(wp, cout):
    return wp[:, :, :cout].permute(2, 0, 1).contiguous()  # [Cin,K,CoutPad] -> [Cout,Cin,K]


def test_pack_conv_roundtrip():
    w = torch.randn(20, 7, 3)
    wp = pack.pack_conv(w)
    assert wp.shape == (7, 3, 24) and torch.equal(unpack_conv(wp, 20), w)
    assert torch.count_nonzero(wp[:, :, 20:]) == 0


@pytest.mark.parametrize("k,s", [(15, 5), (8, 4), (4, 2), (7, 3), (16, 8)])
def test_polyphase_transposed_conv(k, s):
    """ConvTranspose1d == `rate` stride-1 sub-convolutions written with output stride `rate`
    (csrc/api.cu run_generator uses exactly these q0 / nq formulas; phase r writes output q at q - q0)."""
    torch.manual_seed(k * 10 + s)
    cin, cout, T = 6, 4, 23
    w = torch.randn(cin, cout, k)
    b = torch.randn(cout)
    x = torch.randn(2, cin, T)
    p = (k - s) // 2
    ref = F.conv_transpose1d(x, w, b, stride=s, padding=p)
    Lout = ref.shape[-1]
    M = (k + s - 1) // s
    y = torch.zeros_like(ref)
    for r in range(s):
        sub = torch.zeros(cout, cin, M)
        for jp in range(M):
            j = r + s * (M - 1 - jp)
            if j < k:
                sub[:, :, jp] = w[:, :, j].t()
        pr = p - r
        q0 = (pr + s - 1) // s if pr > 0 else 0
        qmax = (Lout - 1 + p - r) // s
        nq = qmax - q0 + 1
        # generic kernel semantics: out[q] = sum_j x[q + j - (M-1)] * sub[j], zero outside [0,T)
        xp = F.pad(x, (M - 1 + 8, M + 8))
        full = F.conv1d(xp, sub, b)  # full[i] <-> q = i - 8
        for t in range(nq):
            q = q0 + t
            y[:, :, q * s + r - p] = full[:, :, q + 8]
    assert torch.allclose(y, ref, atol=1e-5), (y - ref).abs().max()


@pytest.mark.parametrize("k,s", [(8, 4), (4, 2), (16, 8)])
def test_ups_combined_is_the_transposed_conv(k, s):
    """pack.ups_combined: the polyphase sub-filters as ONE Conv1d with rate * Cout channels and M + 1 taps whose
    channel co * rate + slot at frame i is sample rate * i + slot of ConvTranspose1d (generator.py:183) —
    what csrc/conv_tc.cu's interleaved epilogue (ConvTcParams::ilv) stores."""
    torch.manual_seed(k + s)
    cin, cout, T = 6, 4, 19
    w = torch.randn(cin, cout, k)
    b = torch.randn(cout)
    x = torch.randn(2, cin, T)
    p = (k - s) // 2
    ref = F.conv_transpose1d(x, w, b, stride=s, padding=p)
    assert ref.shape[-1] == T * s
    M = (k + s - 1) // s
    subs = []
    for r in range(s):
        sub = torch.zeros(cout, cin, M)
        for jp in range(M):
            j = r + s * (M - 1 - jp)
            if j < k:
                sub[:, :, jp] = w[:, :, j].t()
        subs.append(sub)
    wc, bc = pack.ups_combined(subs, b, s, p)
    assert wc.shape == (cout * s, cin, M + 1)
    yc = F.conv1d(F.pad(x, (M - 1, 1)), wc, bc)              # frame i reads x[i - (M-1) .. i + 1]
    got = yc.view(2, cout, s, T).permute(0, 1, 3, 2).reshape(2, cout, T * s)
    assert torch.allclose(got, ref, atol=1e-5), (got - ref).abs().max()
    # with the noise conv of the stage riding as extra input channels gathered from the padded source
    sf, kch, PADF = 4, 8, 32
    src = torch.randn(2, 1, T * s * sf)
    wn, bn = torch.randn(cout, 1, 2 * sf), torch.randn(cout)
    ref2 = ref + F.conv1d(src, wn, bn, stride=sf, padding=sf // 2)
    wc2, bc2 = pack.ups_combined(subs, b, s, p, wn, bn, sf, kch)
    cin1 = (cin + kch - 1) // kch * kch
    nc = s * sf + sf
    assert wc2.shape == (cout * s, cin1 + nc, M + 1)
    srcp = F.pad(src[:, 0], (PADF, 128))
    x2 = torch.stack([srcp[:, PADF - sf // 2 + ci: PADF - sf // 2 + ci + sf * s * T: sf * s] for ci in range(nc)], 1)
    xin = torch.cat([x, torch.zeros(2, cin1 - cin, T), x2], 1)
    yc2 = F.conv1d(F.pad(xin, (M - 1, 1)), wc2, bc2)
    got2 = yc2.view(2, cout, s, T).permute(0, 1, 3, 2).reshape(2, cout, T * s)
    assert torch.allclose(got2, ref2, atol=1e-4), (got2 - ref2).abs().max()


def test_packed_model_tensor_inventory(hp, sd):
    cfg = pack.config_from_hp(hp)
    items = dict(pack.pack_svc_state_dict(sd, cfg))
    # gate interleave: packed channel 2c is tanh row c, 2c+1 is sigmoid row c
    H = cfg["hidden_channels"]
    w = pack.fold_weight_norm(sd, "flow.flows.0.enc.in_layers.0")
    wp = unpack_conv(items["flow.0.in.0.w"], 2 * H)
    assert torch.equal(wp[0::2], w[:H]) and torch.equal(wp[1::2], w[H:])
    # qkv concat
    q = unpack_conv(items["enc.0.qkv.w"], 3 * H)
    assert torch.equal(q[H:2 * H], sd["enc_p.enc.attn_layers.0.conv_k.weight"])
    # snake parameters
    ea = items["dec.res.0.act.0.ea"]
    assert torch.allclose(ea, torch.exp(sd["dec.resblocks.0.activations.0.act.alpha"]))
    blob, table = pack.build_blob(list(items.items()))
    assert all(off % 256 == 0 for _, off, _ in table)
    name, off, n = table[5]
    assert torch.equal(blob[off // 4: off // 4 + n], items[name].reshape(-1))


def test_last_stage_of_rate_4_has_no_combined_image(hp):
    """The combined up-sampler image (pack.ups_combined) carries the noise conv of a stage before the last; the last
    stage's noise conv has kernel 1, so a last stage of rate 4 and kernel 8 packs without `comb` tensors."""
    from whisper_vits_svc_b200 import hparams, synth
    hpx = hparams.override(hp, gen__upsample_rates=[4, 4], gen__upsample_kernel_sizes=[8, 8],
                           gen__upsample_initial_channel=64)
    names = [n for n, _ in pack.pack_svc_state_dict(synth.svc_state_dict(hpx, 7), pack.config_from_hp(hpx))]
    assert "dec.ups.0.comb.tc" in names and "dec.ups.0.comb.b" in names
    assert not any(n.startswith("dec.ups.1.comb") for n in names)


def test_whisper_conv2_weight_image_layout():
    """The stem's stride-2 conv runs as a GEMM over an im2col image (csrc/whisper_gemm.cu:
    im2col_s2_image): its weight must reach the kernel as W2[co][j*D + ci] = w[co][ci][j] in the bf16
    GEMM tile image [N/256][K/64][8][256][8]."""
    from whisper_vits_svc_b200 import synth, whisper_infer
    dims = dict(synth.WHISPER_LARGE_V2_DIMS, n_audio_state=256, n_audio_head=4, n_audio_layer=4)
    ck = synth.whisper_checkpoint(dims, seed=3)
    items, cfg = whisper_infer.pack_whisper(ck)
    named = dict(items)
    assert "conv2.w" not in named and "conv2.wimg" in named
    D = 256
    img = named["conv2.wimg"].view(torch.bfloat16).view(D // 256, 3 * D // 64, 8, 256, 8).float()
    w = ck["model_state_dict"]["encoder.conv2.weight"].float().bfloat16().float()  # [co, ci, j]
    g = torch.Generator().manual_seed(0)
    for _ in range(200):
        co = int(torch.randint(0, D, (1,), generator=g)); ci = int(torch.randint(0, D, (1,), generator=g))
        j = int(torch.randint(0, 3, (1,), generator=g))
        k = j * D + ci
        assert float(img[co // 256, k // 64, (k % 64) // 8, co % 256, k % 8]) == float(w[co, ci, j])


def test_stem_conv2_im2col_equivalence():
    """The identity the device path relies on (csrc/whisper_gemm.cu:im2col_s2_image + epilogue 3):
    Conv1d(D, D, k=3, stride=2, padding=1)(h)[b, :, t2] == A[b*n2 + t2, :] @ W2^T with
    A[m, j*D + ci] = h[b, ci, 2*t2 + j - 1] (zero outside) and W2[co, j*D + ci] = w[co, ci, j]."""
    g = torch.Generator().manual_seed(4)
    B, D, n = 2, 16, 37
    h = torch.randn(B, D, n, generator=g)
    w = torch.randn(D, D, 3, generator=g)
    bias = torch.randn(D, generator=g)
    ref = F.conv1d(h, w, bias, stride=2, padding=1)            # [B, D, n2]
    n2 = (n - 1) // 2 + 1
    assert ref.shape[-1] == n2
    A = torch.zeros(B * n2, 3 * D)
    for b in range(B):
        for t2 in range(n2):
            for j in range(3):
                t = 2 * t2 + j - 1
                if 0 <= t < n:
                    A[b * n2 + t2, j * D:(j + 1) * D] = h[b, :, t]
    W2 = w.permute(0, 2, 1).reshape(D, 3 * D)
    got = (A @ W2.t() + bias).view(B, n2, D).permute(0, 2, 1)
    assert torch.allclose(got, ref, atol=1e-4)


@pytest.mark.parametrize("C,k,dil", [(20, 3, 1), (20, 7, 3), (20, 11, 5), (10, 11, 5), (10, 3, 3), (40, 7, 5), (40, 11, 5)])
def test_conv_s2d_image_is_the_dilated_conv(C, k, dil):
    """csrc/amp_s2d.cu multiplies rows of r consecutive samples (all channels) by block-Toeplitz matrices:
    sum over row offsets m of X'[tau + m] @ W_m^T must equal F.conv1d(x, w, dilation, 'same') — checked
    through the packed bf16 hi/lo image (hi + lo reproduces fp32 weights to ~2^-16 relative)."""
    import torch.nn.functional as F
    from whisper_vits_svc_b200 import pack
    r = pack.s2d_factor(C)
    assert C * r == pack.S2D_WIDTH
    g = torch.Generator().manual_seed(C + k + dil)
    w = torch.randn(C, C, k, generator=g) / (C * k) ** 0.5
    x = torch.randn(2, C, r * 29, generator=g)
    ref = F.conv1d(x, w, dilation=dil, padding=dil * (k - 1) // 2)
    mlo, mhi = pack.s2d_taps(k, dil, r)
    P = dil * (k - 1) // 2
    assert mlo == -(-P // r) and mhi == (r - 1 + P) // r and mlo <= 8 and mhi <= 8   # fits the kernel's A panel
    img = pack.pack_conv_s2d(w, dil, r).view(torch.bfloat16).view(mlo + mhi + 1, 2, 20, 160, 8).float()
    W = (img[:, 0] + img[:, 1]).permute(0, 2, 1, 3).reshape(mlo + mhi + 1, 160, 160)      # [tap, n, k]
    assert (W - pack.conv_s2d_matrices(w, dil, r)).abs().max() <= 2e-5
    X = x.view(2, C, -1, r).permute(0, 2, 1, 3).reshape(2, -1, C * r)
    n = X.shape[1]
    Xp = F.pad(X, (0, 0, mlo, mhi))
    Y = sum(Xp[:, i:i + n] @ W[i].t() for i in range(mlo + mhi + 1))
    y = Y.view(2, n, C, r).permute(0, 2, 1, 3).reshape(2, C, -1)
    assert (y - ref).abs().max() <= 1e-4


@pytest.mark.parametrize("n", [7, 8, 301, 3000])
def test_conv2_image_scatter_rule(n):
    """csrc/whisper_gemm.cu epilogue 5: conv1's output frame t lands in conv2's im2col image at (t/2, tap 1) when even and
    at ((t+1)/2, tap 0), ((t-1)/2, tap 2) when odd — together exactly A2[t2][j] = h1[2 t2 + j - 1] (zero for t = -1 / n)."""
    n2 = (n - 1) // 2 + 1
    h1 = np.arange(1, n + 1, dtype=np.float64)
    want = np.zeros((n2, 3))
    for t2 in range(n2):
        for j in range(3):
            t = 2 * t2 + j - 1
            if 0 <= t < n:
                want[t2, j] = h1[t]
    got = np.zeros((n2, 3))
    for t in range(n):
        if t & 1:
            if (t + 1) // 2 < n2:
                got[(t + 1) // 2, 0] = h1[t]
            got[(t - 1) // 2, 2] = h1[t]
        else:
            got[t // 2, 1] = h1[t]
    assert np.array_equal(got, want)


@pytest.mark.parametrize("n,taps", [(9, 3), (10, 3), (64015, 3), (8, 2), (9, 2), (2000, 2)])
def test_valid_stride2_image_scatter_rule(n, taps):
    """csrc/whisper_gemm.cu epilogue 6 / csrc/hubert_api.cu:hubert_conv0_pack_kernel (HuBERT stem, valid stride-2 convs):
    frame t = 2 t2 + j feeds (t/2, 0) and (t/2 - 1, 2) when even, ((t-1)/2, 1) when odd; every entry of the next conv's
    image A[t2][j] = h[2 t2 + j], t2 < (n - taps) // 2 + 1, is written exactly once."""
    tn = (n - taps) // 2 + 1
    h = np.arange(1, n + 1, dtype=np.float64)
    want = np.stack([h[j:j + 2 * tn:2][:tn] for j in range(taps)], 1)
    got = np.zeros((tn, taps))
    hits = np.zeros((tn, taps), dtype=np.int64)

    def put(t2, j, v):
        if 0 <= t2 < tn:
            got[t2, j] = v
            hits[t2, j] += 1

    for t in range(n):
        if t & 1:
            put((t - 1) >> 1, 1, h[t])
        else:
            put(t >> 1, 0, h[t])
            if taps == 3:
                put((t >> 1) - 1, 2, h[t])
    assert np.array_equal(got, want) and (hits == 1).all()
