"""Host-side weight packer: reference checkpoint -> one fp32 device blob + name table.

Runs once at load time (the reference re-materialises weight-norm on every forward because
svc_inference.py:169 calls nn.Module.eval(), not Generator.eval(inference=True); folding once is
what vits_decoder/generator.py:154-158 does for inference).  Everything arithmetic here is the
reference's own parameter algebra (torch._weight_norm, exp of the Snake log-scale parameters);
the data path never touches the host again.

Packed tensors (all fp32, each 256-byte aligned in the blob):

  <conv>.w   [Cin][K][CoutPad8]  output channel innermost, padded to a multiple of 8
  <conv>.b   [Cout]
  flow.<f>.in.<l>.*   output channels interleaved (tanh_c, sigmoid_c) so the WaveNet gate
                      (vits/commons.py:126-133) is a conv epilogue
  enc.<i>.qkv.*       conv_q | conv_k | conv_v concatenated along Cout (attentions.py:216-218)
  dec.ups.<i>.ph<r>.w ConvTranspose1d split into `rate` polyphase sub-filters:
                      w_r[co][ci][j'] = w[ci][co][r + rate*(M-1-j')], M = ceil(k/rate)
  dec.res.<n>.c{1,2}.<d>.tc   the same AMP conv as bf16 hi/lo tensor-core tiles (pack_conv_tc)
  dec.res.<n>.act.<a>.ea / .ib   exp(alpha), 1/(exp(beta)+1e-9)   (alias/act.py:85-91)
  dec.res.<n>.act.<a>.fu / .fd   the 12 up / down taps stored in the checkpoint
"""
from __future__ import annotations

import ctypes
import math
from typing import Dict, List, Tuple

import numpy as np
import torch

ALIGN = 256


def fold_weight_norm(sd, prefix: str) -> torch.Tensor:
    if prefix + ".weight" in sd:
        return sd[prefix + ".weight"].float()
    return torch._weight_norm(sd[prefix + ".weight_v"].float(), sd[prefix + ".weight_g"].float(), 0)


def pack_conv(w: torch.Tensor) -> torch.Tensor:
    """[Cout, Cin, K] -> [Cin, K, CoutPad8] (zero padded)."""
    cout, cin, k = w.shape
    cp = (cout + 7) // 8 * 8
    out = torch.zeros(cin, k, cp, dtype=torch.float32)
    out[:, :, :cout] = w.permute(1, 2, 0)
    return out.contiguous()


def pack_conv_tc(w: torch.Tensor) -> torch.Tensor:
    """[C, C, K] fp32 -> the tensor-core image bf16 [K][2 (hi, lo)][Cp/8][Cp][8] (Cp = C rounded up
    to 16): per tap and split part, the B operand W_tap[n = co][k = ci] in the K-major panel layout
    of csrc/tc.cuh, so one tap is one contiguous bulk copy.  hi = bf16(w), lo = bf16(w - hi).
    Returned as a float32 *view* of the bf16 bytes (the blob is fp32-typed; bits are preserved)."""
    cout, cin, k = w.shape
    assert cout == cin
    cp = (cout + 15) // 16 * 16
    wp = torch.zeros(k, cp, cp, dtype=torch.float32)
    wp[:, :cout, :cin] = w.permute(2, 0, 1)
    hi = wp.bfloat16()
    lo = (wp - hi.float()).bfloat16()
    st = torch.stack([hi, lo], 1)                                  # [K, 2, n, k]
    img = st.view(k, 2, cp, cp // 8, 8).permute(0, 1, 3, 2, 4).contiguous()  # [K, 2, kc, n, 8]
    return img.view(torch.float32).reshape(-1)


S2D_WIDTH = 160   # K' = N' = C * r of the space-to-depth AMP links (csrc/amp_s2d.cu)


def s2d_factor(c: int) -> int:
    """Time samples folded into the channel dimension so that C * r = 160 (0 = stage not eligible)."""
    return S2D_WIDTH // c if c and S2D_WIDTH % c == 0 and S2D_WIDTH // c in (4, 8, 16) else 0


def s2d_taps(k: int, dil: int, r: int):
    """Row offsets m = -mlo .. mhi of the block-Toeplitz form of a 'same' Conv1d(k, dilation) over rows of r
    samples: output sample r*tau + po needs input samples r*tau + po + j*dil - P, P = dil*(k-1)/2."""
    P = dil * (k - 1) // 2
    mlo = -((-P) // r)             # ceil(P / r)
    mhi = (r - 1 + P) // r
    return mlo, mhi


def conv_s2d_matrices(w: torch.Tensor, dil: int, r: int) -> torch.Tensor:
    """[C, C, k] -> [ntaps, N' = C*r, K' = C*r] fp32 block-Toeplitz matrices W_m with
    y'[tau][(co, po)] = sum_m sum_(ci, pi) W_m[(co, po)][(ci, pi)] * x'[tau + m][(ci, pi)],
    x'[tau][(c, p)] = x[c][r*tau + p] (index = c*r + p): the dilated Conv1d as `ntaps` dense 160 x 160
    products over rows of r consecutive samples (csrc/amp_s2d.cu; vits_decoder/bigv.py:22-39)."""
    cout, cin, k = w.shape
    P = dil * (k - 1) // 2
    mlo, mhi = s2d_taps(k, dil, r)
    W = torch.zeros(mlo + mhi + 1, cout, r, cin, r, dtype=torch.float32)
    for j in range(k):
        off = j * dil - P                      # input sample offset of tap j
        for po in range(r):
            m, pi = divmod(po + off, r)        # r*m + pi = po + off
            W[m + mlo, :, po, :, pi] += w[:, :, j]
    return W.reshape(mlo + mhi + 1, cout * r, cin * r)


def pack_conv_s2d(w: torch.Tensor, dil: int, r: int) -> torch.Tensor:
    """The matrices of conv_s2d_matrices as bf16 hi/lo tensor-core tiles [ntaps][2 (hi, lo)][K'/8][N'][8]
    (K-major panel layout of csrc/tc.cuh: one (tap, part) = one contiguous 51,200-byte bulk copy),
    returned as a float32 view of the bytes."""
    W = conv_s2d_matrices(w, dil, r)                          # [T, n, k]
    T, n, k = W.shape
    assert n == S2D_WIDTH and k == S2D_WIDTH, (n, k)
    hi = W.bfloat16()
    lo = (W - hi.float()).bfloat16()
    st = torch.stack([hi, lo], 1)                              # [T, 2, n, k]
    img = st.view(T, 2, n, k // 8, 8).permute(0, 1, 3, 2, 4).contiguous()   # [T, 2, kc, n, 8]
    return img.view(torch.float32).reshape(-1)


S2D_SLOT_GROUPS = (0, 1, 3, 2)   # phase group held by each 40-column slot of csrc/amp_s2d.cu


def s2d_column_order(r: int) -> torch.Tensor:
    """Output column n of the kernel's slot order -> column c*r + p of conv_s2d_matrices.  Slot s = n // 40 holds
    the g = r/4 phases p = g*q + j of phase group q = S2D_SLOT_GROUPS[s], channel by channel: n = 40 s + g c + j.
    Every edge tap then reaches only the first 40 or 80 columns of a half (s2d_tap_cols)."""
    g = r // 4
    n = torch.arange(S2D_WIDTH)
    q = torch.tensor(S2D_SLOT_GROUPS)[n // 40]
    c, j = (n % 40) // g, (n % 40) % g
    return c * r + g * q + j


def s2d_tap_cols(k: int, dil: int, r: int):
    """Per Toeplitz tap m = -mlo .. mhi, the output columns [n0, n1) of the slot order its matrix can reach.
    Tap m reaches the phases max(0, r m - P) .. min(r - 1, r m + r - 1 + P); an edge tap that reaches only
    phase groups {0}, {0, 1}, {3} or {3, 2} keeps [0, 40), [0, 80), [80, 120) or [80, 160), every other tap
    all 160 columns (csrc/amp_s2d.cu:s2d_tap_plan)."""
    P = dil * (k - 1) // 2
    mlo, mhi = s2d_taps(k, dil, r)
    g = r // 4
    cols = []
    for m in range(-mlo, mhi + 1):
        q0, q1 = max(0, r * m - P) // g, min(r - 1, r * m + r - 1 + P) // g
        if q0 == 0 and q1 <= 1:
            cols.append((0, 40 * (q1 + 1)))
        elif q1 == 3 and q0 >= 2:
            cols.append((80, 80 + 40 * (4 - q0)))
        else:
            cols.append((0, S2D_WIDTH))
    return cols


def pack_conv_s2d_slots(w: torch.Tensor, dil: int, r: int) -> torch.Tensor:
    """pack_conv_s2d's image with the output (N') index in the slot order of s2d_column_order: the layout
    csrc/amp_s2d.cu reads, so that an edge tap's reached columns are one contiguous run per octet."""
    T = sum(s2d_taps(w.shape[-1], dil, r)) + 1
    img = pack_conv_s2d(w, dil, r).view(torch.bfloat16).view(T, 2, S2D_WIDTH // 8, S2D_WIDTH, 8)
    return img[:, :, :, s2d_column_order(r)].contiguous().view(torch.float32).reshape(-1)


S2D_FOLD_MAX = 5   # largest fold of a folded S2D image (csrc/amp_s2d.cu)


def s2d_tile(r: int, fin: int, fout: int, mlo: int, mhi: int):
    """(halo, stride, a_off) of a link's tiles: halo rows on each side, useful rows per tile, A-panel row of the
    tile's first row, for an input image of fold fin and an output image of fold fout — must match
    csrc/amp_s2d.cu:s2d_tile.  A folded input has tiles of whole blocks and a halo of one block; a folded output has
    whole output blocks of useful rows."""
    if fin > 1:
        rows = min(128, 144 - (mlo + mhi) * fin) // fin * fin
        return fin, rows - 2 * fin, mlo * fin
    halo = 1 if r >= 8 else 2
    return halo, (128 - 2 * halo) // fout * fout, 8


def _col_units(k: int, dil: int, r: int) -> int:
    return sum((n1 - n0) // 40 for n0, n1 in s2d_tap_cols(k, dil, r))


def s2d_fold(k: int, dil: int, r: int) -> int:
    """The fold a c1 link Conv1d(k, dil) reads its input in: dil when the link has more than 3 full taps of column
    work and the undilated conv's column work per useful tile row is lower, else 1 — must match
    csrc/amp_s2d.cu:s2d_tap_plan.  Folded, row
    b*dil + q of the image holds the samples b*r*dil + q + j*dil and tap m shifts by m*dil rows."""
    if dil < 2 or dil > S2D_FOLD_MAX:
        return 1
    mlo, mhi = s2d_taps(k, dil, r)
    ulo, uhi = s2d_taps(k, 1, r)
    _, s1, _ = s2d_tile(r, 1, 1, mlo, mhi)
    hd, sd, ad = s2d_tile(r, dil, 1, ulo, uhi)
    if sd <= 0 or hd + ad > 16:
        return 1
    cu = _col_units(k, dil, r)      # links of up to 3 full taps are bound by their Snake epilogue: left unfolded
    return dil if cu > 12 and _col_units(k, 1, r) * s1 < cu * sd else 1


def pack_conv_s2d_link(w: torch.Tensor, dil: int, r: int) -> torch.Tensor:
    """The weights of a link Conv1d(w, dil) as csrc/amp_s2d.cu runs it: pack_conv_s2d_slots of the conv, or of
    the undilated conv when the link reads a folded input (s2d_fold)."""
    return pack_conv_s2d_slots(w, 1 if s2d_fold(w.shape[-1], dil, r) > 1 else dil, r)


def tc_tiling(cout: int, cin: int):
    """(kch, cin_pad, bn, ntiles) — must match csrc/api.cu:tc_tiling."""
    kch = 32
    cin_pad = (cin + kch - 1) // kch * kch
    cp16 = (cout + 15) // 16 * 16
    ntiles = (cp16 + 255) // 256
    bn = ((cp16 + ntiles - 1) // ntiles + 15) // 16 * 16
    return kch, cin_pad, bn, ntiles


def pack_conv_tc_general(w: torch.Tensor) -> torch.Tensor:
    """[Cout, Cin, K] fp32 -> bf16 tiles [K][ncc][2 (hi,lo)][ntiles][kch/8][bn][8] for
    csrc/conv_tc.cu: per (tap, input-channel chunk, split part, output tile) the B operand
    W[n = co][k = ci] in the K-major panel layout, one contiguous bulk copy each."""
    cout, cin, k = w.shape
    kch, cin_pad, bn, ntiles = tc_tiling(cout, cin)
    ncc = cin_pad // kch
    wp = torch.zeros(k, ntiles * bn, cin_pad, dtype=torch.float32)
    wp[:, :cout, :cin] = w.permute(2, 0, 1)
    hi = wp.bfloat16()
    lo = (wp - hi.float()).bfloat16()
    st = torch.stack([hi, lo], 1)                               # [K, 2, N, Kin]
    st = st.view(k, 2, ntiles, bn, ncc, kch // 8, 8)            # K, part, nt, n, cc, kc, e
    img = st.permute(0, 4, 1, 2, 5, 3, 6).contiguous()          # K, cc, part, nt, kc, n, e
    return img.view(torch.float32).reshape(-1)


def ups_combined(subs, bias: torch.Tensor, rate: int, pad: int, wn: torch.Tensor = None, bn: torch.Tensor = None,
                 sf: int = 0, kch: int = 32):
    """The `rate` polyphase sub-filters of a ConvTranspose1d (M taps each, [Cout, Cin, M]) as ONE Conv1d with
    rate * Cout output channels and M + 1 taps (padding M - 1): output channel co * rate + s at frame i is the
    transposed conv's output sample rate * i + s of channel co.  Phase r starts at frame q0_r = ceil((pad - r) /
    rate) (0 when r >= pad) and lands on slot s_r = rate * q0_r + r - pad; a phase with q0 = 1 reads x one frame
    later, i.e. its taps sit one position further right in the common window.  The tensor-core conv then reads
    the stage input once instead of `rate` times and its epilogue stores `rate` consecutive samples per thread
    (csrc/conv_tc.cu, ConvTcParams::ilv) — no phase scratch, no interleave pass.

    With wn ([Cout, 1, 2 sf], bn): noise_convs[i] (Conv1d(1, Cout, 2 sf, stride sf, padding sf / 2) over the
    harmonic source, generator.py:185-186) rides in the same GEMM as extra input channels behind the main ones
    (padded to a multiple of kch): at frame i channel ci' is source sample sf * rate * i - sf / 2 + ci', ci' <
    rate * sf + sf, and output slot s takes tap j of the noise filter from channel s * sf + j at the window tap
    that reads frame i.  (ConvTcParams::x2: the kernel gathers those channels from the padded source.)"""
    cout, cin, M = subs[0].shape
    cin1 = (cin + kch - 1) // kch * kch if wn is not None else cin
    nc = rate * sf + wn.shape[-1] - sf if wn is not None else 0
    w = torch.zeros(cout * rate, cin1 + nc, M + 1)
    b = torch.zeros(cout * rate)
    for r in range(rate):
        q0 = (pad - r + rate - 1) // rate if pad > r else 0
        assert q0 in (0, 1)
        s = rate * q0 + r - pad
        assert 0 <= s < rate
        w[s::rate, :cin, q0:q0 + M] = subs[r]
        b[s::rate] = bias
    if wn is not None:
        assert wn.shape[-1] == 2 * sf and wn.shape[1] == 1
        for s in range(rate):
            w[s::rate, cin1 + s * sf:cin1 + s * sf + 2 * sf, M - 1] = wn[:, 0, :]
            b[s::rate] += bn
    return w, b


def config_from_hp(hp, precision: int = 0) -> dict:
    rates = [int(x) for x in hp.gen.upsample_rates]
    ks = [int(x) for x in hp.gen.upsample_kernel_sizes]
    rk = [int(x) for x in hp.gen.resblock_kernel_sizes]
    rd = [[int(y) for y in x] for x in hp.gen.resblock_dilation_sizes]
    return dict(
        ppg_dim=int(hp.vits.ppg_dim), vec_dim=int(hp.vits.vec_dim), spk_dim=int(hp.vits.spk_dim),
        inter_channels=int(hp.vits.inter_channels), hidden_channels=int(hp.vits.hidden_channels),
        filter_channels=int(hp.vits.filter_channels),
        # constants hard-coded by the reference at vits/models.py:220-238
        enc_layers=6, enc_heads=2, enc_kernel=3, enc_window=4, n_flows=4, wn_layers=4, wn_kernel=5,
        gen_input=int(hp.gen.upsample_input), gen_initial_channel=int(hp.gen.upsample_initial_channel),
        n_ups=len(rates), up_rates=rates, up_kernels=ks, n_res=len(rk), res_kernels=rk,
        res_dilations=rd, sampling_rate=int(hp.data.sampling_rate), n_harmonics=11,
        precision=int(precision))


def pack_svc_state_dict(sd: Dict[str, torch.Tensor], cfg: dict) -> List[Tuple[str, torch.Tensor]]:
    """Return [(packed_name, fp32 tensor)] in blob order."""
    out: List[Tuple[str, torch.Tensor]] = []

    def put(name, t):
        out.append((name, t.detach().float().contiguous()))

    def conv(name, w, b=None, tc=False):
        put(name + ".w", pack_conv(w))
        if b is not None:
            put(name + ".b", b)
        if tc:
            put(name + ".tc", pack_conv_tc_general(w))

    H = cfg["hidden_channels"]
    conv("enc_p.pre", sd["enc_p.pre.weight"], sd["enc_p.pre.bias"], tc=True)
    conv("enc_p.hub", sd["enc_p.hub.weight"], sd["enc_p.hub.bias"], tc=True)
    put("enc_p.pit", sd["enc_p.pit.weight"])
    for i in range(cfg["enc_layers"]):
        a = f"enc_p.enc.attn_layers.{i}"
        wq = torch.cat([sd[f"{a}.conv_{n}.weight"] for n in "qkv"], 0)
        bq = torch.cat([sd[f"{a}.conv_{n}.bias"] for n in "qkv"], 0)
        conv(f"enc.{i}.qkv", wq, bq, tc=True)
        conv(f"enc.{i}.o", sd[f"{a}.conv_o.weight"], sd[f"{a}.conv_o.bias"], tc=True)
        put(f"enc.{i}.ek", sd[f"{a}.emb_rel_k"][0])
        put(f"enc.{i}.ev", sd[f"{a}.emb_rel_v"][0])
        put(f"enc.{i}.ln1.g", sd[f"enc_p.enc.norm_layers_1.{i}.gamma"])
        put(f"enc.{i}.ln1.b", sd[f"enc_p.enc.norm_layers_1.{i}.beta"])
        f = f"enc_p.enc.ffn_layers.{i}"
        conv(f"enc.{i}.ffn1", sd[f"{f}.conv_1.weight"], sd[f"{f}.conv_1.bias"], tc=True)
        conv(f"enc.{i}.ffn2", sd[f"{f}.conv_2.weight"], sd[f"{f}.conv_2.bias"], tc=True)
        put(f"enc.{i}.ln2.g", sd[f"enc_p.enc.norm_layers_2.{i}.gamma"])
        put(f"enc.{i}.ln2.b", sd[f"enc_p.enc.norm_layers_2.{i}.beta"])
    conv("enc_p.proj", sd["enc_p.proj.weight"], sd["enc_p.proj.bias"], tc=True)

    for fidx in range(cfg["n_flows"]):
        p = f"flow.flows.{2 * fidx}"
        q = f"flow.{fidx}"
        conv(q + ".pre", sd[p + ".pre.weight"], sd[p + ".pre.bias"], tc=True)
        for l in range(cfg["wn_layers"]):
            w = fold_weight_norm(sd, f"{p}.enc.in_layers.{l}")
            b = sd[f"{p}.enc.in_layers.{l}.bias"]
            idx = torch.stack([torch.arange(H), torch.arange(H) + H], 1).reshape(-1)  # (t0,s0,t1,s1,..)
            conv(f"{q}.in.{l}", w[idx], b[idx], tc=True)
            conv(f"{q}.rs.{l}", fold_weight_norm(sd, f"{p}.enc.res_skip_layers.{l}"),
                 sd[f"{p}.enc.res_skip_layers.{l}.bias"], tc=True)
        conv(q + ".post", sd[p + ".post.weight"], sd[p + ".post.bias"], tc=True)
        put(q + ".snac.w", sd[p + ".snac.weight"][:, :, 0])
        put(q + ".snac.b", sd[p + ".snac.bias"])

    put("dec.adapter.scale.w", sd["dec.adapter.W_scale.weight"])
    put("dec.adapter.scale.b", sd["dec.adapter.W_scale.bias"])
    put("dec.adapter.bias.w", sd["dec.adapter.W_bias.weight"])
    put("dec.adapter.bias.b", sd["dec.adapter.W_bias.bias"])
    conv("dec.conv_pre", sd["dec.conv_pre.weight"], sd["dec.conv_pre.bias"], tc=True)
    put("dec.merge_w", sd["dec.m_source.merge_w"].reshape(-1))
    put("dec.merge_b", sd["dec.m_source.merge_b"].reshape(-1))
    for i, (rate, k) in enumerate(zip(cfg["up_rates"], cfg["up_kernels"])):
        w = fold_weight_norm(sd, f"dec.ups.{i}")  # [Cin, Cout, k]
        M = (k + rate - 1) // rate
        subs = []
        for r in range(rate):
            sub = torch.zeros(w.shape[1], w.shape[0], M)
            for jp in range(M):
                j = r + rate * (M - 1 - jp)
                if j < k:
                    sub[:, :, jp] = w[:, :, j].t()
            subs.append(sub)
            put(f"dec.ups.{i}.ph{r}.w", pack_conv(sub))
            put(f"dec.ups.{i}.ph{r}.tc", pack_conv_tc_general(sub))
        put(f"dec.ups.{i}.b", sd[f"dec.ups.{i}.bias"])
        wn = sd[f"dec.noise_convs.{i}.weight"]
        if rate == 4 and M == 2 and i + 1 < cfg["n_ups"]:   # must match csrc/api.cu:resolve
            sf_c = int(np.prod(cfg["up_rates"][i + 1:]))
            assert wn.shape[-1] == 2 * sf_c, "combined up-sampling stage: noise filter must be 2 * prod(later rates) long"
            wc, bc = ups_combined(subs, sd[f"dec.ups.{i}.bias"].float(), rate, (k - rate) // 2, wn.float(),
                                  sd[f"dec.noise_convs.{i}.bias"].float(), sf_c)
            put(f"dec.ups.{i}.comb.tc", pack_conv_tc_general(wc))
            put(f"dec.ups.{i}.comb.b", bc)
        conv(f"dec.noise.{i}", wn, sd[f"dec.noise_convs.{i}.bias"])
        if wn.shape[-1] > 8:
            # long noise filter = Conv1d(1->C, K=2*sf, stride sf): on the source reshaped to sf "channels"
            # per frame (space-to-depth) it is a 2-tap convolution, which the tensor-core conv handles:
            # w2[co][ci][j] = w[co][0][sf*j + ci]
            sf_ = wn.shape[-1] // 2
            w2 = wn[:, 0, :].reshape(wn.shape[0], 2, sf_).permute(0, 2, 1).contiguous()
            put(f"dec.noise.{i}.tc", pack_conv_tc_general(w2))
    n_blocks = cfg["n_ups"] * cfg["n_res"]
    for n in range(n_blocks):
        p = f"dec.resblocks.{n}"
        stage, j = divmod(n, cfg["n_res"])
        ch = cfg["gen_initial_channel"] >> (stage + 1)
        r = s2d_factor(ch)
        for d in range(3):
            w1 = fold_weight_norm(sd, f"{p}.convs1.{d}")
            w2 = fold_weight_norm(sd, f"{p}.convs2.{d}")
            conv(f"dec.res.{n}.c1.{d}", w1, sd[f"{p}.convs1.{d}.bias"])
            conv(f"dec.res.{n}.c2.{d}", w2, sd[f"{p}.convs2.{d}.bias"])
            put(f"dec.res.{n}.c1.{d}.tc", pack_conv_tc(w1))
            put(f"dec.res.{n}.c2.{d}.tc", pack_conv_tc(w2))
            if r:   # narrow stages: block-Toeplitz matrices for csrc/amp_s2d.cu
                put(f"dec.res.{n}.c1.{d}.s2d", pack_conv_s2d_link(w1, cfg["res_dilations"][j][d], r))
                put(f"dec.res.{n}.c2.{d}.s2d", pack_conv_s2d_slots(w2, 1, r))
        for a in range(6):
            _snake(put, f"dec.res.{n}.act.{a}", sd, f"{p}.activations.{a}")
    _snake(put, "dec.post.act", sd, "dec.activation_post")
    conv("dec.conv_post", sd["dec.conv_post.weight"])
    return out


def _snake(put, name, sd, p):
    put(name + ".ea", torch.exp(sd[p + ".act.alpha"].float()))
    put(name + ".ib", 1.0 / (torch.exp(sd[p + ".act.beta"].float()) + 1e-9))
    put(name + ".fu", sd[p + ".upsample.filter"].reshape(-1))
    put(name + ".fd", sd[p + ".downsample.lowpass.filter"].reshape(-1))


def build_blob(items: List[Tuple[str, torch.Tensor]]):
    """-> (flat fp32 CPU tensor, [(name, offset_bytes, numel)])."""
    table = []
    off = 0
    for name, t in items:
        off = (off + ALIGN - 1) // ALIGN * ALIGN
        table.append((name, off, t.numel()))
        off += t.numel() * 4
    total = (off + ALIGN - 1) // ALIGN * ALIGN
    blob = torch.zeros(total // 4, dtype=torch.float32)
    for (name, o, n), (_, t) in zip(table, items):
        blob[o // 4:o // 4 + n] = t.reshape(-1)
    return blob, table
