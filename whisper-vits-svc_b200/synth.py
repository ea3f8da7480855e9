"""Seeded synthetic checkpoints in the reference's formats.

No pretrained weights ship with the reference (vits_pretrain/, whisper_pretrain/ hold only
READMEs), so benchmarks and parity tests use seeded random weights.  The default
initialisation of the reference zeroes several tensors (flow `post`, SpeakerAdapter weights,
Snake alpha/beta), which would hide bugs, so *every* tensor here is drawn at random with a
scale that keeps activations O(1).

`svc_state_dict(hp, seed)` returns the 903-entry `model_g` dict of svc_export.py:40-45 /
svc_inference.py:61-74 (weight_g/weight_v pairs kept, alias `filter` buffers,
`dec.m_source.merge_w/b`).  `whisper_checkpoint(...)` returns
{"dims":…, "model_state_dict":…} as read by whisper/inference.py:12-20.
"""
from __future__ import annotations

import math
from typing import Dict

import numpy as np
import torch


def kaiser_sinc_filter(cutoff: float, half_width: float, kernel_size: int) -> torch.Tensor:
    """The low-pass prototype the reference stores as a buffer
    (vits_decoder/alias/filter.py:28-57): Kaiser-windowed sinc, normalised to unit sum."""
    half = kernel_size // 2
    delta_f = 4 * half_width
    att = 2.285 * (half - 1) * math.pi * delta_f + 7.95
    if att > 50.0:
        beta = 0.1102 * (att - 8.7)
    elif att >= 21.0:
        beta = 0.5842 * (att - 21) ** 0.4 + 0.07886 * (att - 21.0)
    else:
        beta = 0.0
    win = torch.kaiser_window(kernel_size, beta=beta, periodic=False)
    if kernel_size % 2 == 0:
        t = torch.arange(-half, half) + 0.5
    else:
        t = torch.arange(kernel_size) - half
    f = 2 * cutoff * win * torch.sinc(2 * cutoff * t)
    f = f / f.sum()
    return f.view(1, 1, kernel_size)


MERGE_W = [0.2942, -0.2243, 0.0033, -0.0056, -0.0020, -0.0046,
           0.0221, -0.0083, -0.0241, -0.0036, -0.0581]  # vits_decoder/nsf.py:378-380
MERGE_B = [0.0008]


class _Gen:
    def __init__(self, seed):
        self.g = torch.Generator().manual_seed(seed)

    def n(self, *shape, std=1.0):
        return torch.randn(*shape, generator=self.g) * std

    def conv(self, sd, name, cout, cin, k, gain=1.0, bias=True, wn=False, transposed=False):
        fan = cin * k
        shape = (cin, cout, k) if transposed else (cout, cin, k)
        w = self.n(*shape, std=gain / math.sqrt(fan))
        if wn:
            # weight_norm dim=0: one g per slice of dim 0 (per *input* channel for ConvTranspose1d)
            v = self.n(*shape, std=0.3)
            norm = v.flatten(1).norm(dim=1).view(-1, 1, 1)
            target = w.flatten(1).norm(dim=1).view(-1, 1, 1)
            sd[name + ".weight_g"] = target * (1.0 + 0.1 * self.n(shape[0], 1, 1)).abs()
            sd[name + ".weight_v"] = v
            del norm
        else:
            sd[name + ".weight"] = w
        if bias:
            sd[name + ".bias"] = self.n(cout, std=0.05)


def svc_state_dict(hp, seed: int = 1234) -> Dict[str, torch.Tensor]:
    r = _Gen(seed)
    sd: Dict[str, torch.Tensor] = {}
    H = hp.vits.hidden_channels
    C = hp.vits.inter_channels
    Fc = hp.vits.filter_channels
    # ---- enc_p (vits/models.py:14-37)
    r.conv(sd, "enc_p.pre", H, hp.vits.ppg_dim, 5)
    r.conv(sd, "enc_p.hub", H, hp.vits.vec_dim, 5)
    sd["enc_p.pit.weight"] = r.n(256, H, std=0.5)
    for i in range(6):
        a = f"enc_p.enc.attn_layers.{i}"
        sd[a + ".emb_rel_k"] = r.n(1, 9, H // 2, std=(H // 2) ** -0.5)
        sd[a + ".emb_rel_v"] = r.n(1, 9, H // 2, std=(H // 2) ** -0.5)
        for nm in ("conv_q", "conv_k", "conv_v", "conv_o"):
            r.conv(sd, f"{a}.{nm}", H, H, 1, gain=1.2)
        sd[f"enc_p.enc.norm_layers_1.{i}.gamma"] = 1.0 + r.n(H, std=0.1)
        sd[f"enc_p.enc.norm_layers_1.{i}.beta"] = r.n(H, std=0.1)
        r.conv(sd, f"enc_p.enc.ffn_layers.{i}.conv_1", Fc, H, 3, gain=1.2)
        r.conv(sd, f"enc_p.enc.ffn_layers.{i}.conv_2", H, Fc, 3, gain=1.2)
        sd[f"enc_p.enc.norm_layers_2.{i}.gamma"] = 1.0 + r.n(H, std=0.1)
        sd[f"enc_p.enc.norm_layers_2.{i}.beta"] = r.n(H, std=0.1)
    r.conv(sd, "enc_p.proj", 2 * C, H, 1, gain=0.5)
    # ---- flow (vits/models.py:55-80, vits/modules.py:250-286)
    for f in range(4):
        p = f"flow.flows.{2 * f}"
        r.conv(sd, p + ".pre", H, C // 2, 1)
        for i in range(4):
            r.conv(sd, f"{p}.enc.in_layers.{i}", 2 * H, H, 5, wn=True)
            r.conv(sd, f"{p}.enc.res_skip_layers.{i}", 2 * H if i < 3 else H, H, 1, wn=True, gain=0.7)
        r.conv(sd, p + ".post", C // 2, H, 1, gain=0.5)
        r.conv(sd, p + ".snac", C, hp.vits.spk_dim, 1, gain=2.0)
    # ---- dec (vits_decoder/generator.py:52-110)
    U = hp.gen.upsample_input
    ch0 = hp.gen.upsample_initial_channel
    sd["dec.adapter.W_scale.weight"] = r.n(U, hp.vits.spk_dim, std=0.5)
    sd["dec.adapter.W_scale.bias"] = 1.0 + r.n(U, std=0.1)
    sd["dec.adapter.W_bias.weight"] = r.n(U, hp.vits.spk_dim, std=0.5)
    sd["dec.adapter.W_bias.bias"] = r.n(U, std=0.1)
    r.conv(sd, "dec.conv_pre", ch0, U, 7)
    sd["dec.m_source.merge_w"] = torch.tensor([MERGE_W], dtype=torch.float32)
    sd["dec.m_source.merge_b"] = torch.tensor(MERGE_B, dtype=torch.float32)
    rates = list(hp.gen.upsample_rates)
    ksz = list(hp.gen.upsample_kernel_sizes)
    filt = kaiser_sinc_filter(0.25, 0.3, 12)
    ch = ch0
    for i, (u, k) in enumerate(zip(rates, ksz)):
        cin, cout = ch0 // (2 ** i), ch0 // (2 ** (i + 1))
        # effective fan-in of a transposed conv is cin*k/u taps per output sample
        r.conv(sd, f"dec.ups.{i}", cout, cin, k, wn=True, transposed=True, gain=math.sqrt(u))
        if i + 1 < len(rates):
            s = int(np.prod(rates[i + 1:]))
            r.conv(sd, f"dec.noise_convs.{i}", cout, 1, 2 * s, gain=2.0)
        else:
            r.conv(sd, f"dec.noise_convs.{i}", cout, 1, 1, gain=1.0)
        ch = cout
    rk = list(hp.gen.resblock_kernel_sizes)
    for i in range(len(rates)):
        ch = ch0 // (2 ** (i + 1))
        for j, k in enumerate(rk):
            p = f"dec.resblocks.{i * len(rk) + j}"
            for d in range(3):
                r.conv(sd, f"{p}.convs1.{d}", ch, ch, k, wn=True, gain=0.8)
                r.conv(sd, f"{p}.convs2.{d}", ch, ch, k, wn=True, gain=0.4)
            for a in range(6):
                sd[f"{p}.activations.{a}.act.alpha"] = r.n(ch, std=0.4)
                sd[f"{p}.activations.{a}.act.beta"] = r.n(ch, std=0.4)
                sd[f"{p}.activations.{a}.upsample.filter"] = filt.clone()
                sd[f"{p}.activations.{a}.downsample.lowpass.filter"] = filt.clone()
    sd["dec.activation_post.act.alpha"] = r.n(ch, std=0.4)
    sd["dec.activation_post.act.beta"] = r.n(ch, std=0.4)
    sd["dec.activation_post.upsample.filter"] = filt.clone()
    sd["dec.activation_post.downsample.lowpass.filter"] = filt.clone()
    r.conv(sd, "dec.conv_post", 1, ch, 7, bias=False, gain=0.12)
    return {k: v.float().contiguous() for k, v in sd.items()}


WHISPER_LARGE_V2_DIMS = dict(n_mels=80, n_audio_ctx=1500, n_audio_state=1280, n_audio_head=20,
                             n_audio_layer=32, n_vocab=51865, n_text_ctx=448, n_text_state=1280,
                             n_text_head=20, n_text_layer=32)


def whisper_checkpoint(dims: dict | None = None, seed: int = 1234, kept_layers: int | None = None):
    """Encoder-only synthetic Whisper checkpoint.  whisper/inference.py:16-20 deletes the decoder
    and the last quarter of the encoder blocks and loads with strict=False, so only encoder keys
    of the kept blocks matter; `kept_layers` defaults to n_audio_layer - n_audio_layer//4."""
    dims = dict(dims or WHISPER_LARGE_V2_DIMS)
    n_layer = dims["n_audio_layer"]
    kept = kept_layers if kept_layers is not None else n_layer - n_layer // 4
    D = dims["n_audio_state"]
    r = _Gen(seed)
    sd: Dict[str, torch.Tensor] = {}
    sd["encoder.conv1.weight"] = r.n(D, dims["n_mels"], 3, std=1.0 / math.sqrt(3 * dims["n_mels"]))
    sd["encoder.conv1.bias"] = r.n(D, std=0.05)
    sd["encoder.conv2.weight"] = r.n(D, D, 3, std=1.0 / math.sqrt(3 * D))
    sd["encoder.conv2.bias"] = r.n(D, std=0.05)
    for i in range(kept):
        b = f"encoder.blocks.{i}"
        for nm in ("query", "key", "value", "out"):
            sd[f"{b}.attn.{nm}.weight"] = r.n(D, D, std=0.8 / math.sqrt(D))
            if nm != "key":
                sd[f"{b}.attn.{nm}.bias"] = r.n(D, std=0.05)
        sd[f"{b}.attn_ln.weight"] = 1.0 + r.n(D, std=0.1)
        sd[f"{b}.attn_ln.bias"] = r.n(D, std=0.1)
        sd[f"{b}.mlp.0.weight"] = r.n(4 * D, D, std=1.0 / math.sqrt(D))
        sd[f"{b}.mlp.0.bias"] = r.n(4 * D, std=0.05)
        sd[f"{b}.mlp.2.weight"] = r.n(D, 4 * D, std=0.5 / math.sqrt(4 * D))
        sd[f"{b}.mlp.2.bias"] = r.n(D, std=0.05)
        sd[f"{b}.mlp_ln.weight"] = 1.0 + r.n(D, std=0.1)
        sd[f"{b}.mlp_ln.bias"] = r.n(D, std=0.1)
    sd["encoder.ln_post.weight"] = 1.0 + r.n(D, std=0.1)
    sd["encoder.ln_post.bias"] = r.n(D, std=0.1)
    return {"dims": dims, "model_state_dict": {k: v.float().contiguous() for k, v in sd.items()}}


HUBERT_SOFT_DIMS = dict(conv_dim=512, d_model=768, n_head=12, d_ff=3072, n_layer=12, out_dim=256, pos_kernel=128, pos_groups=16)


def hubert_checkpoint(seed: int = 1234, n_layer: int = 12):
    """Synthetic HuBERT-Soft state dict in the reference's format (hubert/hubert_model.py:11-30,75-130: the keys
    `hubert_soft()` loads, :212-222).  No pretrained weights exist in the container (hubert_pretrain/ holds a README)."""
    r = _Gen(seed)
    C, D, FF = 512, 768, 3072
    sd: Dict[str, torch.Tensor] = {}
    sd["masked_spec_embed"] = r.n(D, std=0.3)
    sd["feature_extractor.conv0.weight"] = r.n(C, 1, 10, std=0.3)
    sd["feature_extractor.norm0.weight"] = 1.0 + r.n(C, std=0.1)
    sd["feature_extractor.norm0.bias"] = r.n(C, std=0.1)
    for i, k in enumerate((3, 3, 3, 3, 2, 2), 1):
        sd[f"feature_extractor.conv{i}.weight"] = r.n(C, C, k, std=1.4 / math.sqrt(C * k))
    sd["feature_projection.norm.weight"] = 1.0 + r.n(C, std=0.1)
    sd["feature_projection.norm.bias"] = r.n(C, std=0.1)
    sd["feature_projection.projection.weight"] = r.n(D, C, std=1.0 / math.sqrt(C))
    sd["feature_projection.projection.bias"] = r.n(D, std=0.05)
    v = r.n(D, 48, 128, std=1.0 / math.sqrt(48 * 128))
    sd["positional_embedding.conv.weight_v"] = v
    sd["positional_embedding.conv.weight_g"] = v.pow(2).sum((0, 1), keepdim=True).sqrt() * (1.0 + r.n(1, 1, 128, std=0.1))
    sd["positional_embedding.conv.bias"] = r.n(D, std=0.05)
    sd["norm.weight"] = 1.0 + r.n(D, std=0.1)
    sd["norm.bias"] = r.n(D, std=0.1)
    for i in range(n_layer):
        b = f"encoder.layers.{i}"
        sd[f"{b}.self_attn.in_proj_weight"] = r.n(3 * D, D, std=0.8 / math.sqrt(D))
        sd[f"{b}.self_attn.in_proj_bias"] = r.n(3 * D, std=0.05)
        sd[f"{b}.self_attn.out_proj.weight"] = r.n(D, D, std=0.8 / math.sqrt(D))
        sd[f"{b}.self_attn.out_proj.bias"] = r.n(D, std=0.05)
        sd[f"{b}.linear1.weight"] = r.n(FF, D, std=1.0 / math.sqrt(D))
        sd[f"{b}.linear1.bias"] = r.n(FF, std=0.05)
        sd[f"{b}.linear2.weight"] = r.n(D, FF, std=0.5 / math.sqrt(FF))
        sd[f"{b}.linear2.bias"] = r.n(D, std=0.05)
        for nm in ("norm1", "norm2"):
            sd[f"{b}.{nm}.weight"] = 1.0 + r.n(D, std=0.1)
            sd[f"{b}.{nm}.bias"] = r.n(D, std=0.1)
    sd["proj.weight"] = r.n(256, D, std=1.0 / math.sqrt(D))
    sd["proj.bias"] = r.n(256, std=0.05)
    sd["label_embedding.weight"] = r.n(100, 256, std=1.0)
    return {k: v.float().contiguous() for k, v in sd.items()}


def speaker_checkpoint(seed: int = 1234):
    """Synthetic LSTMSpeakerEncoder(80, 256, 768, 3) checkpoint {"model": state_dict} under the reference's keys
    (speaker/models/lstm.py:8-20,35-47).  Weights are xavier-normal like `_init_layers`, but the biases are random too
    (the reference zeroes them) so the bias paths are exercised."""
    r = _Gen(seed)
    H, P = 768, 256
    sd: Dict[str, torch.Tensor] = {}
    for l in range(3):
        n_in = 80 if l == 0 else P
        b = f"layers.{l}."
        sd[b + "lstm.weight_ih_l0"] = r.n(4 * H, n_in, std=math.sqrt(2.0 / (4 * H + n_in)))
        sd[b + "lstm.weight_hh_l0"] = r.n(4 * H, H, std=math.sqrt(2.0 / (5 * H)))
        sd[b + "lstm.bias_ih_l0"] = r.n(4 * H, std=0.1)
        sd[b + "lstm.bias_hh_l0"] = r.n(4 * H, std=0.1)
        sd[b + "linear.weight"] = r.n(P, H, std=math.sqrt(2.0 / (P + H)))
    return {"model": {k: v.float().contiguous() for k, v in sd.items()}}
