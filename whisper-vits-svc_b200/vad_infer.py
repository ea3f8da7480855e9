"""Silero voice-activity detector on the H100 path -- host-side mirror of the reference's `vad/utils.py`
(`init_jit_model`, `get_speech_timestamps`) and the silencing rule of `svc_inference_post.py`, behind the C ABI
(`svcb_vad_*`, csrc/vad_api.cu).  No CPU fallback: a CUDA (sm_90a) device is required for the probabilities.

`load_model` opens `silero_vad.jit` only as a container of tensors (the TorchScript is never run) and reads the 16 kHz
branch `_model.*`; any other layout is rejected.  The host keeps the steps that decide shapes: the speech segments
(`get_speech_timestamps`, restated from the reference's 16 kHz semantics) and the mask.  Audio with no samples never
reaches the device: it has no windows, so no probabilities and no speech.
"""
from __future__ import annotations

import ctypes  # noqa: F401  (callers build svcb_vad_probs offset arrays through vad_infer.ctypes)
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

from . import _lib, pack

SAMPLE_RATE = 16000
WINDOW = 512          # samples per probability
FILTER_LENGTH, HOP_LENGTH, TO_PAD = 256, 64, 3
HIDDEN = 64
BN_EPS = 1e-5


def _block(p, cin, cout, proj=True):
    d = {f"{p}.dw_conv.0.weight": (cin, 1, 5), f"{p}.dw_conv.0.bias": (cin,),
         f"{p}.pw_conv.0.weight": (cout, cin, 1), f"{p}.pw_conv.0.bias": (cout,)}
    if proj:
        d.update({f"{p}.proj.weight": (cout, cin, 1), f"{p}.proj.bias": (cout,)})
    return d


def _conv_bn(i, c):
    return {f"encoder.{i}.weight": (c, c, 1), f"encoder.{i}.bias": (c,),
            **{f"encoder.{i + 1}.{n}": (c,) for n in ("weight", "bias", "running_mean", "running_var")}}


# the 16 kHz branch of silero_vad.jit (keys below `_model.`) and the shapes the device path implements
SHAPES: Dict[str, Tuple[int, ...]] = {
    "feature_extractor.forward_basis_buffer": (2 * (FILTER_LENGTH // 2 + 1), 1, FILTER_LENGTH),
    "adaptive_normalization.filter_": (1, 1, 2 * TO_PAD + 1),
    **_block("first_layer.0", 258, 16),
    **_conv_bn(0, 16), **_block("encoder.3.0", 16, 32),
    **_conv_bn(4, 32), **_block("encoder.7.0", 32, 32, proj=False),
    **_conv_bn(8, 32), **_block("encoder.11.0", 32, 64),
    **_conv_bn(12, 64),
    **{f"decoder.rnn.{w}_l{l}": (4 * HIDDEN, HIDDEN) for l in (0, 1) for w in ("weight_ih", "weight_hh")},
    **{f"decoder.rnn.{b}_l{l}": (4 * HIDDEN,) for l in (0, 1) for b in ("bias_ih", "bias_hh")},
    "decoder.decoder.1.weight": (1, HIDDEN, 1), "decoder.decoder.1.bias": (1,),
}


# ------------------------------------------------------------------------------------------------ the model file
def check_model(sd: Dict[str, torch.Tensor], filter_length, hop_length, to_pad) -> Dict[str, torch.Tensor]:
    """The 16 kHz branch's tensors (keys without `_model.`) and STFT / normalisation settings -> fp32 tensors, or a
    ValueError naming what differs from the Silero VAD layout the device path implements."""
    what = "not the Silero VAD 16 kHz model this build implements (vad/assets/silero_vad.jit)"
    missing = [k for k in SHAPES if k not in sd]
    if missing:
        raise ValueError(f"{what}: missing _model.{missing[0]}" + (f" and {len(missing) - 1} more" if len(missing) > 1 else ""))
    for k, shape in SHAPES.items():
        if tuple(sd[k].shape) != shape:
            raise ValueError(f"{what}: _model.{k} has shape {tuple(sd[k].shape)}, need {shape}")
    for name, got, need in (("filter_length", filter_length, FILTER_LENGTH), ("hop_length", hop_length, HOP_LENGTH),
                            ("to_pad", to_pad, TO_PAD)):
        if got != need:
            raise ValueError(f"{what}: {name} is {got!r}, need {need}")
    return {k: sd[k].detach().float().contiguous() for k in SHAPES}


def read_model(path: str) -> Dict[str, torch.Tensor]:
    """silero_vad.jit -> the checked 16 kHz tensors.  The file is opened as a tensor container only."""
    m = torch.jit.load(path, map_location="cpu")
    sd = {k[len("_model."):]: v for k, v in m.state_dict().items() if k.startswith("_model.")}
    inner = getattr(m, "_model", None)
    fe = getattr(inner, "feature_extractor", None)
    an = getattr(inner, "adaptive_normalization", None)
    return check_model(sd, getattr(fe, "filter_length", None), getattr(fe, "hop_length", None), getattr(an, "to_pad", None))


# ------------------------------------------------------------------------------------------------ packing
def pack_vad(sd: Dict[str, torch.Tensor]) -> List[Tuple[str, torch.Tensor]]:
    """-> [(name, fp32 tensor)], the names csrc/vad_api.cu reads.  BatchNorm becomes an eval scale and shift."""
    basis = sd["feature_extractor.forward_basis_buffer"].reshape(2, FILTER_LENGTH // 2 + 1, FILTER_LENGTH)
    # bins 0..127 as [re / im][k / 4][bin][4] (a thread's four taps are one float4); bin 128 apart
    basis4 = basis[:, :128].reshape(2, 128, FILTER_LENGTH // 4, 4).permute(0, 2, 1, 3)
    items = [("vad.basis4", basis4), ("vad.nyq", basis[:, 128]), ("vad.filt", sd["adaptive_normalization.filter_"])]
    for name, p, proj in (("fl", "first_layer.0", True), ("b1", "encoder.3.0", True), ("b2", "encoder.7.0", False),
                          ("b3", "encoder.11.0", True)):
        items += [(f"vad.{name}.dw_w", sd[f"{p}.dw_conv.0.weight"]), (f"vad.{name}.dw_b", sd[f"{p}.dw_conv.0.bias"]),
                  (f"vad.{name}.pw_w", sd[f"{p}.pw_conv.0.weight"]), (f"vad.{name}.pw_b", sd[f"{p}.pw_conv.0.bias"])]
        if proj:
            items += [(f"vad.{name}.pj_w", sd[f"{p}.proj.weight"]), (f"vad.{name}.pj_b", sd[f"{p}.proj.bias"])]
    for i in (0, 4, 8, 12):
        bn = {n: sd[f"encoder.{i + 1}.{n}"].double() for n in ("weight", "bias", "running_mean", "running_var")}
        scale = bn["weight"] / torch.sqrt(bn["running_var"] + BN_EPS)
        items += [(f"vad.e{i}.w", sd[f"encoder.{i}.weight"]), (f"vad.e{i}.b", sd[f"encoder.{i}.bias"]),
                  (f"vad.e{i}.bn", torch.cat([scale, bn["bias"] - bn["running_mean"] * scale]).float())]
    r = {k: sd[f"decoder.rnn.{k}"] for k in ("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0",
                                             "weight_ih_l1", "weight_hh_l1", "bias_ih_l1", "bias_hh_l1")}
    items += [("vad.wih0t", r["weight_ih_l0"].t()), ("vad.b0", r["bias_ih_l0"] + r["bias_hh_l0"]),
              ("vad.wrec", torch.stack([r["weight_hh_l0"].t(), r["weight_ih_l1"].t(), r["weight_hh_l1"].t()])),
              ("vad.b1sum", r["bias_ih_l1"] + r["bias_hh_l1"]),
              ("vad.dec", torch.cat([sd["decoder.decoder.1.weight"].reshape(-1), sd["decoder.decoder.1.bias"]]))]
    return [(n, t.float().contiguous()) for n, t in items]


# ------------------------------------------------------------------------------------------------ the model
def windows(n_samples: int) -> int:
    """Probabilities of n_samples of 16 kHz audio: ceil(n / 512); the last window is zero-padded."""
    return -(-int(n_samples) // WINDOW) if n_samples > 0 else 0


_stream = _lib.stream   # the stream argument of a direct svcb_vad_* call on a VadB200's `_handle`


class VadB200:
    """The 16 kHz Silero VAD, for inference on ragged batches of recordings."""

    def __init__(self, tensors: Dict[str, torch.Tensor], device):
        self.device = _lib.cuda_device(device)
        blob_cpu, table = pack.build_blob(pack_vad(tensors))
        self._handle = _lib.Handle("vad", table, blob_cpu.to(self.device))

    @torch.no_grad()
    def speech_probs_device(self, wavs: Sequence, features: bool = False):
        """Ragged batch of 16 kHz waveforms -> (probs [sum W_b] on the device, window offsets [B + 1]) and, with
        `features`, the encoder outputs [sum W_b, 64]."""
        flat, so = _lib.ragged(wavs, self.device)
        B = len(so) - 1
        wo = list(_lib.offsets(windows(so[b + 1] - so[b]) for b in range(B)))
        W = wo[-1]
        probs = torch.empty(max(W, 1), device=self.device, dtype=torch.float32)
        feat = torch.empty(max(W, 1), HIDDEN, device=self.device, dtype=torch.float32) if features else None
        if W > 0:
            ws = self._handle.workspace(_lib.load().svcb_vad_workspace_bytes(self._handle, B, W))
            self._handle.call("vad_probs", flat.data_ptr(), so, B, probs.data_ptr(),
                              feat.data_ptr() if features else None, ws.data_ptr(), ws.numel())
        out = (probs[:W], wo)
        return out + (feat[:W],) if features else out

    def speech_probs(self, wavs: Sequence, features: bool = False):
        """Ragged batch of 16 kHz waveforms -> a list of per-window fp32 probabilities (and of [W_b, 64] encoder
        outputs with `features`)."""
        r = self.speech_probs_device(wavs, features)
        probs = _lib.split(r[0].cpu().numpy(), r[1])
        return (probs, _lib.split(r[2].cpu().numpy(), r[1])) if features else probs


def load_model(path: str, device="cuda") -> VadB200:
    """vad/utils.py:init_jit_model in effect: silero_vad.jit -> the device model."""
    return VadB200(read_model(path), device)


# ------------------------------------------------------------------------------------------------ segments (host)
def get_speech_timestamps(probs, n_samples: int, threshold: float = 0.5, min_speech_duration_ms: int = 250,
                          max_speech_duration_s: float = float("inf"), min_silence_duration_ms: int = 100,
                          speech_pad_ms: int = 30, window_size_samples: int = WINDOW) -> List[dict]:
    """Speech segments [{'start', 'end'}] in samples from one probability per window of n_samples of 16 kHz audio,
    with the semantics of vad/utils.py:get_speech_timestamps (return_seconds False).

    A segment opens at the first window at or above `threshold` and closes once the probability has stayed below
    `threshold - 0.15` for `min_silence_duration_ms`; it ends where that silence began.  Segments of
    `min_speech_duration_ms` or less are dropped.  A segment longer than `max_speech_duration_s` (less one window and
    both pads) is cut at the start of its last silence of more than 98 ms, where it resumes at the next speech window,
    or else just before the limit.  An open segment runs to the end of the audio.  Each segment is then widened by
    `speech_pad_ms`, and the gap between neighbours closer than two pads is split between them."""
    sr = SAMPLE_RATE
    step = window_size_samples
    min_speech = sr * min_speech_duration_ms / 1000
    pad = sr * speech_pad_ms / 1000
    max_speech = sr * max_speech_duration_s - step - 2 * pad
    min_silence = sr * min_silence_duration_ms / 1000
    min_silence_at_max = sr * 98 / 1000
    low = threshold - 0.15

    segs: List[dict] = []
    active = False
    start = 0
    silence_from = 0      # first window of the current silence (0: none)
    cut_at = 0            # where a segment over the limit may be cut: the start of an earlier long silence
    resume_at = 0         # the first speech window after that silence
    for i, p in enumerate(float(x) for x in probs):
        pos = step * i
        if p >= threshold and silence_from:
            silence_from = 0
            if resume_at < cut_at:
                resume_at = pos
        if p >= threshold and not active:
            active, start = True, pos
            continue
        if active and pos - start > max_speech:
            if cut_at:
                segs.append({"start": start, "end": cut_at})
                if resume_at < cut_at:     # still in that silence: close
                    active = False
                else:
                    start = resume_at
                cut_at = resume_at = silence_from = 0
            else:
                segs.append({"start": start, "end": pos})
                cut_at = resume_at = silence_from = 0
                active = False
                continue
        if p < low and active:
            if not silence_from:
                silence_from = pos
            if pos - silence_from > min_silence_at_max:
                cut_at = silence_from
            if pos - silence_from < min_silence:
                continue
            if silence_from - start > min_speech:
                segs.append({"start": start, "end": silence_from})
            cut_at = resume_at = silence_from = 0
            active = False
            continue
    if active and n_samples - start > min_speech:
        segs.append({"start": start, "end": n_samples})

    for i, s in enumerate(segs):
        if i == 0:
            s["start"] = int(max(0, s["start"] - pad))
        if i + 1 < len(segs):
            gap = segs[i + 1]["start"] - s["end"]
            if gap < 2 * pad:
                s["end"] += int(gap // 2)
                segs[i + 1]["start"] = int(max(0, segs[i + 1]["start"] - gap // 2))
            else:
                s["end"] = int(min(n_samples, s["end"] + pad))
                segs[i + 1]["start"] = int(max(0, segs[i + 1]["start"] - pad))
        else:
            s["end"] = int(min(n_samples, s["end"] + pad))
    return segs


def silence_outside_speech(timestamps: Sequence[dict], n_ref16: int, svc32: np.ndarray) -> np.ndarray:
    """svc_inference_post.py's rule: a 0/1 mask over each segment's [start, end) of the 16 kHz reference, each sample
    repeated for 32 kHz; both signals cut to the shorter; the converted audio zeroed where the mask is 0."""
    mask = np.zeros(int(n_ref16), np.float32)
    for t in timestamps:
        mask[t["start"]:t["end"]] = 1
    mask = np.repeat(mask, 2, -1)
    n = min(mask.shape[0], svc32.shape[0])
    out = np.array(svc32[:n], np.float32, copy=True)
    out[mask[:n] == 0] = 0
    return out
