"""LSTM speaker encoder on the H100 path — host-side mirror of the reference's `speaker/infer.py` (`read_json`, the
checkpoint and config loading), `speaker/utils/audio.py` (`AudioProcessor.load_wav`, `melspectrogram`) and
`speaker/models/lstm.py` (`LSTMSpeakerEncoder.compute_embedding`) behind the C ABI (`svcb_speaker_*`,
csrc/speaker_api.cu).  No CPU fallback: a CUDA (sm_90a) device is required.

The host keeps the steps that decide shapes: reading and resampling the wav (`whisper_infer.load_audio`, with its
documented resampler deviation), the 160-sample margin, a restatement of librosa 0.10.1's `effects.trim` and the
volume normalisation.  The mel front end and the LSTM run on the device.  Silent audio, where the reference divides
by zero or fails on an empty array, raises `SvcbError`; so does audio of 512 samples or fewer after trimming, which the
device STFT's reflect padding cannot frame (the reference still embeds it).
"""
from __future__ import annotations

import ctypes
import json
import re
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

from . import _lib, pack
from .whisper_infer import _bf16_as_f32, load_audio, mel_filters

SAMPLE_RATE = 16000
N_FFT = 1024
HOP = 256
N_MELS = 80
HIDDEN = 768
PROJ = 256
LAYERS = 3
CTAS, UNITS = 128, 6          # the recurrence's CTAs and hidden units per CTA (csrc/speaker_api.cu)
K0 = 128                      # layer 0's input width (80 mels) padded to whole 64-wide GEMM k-tiles
MARGIN = 160                  # AudioProcessor.trim_silence: int(sample_rate * 0.01) samples cut at each end
NUM_WINDOWS, WINDOW = 10, 250  # compute_embedding's defaults


# ------------------------------------------------------------------------------------------------ config
def read_json(json_path: str) -> dict:
    """speaker/infer.py:14-35: plain JSON, or JSON with `//` comments and backslash line continuations."""
    with open(json_path, "r", encoding="utf-8") as f:
        text = f.read()
    try:
        return dict(json.loads(text))
    except json.decoder.JSONDecodeError:
        text = re.sub(r"\\\n", "", text)
        text = re.sub(r"//.*\n", "\n", text)
        return dict(json.loads(text))


# what this encoder implements; AudioProcessor's defaults (speaker/utils/audio.py:229-261) where the key is absent
_AUDIO_FIXED = dict(num_mels=N_MELS, sample_rate=SAMPLE_RATE, fft_size=N_FFT, win_length=N_FFT, hop_length=HOP,
                    log_func="np.log10", signal_norm=True, symmetric_norm=True, clip_norm=True, spec_gain=20,
                    stft_pad_mode="reflect", mel_fmin=0.0, do_amp_to_db_mel=True)
_AUDIO_DEFAULTS = dict(log_func="np.log10", clip_norm=True, spec_gain=20, stft_pad_mode="reflect", mel_fmin=0.0,
                       do_amp_to_db_mel=True, preemphasis=0.0, trim_db=60, max_norm=1.0)
_MODEL_FIXED = dict(input_dim=N_MELS, proj_dim=PROJ, lstm_dim=HIDDEN, num_lstm_layers=LAYERS, use_lstm_with_projection=True)


def audio_params(config: dict) -> dict:
    """Validate a speaker-encoder config (speaker_pretrain/config.json) against what the device path implements and
    return the values it passes through: preemphasis, ref_level_db, min_level_db, max_norm, trim_db."""
    def bad(what):
        raise ValueError(f"unsupported speaker encoder config: {what}")

    name = config.get("model_name", "lstm")
    if name != "lstm":
        bad(f"model_name {name!r} (only the LSTM encoder is implemented)")
    for key in ("model_params", "model"):
        mp = config.get(key)
        if isinstance(mp, dict):
            if mp.get("model_name", "lstm") != "lstm":
                bad(f"{key}.model_name {mp.get('model_name')!r}")
            for k, v in _MODEL_FIXED.items():
                if k in mp and mp[k] != v:
                    bad(f"{key}.{k} = {mp[k]!r}, need {v!r}")
    a = config.get("audio")
    if not isinstance(a, dict):
        bad("no audio section")
    get = lambda k: a.get(k, _AUDIO_DEFAULTS.get(k))   # noqa: E731
    for k, v in _AUDIO_FIXED.items():
        got = get(k)
        if got is None or (isinstance(v, bool) and got is not v) or got != v:
            bad(f"audio.{k} = {got!r}, need {v!r}")
    if get("mel_fmax") not in (None, SAMPLE_RATE / 2):
        bad(f"audio.mel_fmax = {get('mel_fmax')!r}, need {SAMPLE_RATE / 2}")
    if a.get("stats_path"):
        bad("audio.stats_path (mean-variance scaling) is not implemented")
    out = {k: float(get(k)) if get(k) is not None else None for k in ("preemphasis", "ref_level_db", "min_level_db", "max_norm", "trim_db")}
    for k, v in out.items():
        if v is None or not np.isfinite(v):
            bad(f"audio.{k} missing")
    if out["min_level_db"] == 0.0:
        bad("audio.min_level_db is 0")
    return out


# ------------------------------------------------------------------------------------------------ packing
def gate_order() -> np.ndarray:
    """Row j = 24 c + 4 u + g of the packed gate matrices is nn.LSTM row g * 768 + 6 c + u: CTA c's six units with their
    four gates (i, f, g, o) side by side."""
    c, u, g = np.meshgrid(np.arange(CTAS), np.arange(UNITS), np.arange(4), indexing="ij")
    return (g * HIDDEN + c * UNITS + u).reshape(-1)


def _split(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    hi = w.bfloat16().float()
    return hi, w - hi


def _tripled_image(w: torch.Tensor, kseg: int) -> torch.Tensor:
    """[N, K] fp32 -> bf16 tile image of [W_hi | W_hi | W_lo] (each segment zero-padded to kseg): against the activation
    image [x_hi | x_lo | x_hi] one bf16 GEMM gives the bf16x3 product."""
    hi, lo = _split(w.float())
    n, k = w.shape
    seg = lambda t: torch.nn.functional.pad(t, (0, kseg - k))   # noqa: E731
    return _bf16_as_f32(torch.cat([seg(hi), seg(hi), seg(lo)], 1))


def pack_speaker(sd: Dict[str, torch.Tensor], audio: dict) -> List[Tuple[str, torch.Tensor]]:
    """-> [(name, fp32-typed tensor)], the names csrc/speaker_api.cu reads.  State-dict keys: lstm.py:8-20,35-47."""
    perm = torch.from_numpy(gate_order())
    items = [("spk.mel_fb", mel_filters(N_MELS, SAMPLE_RATE, N_FFT).contiguous()),
             ("spk.audio", torch.tensor([audio["preemphasis"], audio["ref_level_db"], audio["min_level_db"], audio["max_norm"]],
                                        dtype=torch.float32))]
    for l in range(LAYERS):
        p = f"layers.{l}."
        wih = sd[p + "lstm.weight_ih_l0"].float()
        whh = sd[p + "lstm.weight_hh_l0"].float()
        want_in = N_MELS if l == 0 else PROJ
        if tuple(wih.shape) != (4 * HIDDEN, want_in) or tuple(whh.shape) != (4 * HIDDEN, HIDDEN):
            raise ValueError(f"layer {l}: LSTM weights {tuple(wih.shape)}, {tuple(whh.shape)}; need ({4 * HIDDEN}, {want_in}), "
                             f"({4 * HIDDEN}, {HIDDEN})")
        items.append((f"spk.l{l}.wih", _tripled_image(wih[perm], K0 if l == 0 else PROJ)))
        bias = sd[p + "lstm.bias_ih_l0"].float() + sd[p + "lstm.bias_hh_l0"].float()
        items.append((f"spk.l{l}.b", bias[perm].contiguous()))
        # the recurrence's resident slices: per CTA [hi, lo][k / 8][24 gate columns][8] bf16 (K-major wgmma panels)
        hi, lo = _split(whh[perm].reshape(CTAS, 4 * UNITS, HIDDEN))
        panel = lambda t: t.bfloat16().view(CTAS, 4 * UNITS, HIDDEN // 8, 8).permute(0, 2, 1, 3)   # noqa: E731
        items.append((f"spk.l{l}.whh", torch.stack([panel(hi), panel(lo)], 1).contiguous().view(torch.float32).reshape(-1)))
        wp = sd[p + "linear.weight"].float()
        if tuple(wp.shape) != (PROJ, HIDDEN):
            raise ValueError(f"layer {l}: projection {tuple(wp.shape)}, need ({PROJ}, {HIDDEN})")
        items.append((f"spk.l{l}.wproj", _tripled_image(wp, HIDDEN)))
    return items


# ------------------------------------------------------------------------------------------------ audio (host)
def trim(y: np.ndarray, top_db: float = 60, frame_length: int = N_FFT, hop_length: int = HOP) -> np.ndarray:
    """librosa 0.10.1 `effects.trim` (ref=np.max, aggregate=np.max) for mono audio: float32 RMS of frames centred with
    zero padding, `amplitude_to_db(ref=np.max)` > -top_db, cut from the first to past the last non-silent frame."""
    y = np.asarray(y, np.float32)
    pad = frame_length // 2
    yp = np.pad(y, (pad, pad), mode="constant")
    n = 1 + (yp.shape[0] - frame_length) // hop_length
    frames = np.lib.stride_tricks.sliding_window_view(yp, frame_length)[::hop_length][:n]
    rms = np.sqrt(np.mean(np.square(frames, dtype=np.float32), axis=-1, dtype=np.float32))
    power = np.square(rms)
    ref = np.square(rms.max())
    db = np.float32(10.0) * np.log10(np.maximum(np.float32(1e-10), power)) - np.float32(10.0) * np.log10(np.maximum(np.float32(1e-10), ref))
    nz = np.flatnonzero(db > -top_db)
    if nz.size == 0:
        return y[:0]
    start = int(nz[0]) * hop_length
    end = min(y.shape[0], (int(nz[-1]) + 1) * hop_length)
    return y[start:end]


def prepare_wav(x: np.ndarray, trim_db: float = 60) -> np.ndarray:
    """AudioProcessor.load_wav after reading (audio.py:714-733, do_trim_silence and do_sound_norm as infer.py sets them):
    the 160-sample margin, trim, then x / max|x| * 0.95."""
    x = np.asarray(x, np.float32)
    x = x[MARGIN:x.shape[0] - MARGIN]
    if x.size == 0 or not np.any(x):
        raise _lib.SvcbError(f"speaker encoder: the audio is silent or shorter than {2 * MARGIN + 1} samples")
    x = trim(x, trim_db)
    if x.shape[0] <= N_FFT // 2:
        raise _lib.SvcbError(f"speaker encoder: {x.shape[0]} samples left after trimming; the reflect-padded STFT needs "
                             f"more than {N_FFT // 2}")
    return x / np.abs(x).max() * np.float32(0.95)


def load_wav(path: str, trim_db: float = 60) -> np.ndarray:
    """AudioProcessor.load_wav(path, sr=16000) as speaker/infer.py configures it."""
    return prepare_wav(load_audio(path, SAMPLE_RATE), trim_db)


def window_offsets(T: int) -> List[int]:
    """compute_embedding's window starts: int(np.linspace(0, T - min(250, T), 10)) (lstm.py:81-92)."""
    L = min(WINDOW, T)
    return [int(o) for o in np.linspace(0, T - L, num=NUM_WINDOWS)]


# ------------------------------------------------------------------------------------------------ the model
class SpeakerEncoderB200:
    """LSTMSpeakerEncoder(80, 256, 768, 3) with its AudioProcessor, for inference."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], audio: dict, device):
        self.device = _lib.cuda_device(device)
        self.audio = dict(audio)
        blob_cpu, table = pack.build_blob(pack_speaker(state_dict, self.audio))
        self._handle = _lib.Handle("speaker", table, blob_cpu.to(self.device))

    @staticmethod
    def frames(n_samples: int) -> int:
        return int(_lib.load().svcb_speaker_frames(int(n_samples)))

    def load_wav(self, path: str) -> np.ndarray:
        return load_wav(path, self.audio["trim_db"])

    @torch.no_grad()
    def mel_batch(self, wavs: Sequence) -> Tuple[torch.Tensor, List[int]]:
        """Ragged batch of prepared waveforms -> (mel [sum T_b, 80] on the device, frame offsets [B + 1])."""
        flat, so = _lib.ragged(wavs, self.device)
        B = len(so) - 1
        fo = list(_lib.offsets(self.frames(so[b + 1] - so[b]) for b in range(B)))
        mel = torch.empty(max(fo[-1], 1), N_MELS, device=self.device, dtype=torch.float32)
        self._handle.call("speaker_mel", flat.data_ptr(), so, B, mel.data_ptr(), None, 0)
        return mel[:fo[-1]], fo

    @torch.no_grad()
    def embed_mels(self, mel: torch.Tensor, frame_offsets: Sequence[int], windows: bool = False):
        """mel [sum T_b, 80] (time-major), frame offsets [B + 1] -> [B, 256] (and the window embeddings [B, 10, 256])."""
        mel = mel.to(self.device, torch.float32).contiguous()
        B = len(frame_offsets) - 1
        ws = self._handle.workspace(_lib.load().svcb_speaker_workspace_bytes(self._handle, B, int(HOP * max(1, mel.shape[0]))))
        out = torch.empty(B, PROJ, device=self.device, dtype=torch.float32)
        wout = torch.empty(B, NUM_WINDOWS, PROJ, device=self.device, dtype=torch.float32) if windows else None
        offs = (ctypes.c_int64 * (B + 1))(*[int(o) for o in frame_offsets])
        self._handle.call("speaker_embed", mel.data_ptr(), offs, B, out.data_ptr(), wout.data_ptr() if windows else None,
                          ws.data_ptr(), ws.numel())
        return (out, wout) if windows else out

    def melspectrogram(self, wav) -> torch.Tensor:
        """AudioProcessor.melspectrogram of one prepared waveform, time-major [T, 80] (the reference returns [80, T])."""
        return self.mel_batch([wav])[0]

    def compute_embedding(self, mel: torch.Tensor) -> torch.Tensor:
        """LSTMSpeakerEncoder.compute_embedding: mel [T, 80] or [1, T, 80] -> [1, 256]."""
        mel = mel.reshape(-1, N_MELS)
        return self.embed_mels(mel, [0, mel.shape[0]])

    def embed(self, wavs: Sequence) -> torch.Tensor:
        """Prepared waveforms (ragged) -> [B, 256]: one call of each device entry point."""
        mel, fo = self.mel_batch(wavs)
        return self.embed_mels(mel, fo)


def load_model(model_path: str, config_path: str, device="cuda") -> SpeakerEncoderB200:
    """speaker/infer.py:63-84: the Coqui checkpoint {"model": state_dict} and its JSON config."""
    audio = audio_params(read_json(config_path))
    state = torch.load(model_path, map_location="cpu", weights_only=False)   # Coqui checkpoints pickle more than tensors
    sd = state["model"] if isinstance(state, dict) and "model" in state else state
    return SpeakerEncoderB200(sd, audio, device)
