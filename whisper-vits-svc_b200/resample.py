"""Resampling of raw recordings for training on the H100 path: `librosa.load(path, sr)` and the int16 normalisation of
the reference's `prepare/preprocess_a.py:resample_wave`, behind the C ABI (`svcb_resample_ragged`,
`svcb_pcm16_normalise_ragged`, csrc/resample_api.cu).  No CPU fallback: a CUDA (sm_90a) device is required.

The resampler is scipy.signal.resample_poly's polyphase Kaiser FIR (the project's resampling rule, as in
`whisper_infer.load_audio`), evaluated with fp64 taps and accumulation and rounded once to float32, so the output is
`resample_poly(x.astype(float64), up, down).astype(float32)`.  librosa 0.10.1 resamples with soxr instead: the lengths
agree, ceil(n sr_out / sr_in), and the values differ slightly.  When the rates are equal nothing is resampled."""
from __future__ import annotations

import math
from typing import List, Sequence, Tuple

import numpy as np
import torch

from . import _lib

_TAPS = {}   # (up, down, device) -> (device fp64 taps, pre_remove)


def scale_pcm(x: np.ndarray) -> np.ndarray:
    """Samples as scipy reads them -> float32, as librosa and torchaudio decode them: integer PCM scaled to [-1, 1)
    (8-bit is unsigned around 128), float PCM as stored."""
    if x.dtype == np.uint8:     # 8-bit WAV is unsigned with the zero level at 128
        x = (x.astype(np.float32) - 128.0) / 128.0
    elif x.dtype.kind in "iu":
        x = x.astype(np.float32) / float(np.iinfo(x.dtype).max + 1)
    return x.astype(np.float32)


def decode_wav(path: str) -> Tuple[int, np.ndarray]:
    """(rate, float32 mono) of a .wav as librosa decodes it: `scale_pcm`, channels averaged."""
    from scipy.io import wavfile
    rate, x = wavfile.read(path)
    x = scale_pcm(x)
    if x.ndim > 1:
        x = x.mean(axis=1)
    return int(rate), x


def load(path: str) -> Tuple[np.ndarray, int]:
    """(float32 mono samples, rate) of a .wav; ValueError for a file without samples or with non-finite ones."""
    rate, x = decode_wav(path)
    if x.shape[0] == 0:
        raise ValueError("no samples")
    if not np.isfinite(x).all():
        raise ValueError("non-finite samples")
    return x, rate


def ratio(sr_in: int, sr_out: int) -> Tuple[int, int]:
    """(up, down): sr_out / sr_in reduced by their gcd."""
    sr_in, sr_out = int(sr_in), int(sr_out)
    if sr_in < 1 or sr_out < 1:
        raise ValueError(f"sampling rates must be positive, got {sr_in} -> {sr_out}")
    g = math.gcd(sr_in, sr_out)
    return sr_out // g, sr_in // g


def out_len(n: int, sr_in: int, sr_out: int) -> int:
    """Samples after resampling n: ceil(n up / down), resample_poly's and librosa's length."""
    up, down = ratio(sr_in, sr_out)
    return -(-int(n) * up // down)


def design(up: int, down: int) -> Tuple[np.ndarray, int]:
    """resample_poly's filter for up/down in fp64, pre-padded so output j sits at input phase (j + pre_remove) down:
    (taps, pre_remove)."""
    from scipy.signal import firwin
    half = 10 * max(up, down)
    h = firwin(2 * half + 1, 1.0 / max(up, down), window=("kaiser", 5.0)) * up
    pre = down - half % down
    return np.concatenate([np.zeros(pre), h]), (half + pre) // down


def _device_taps(up: int, down: int, dev: torch.device):
    key = (up, down, str(dev))
    if key not in _TAPS:
        taps, rm = design(up, down)
        _TAPS[key] = (torch.from_numpy(taps).to(dev), rm)
    return _TAPS[key]


def release_filters() -> None:
    """Free the device filters cached by earlier calls, so that a process running other device work afterwards gets
    their memory back.  The next call designs and uploads its filter again."""
    _TAPS.clear()


def _resample_device(audios: Sequence, sr_in: int, sr_out: int, dev: torch.device):
    """The batch resampled on the device: (flat float32 device tensor, output offsets).  Equal rates copy the input."""
    up, down = ratio(sr_in, sr_out)
    flat, so = _lib.ragged(audios, dev)
    if up == down:
        return flat, so
    B = len(so) - 1
    oo = _lib.offsets(out_len(so[b + 1] - so[b], sr_in, sr_out) for b in range(B))
    taps, rm = _device_taps(up, down, dev)
    y = torch.empty(max(oo[-1], 1), dtype=torch.float32, device=dev)
    _lib.call("resample_ragged", flat.data_ptr(), so, B, up, down, taps.data_ptr(), taps.numel(), rm, y.data_ptr(),
              device=dev)
    return y, oo


@torch.no_grad()
def resample_batch(audios: Sequence, sr_in: int, sr_out: int, device="cuda") -> List[np.ndarray]:
    """Clips at sr_in (ragged, each at least one sample) -> float32 clips at sr_out, one device call."""
    dev = _lib.cuda_device(device)
    if not audios:
        return []
    y, oo = _resample_device(audios, sr_in, sr_out, dev)
    return _lib.split(y.cpu().numpy(), oo)


@torch.no_grad()
def pcm16_batch(audios: Sequence, sr_in: int, sr_out: int, device="cuda") -> Tuple[List[np.ndarray], np.ndarray]:
    """Clips at sr_in -> (int16 clips at sr_out as resample_wave writes them, float32 peaks max|y|), one resampling
    and one normalising call; only the int16 samples and the peaks are copied back.  A peak of 0 marks a silent clip,
    whose samples are zeros (the reference would divide by zero)."""
    dev = _lib.cuda_device(device)
    if not audios:
        return [], np.zeros(0, np.float32)
    y, oo = _resample_device(audios, sr_in, sr_out, dev)
    out = torch.empty(max(oo[-1], 1), dtype=torch.int16, device=dev)
    peak = torch.empty(len(audios), dtype=torch.float32, device=dev)
    _lib.call("pcm16_normalise_ragged", y.data_ptr(), oo, len(audios), out.data_ptr(), peak.data_ptr(), device=dev)
    return _lib.split(out.cpu().numpy(), oo), peak.cpu().numpy()
