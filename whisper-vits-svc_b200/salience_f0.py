"""Salience-based F0 on the H100 path: the reference's `pitch/inference.py:compute_f0_salience`, libf0's Melodia-style
tracker (`pitch/core/salience.py:salience` at 16 kHz, a 2048-sample window, a 320-sample hop and 45-1760 Hz).  The
analysis, harmonic summation and dynamic programming run on the device in fp64 (`svcb_salience_f0_ragged`,
csrc/salience_f0_api.cu); only the reference's repeat and moving average are on the host.  No CPU fallback: a CUDA
(sm_90a) device is required.

Audio is read as `praat_f0.py` reads it: `hubert_infer.load_audio(path, 16000)`, .wav only, resampled with
`resample_poly` where the file is not at 16 kHz (the reference's librosa.load resamples with soxr)."""
from __future__ import annotations

from typing import List, Sequence

import numpy as np
import torch

from . import _lib

SAMPLE_RATE = 16000
HOP = 320
BINS = 636
MIN_SAMPLES = HOP          # two frames: the instantaneous frequency needs a pair


def frames_of(n: int) -> int:
    """Frames of n samples: the centred STFT's n // 320 + 1."""
    return int(n) // HOP + 1


def finish(f0: np.ndarray) -> np.ndarray:
    """compute_f0_salience's host tail: every value twice (20 ms -> 10 ms), then a centred moving average over 3."""
    f0 = np.repeat(f0, 2, -1)
    return np.convolve(f0, np.ones((3,)) / 3, mode="same")


class Extractor:
    """One device and a grow-only workspace for `svcb_salience_f0_ragged`.  `close()` frees the workspace."""

    def __init__(self, device="cuda"):
        self.device = _lib.cuda_device(device)
        self._ws = None

    def workspace(self, nbytes: int) -> torch.Tensor:
        if self._ws is None or self._ws.numel() < nbytes:
            self._ws = None
            self._ws = torch.empty(int(nbytes), dtype=torch.uint8, device=self.device)
        return self._ws

    def close(self) -> None:
        self._ws = None

    @torch.no_grad()
    def raw(self, clips: Sequence, taps: bool = False):
        """Float clips at 16 kHz (each >= 320 samples) -> each one's float64 F0 per 20 ms frame on the device.  With
        taps, also each one's binned spectrogram Y and salience Z ([636, frames] float64) and path bins (int32)."""
        if not clips:
            return []
        flat, so = _lib.ragged(clips, self.device)
        lens = [so[b + 1] - so[b] for b in range(len(so) - 1)]
        fo = _lib.offsets(frames_of(n) if n >= MIN_SAMPLES else 1 for n in lens)   # too short: refused before a launch
        f0 = torch.empty(fo[-1], dtype=torch.float64, device=self.device)
        y = z = path = None
        if taps:
            y = torch.empty(BINS * fo[-1], dtype=torch.float64, device=self.device)
            z = torch.empty_like(y)
            path = torch.empty(fo[-1], dtype=torch.int32, device=self.device)
        ptr = lambda t: t.data_ptr() if t is not None else None
        need = _lib.load().svcb_salience_f0_workspace_bytes(so[-1] - so[0], len(lens))
        ws = self.workspace(need)
        _lib.call("salience_f0_ragged", flat.data_ptr(), so, len(lens), f0.data_ptr(), ptr(y), ptr(z), ptr(path),
                  ws.data_ptr(), ws.numel(), device=self.device)
        out = _lib.split(f0, fo)
        if not taps:
            return out
        bo = [BINS * o for o in fo]
        F = [fo[b + 1] - fo[b] for b in range(len(lens))]
        return [(out[b], y[bo[b]:bo[b + 1]].view(BINS, F[b]), z[bo[b]:bo[b + 1]].view(BINS, F[b]),
                 path[fo[b]:fo[b + 1]]) for b in range(len(lens))]

    def f0_batch(self, clips: Sequence) -> List[np.ndarray]:
        """Float clips at 16 kHz -> each one's float64 F0 as compute_f0_salience returns it (2 (n // 320 + 1) values)."""
        return [finish(f.cpu().numpy()) for f in self.raw(clips)]


def f0_batch(clips: Sequence, device="cuda") -> List[np.ndarray]:
    """Float clips at 16 kHz -> compute_f0_salience's float64 F0 of each; one device call."""
    ex = Extractor(device)
    try:
        return ex.f0_batch(clips)
    finally:
        ex.close()


def dp_paths(zs: Sequence[torch.Tensor], device="cuda") -> List[np.ndarray]:
    """The device's DP and trace back alone on given saliences ([636, frames] float64 each) -> each one's path bins."""
    dev = _lib.cuda_device(device)
    fo = _lib.offsets(z.shape[1] for z in zs)
    flat = torch.cat([torch.as_tensor(z, dtype=torch.float64).reshape(-1) for z in zs]).to(dev)
    path = torch.empty(fo[-1], dtype=torch.int32, device=dev)
    ws = torch.empty(max(1, _lib.load().svcb_salience_dp_workspace_bytes(fo[-1])), dtype=torch.uint8, device=dev)
    _lib.call("salience_dp_ragged", flat.data_ptr(), fo, len(zs), path.data_ptr(), ws.data_ptr(), ws.numel(), device=dev)
    return [p.cpu().numpy() for p in _lib.split(path, fo)]


def compute_f0_salience(path, device="cuda") -> np.ndarray:
    """pitch/inference.py:compute_f0_salience: the file read at 16 kHz, its salience F0 repeated and averaged
    (float64)."""
    from . import hubert_infer
    audio = hubert_infer.load_audio(path, SAMPLE_RATE)
    return f0_batch([audio], device)[0]
