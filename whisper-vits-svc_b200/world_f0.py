"""WORLD DIO + StoneMask F0 on the H100 path: the reference's `prepare/preprocess_f0.py` (pyworld.dio at fs 16 kHz,
f0_ceil 900 and a 10 ms frame period, then pyworld.stonemask, each value rounded with Python's round(v, 1)).  The
whole algorithm runs on the device in fp64 (`svcb_world_f0_ragged`, csrc/f0_api.cu); only the rounding is on the
host.  No CPU fallback: a CUDA (sm_90a) device is required.

Audio is read as `preprocess_crepe.py` reads it: `hubert_infer.load_audio(path, 16000)`, .wav only, resampled with
`resample_poly` where the file is not at 16 kHz.  The reference uses librosa.load, which decodes more containers and
resamples with soxr, so F0 of files not at 16 kHz differs slightly from the reference's, as for the other CLIs."""
from __future__ import annotations

from typing import List, Sequence

import numpy as np
import torch

from . import _lib

SAMPLE_RATE = 16000
HOP = 160                 # 10 ms at 16 kHz
MIN_SAMPLES = 3 * HOP     # 480: shorter clips have at most 3 frames, for which WORLD's contour fix writes nothing


def frames_of(n: int) -> int:
    """pyworld.dio's frame count for n samples: int(1000 n / 16000 / 10) + 1 = n // 160 + 1."""
    return int(n) // HOP + 1


def round1(f0) -> np.ndarray:
    """float64 values as Python's round(v, 1) gives them (the exact decimal value rounded, ties to even): the
    reference rounds each value so."""
    return np.array([round(v, 1) for v in np.asarray(f0, np.float64).reshape(-1).tolist()], np.float64)


class Extractor:
    """One device and a grow-only workspace for `svcb_world_f0_ragged`.  `close()` frees the workspace."""

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
    def raw(self, clips: Sequence) -> List[torch.Tensor]:
        """Float clips at 16 kHz (each >= 1 sample) -> each one's float64 F0 on the device, before rounding."""
        if not clips:
            return []
        xs = [torch.as_tensor(np.asarray(c, np.float64).reshape(-1)) if not torch.is_tensor(c) else c.double().reshape(-1)
              for c in clips]
        so = _lib.offsets(x.numel() for x in xs)
        flat = torch.empty(so[-1], dtype=torch.float64, device=self.device)
        for b, x in enumerate(xs):
            flat[so[b]:so[b + 1]].copy_(x)
        fo = _lib.offsets(frames_of(x.numel()) for x in xs)
        out = torch.empty(fo[-1], dtype=torch.float64, device=self.device)
        need = _lib.load().svcb_world_f0_workspace_bytes(so[-1] - so[0], len(xs))
        ws = self.workspace(need)
        _lib.call("world_f0_ragged", flat.data_ptr(), so, len(xs), out.data_ptr(), ws.data_ptr(), ws.numel(),
                  device=self.device)
        return _lib.split(out, fo)

    def f0_batch(self, clips: Sequence) -> List[np.ndarray]:
        """Float clips at 16 kHz -> each one's float64 F0 as the reference saves it (rounded to 0.1)."""
        return [round1(f.cpu().numpy()) for f in self.raw(clips)]


def f0_batch(clips: Sequence, device="cuda") -> List[np.ndarray]:
    """Float clips at 16 kHz -> float64 F0 arrays of n // 160 + 1 frames, rounded as the reference rounds them; one
    device call."""
    ex = Extractor(device)
    try:
        return ex.f0_batch(clips)
    finally:
        ex.close()
