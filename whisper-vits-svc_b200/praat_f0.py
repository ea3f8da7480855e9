"""Praat's autocorrelation F0 on the H100 path: the reference's `prepare/preprocess_f0_mouth.py` and
`pitch/inference.py:compute_f0_mouth` (parselmouth's `Sound.to_pitch_ac` at a 0.01 s time step, pitch floor 30 Hz,
ceiling 1000 Hz and voicing threshold 0.5, padded with 6 zeros on each side).  The whole analysis and path finder
run on the device in fp64 (`svcb_praat_f0_ragged`, csrc/praat_f0_api.cu); only the padding is on the host.  No CPU
fallback: a CUDA (sm_90a) device is required.

Audio is read as `preprocess_f0.py` reads it: `hubert_infer.load_audio(path, 16000)`, .wav only, resampled with
`resample_poly` where the file is not at 16 kHz.  The reference uses librosa.load, which decodes more containers and
resamples with soxr, so F0 of files not at 16 kHz differs slightly from the reference's, as for the other CLIs."""
from __future__ import annotations

import math
from typing import List, Sequence

import numpy as np
import torch

from . import _lib

SAMPLE_RATE = 16000
PAD = 1024 // 160          # the reference's lpad = rpad
MIN_SAMPLES = 1600         # the 0.1 s window (3 periods of the 30 Hz floor): shorter clips have no frame


def frames_of(n: int) -> int:
    """Praat's frame count for n samples: floor((n / 16000 - 0.1) / 0.01) + 1 in double precision (about
    n // 160 - 9; on the 160-sample grid the floor sits on its edge: 1760 samples give one frame), 0 below 1600."""
    dur = int(n) * (1.0 / SAMPLE_RATE)
    if dur < 0.1:
        return 0
    return max(0, math.floor((dur - 0.1) / 0.01) + 1)


class Extractor:
    """One device and a grow-only workspace for `svcb_praat_f0_ragged`.  `close()` frees the workspace."""

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
        """Float clips at 16 kHz (each >= 1600 samples) -> each one's float64 F0 per frame on the device, unpadded."""
        if not clips:
            return []
        xs = [torch.as_tensor(np.asarray(c, np.float64).reshape(-1)) if not torch.is_tensor(c) else c.double().reshape(-1)
              for c in clips]
        so = _lib.offsets(x.numel() for x in xs)
        flat = torch.empty(so[-1], dtype=torch.float64, device=self.device)
        for b, x in enumerate(xs):
            flat[so[b]:so[b + 1]].copy_(x)
        fo = _lib.offsets(max(1, frames_of(x.numel())) for x in xs)   # too short: rejected by the call, before a launch
        out = torch.empty(fo[-1], dtype=torch.float64, device=self.device)
        need = _lib.load().svcb_praat_f0_workspace_bytes(so[-1] - so[0], len(xs))
        ws = self.workspace(need)
        _lib.call("praat_f0_ragged", flat.data_ptr(), so, len(xs), out.data_ptr(), ws.data_ptr(), ws.numel(),
                  device=self.device)
        return _lib.split(out, fo)

    def f0_batch(self, clips: Sequence) -> List[np.ndarray]:
        """Float clips at 16 kHz -> each one's float64 F0 as the reference saves it (6 zeros on each side)."""
        return [np.pad(f.cpu().numpy(), [[PAD, PAD]], mode="constant") for f in self.raw(clips)]


def f0_batch(clips: Sequence, device="cuda") -> List[np.ndarray]:
    """Float clips at 16 kHz -> padded float64 F0 arrays of frames_of(n) + 12 values; one device call."""
    ex = Extractor(device)
    try:
        return ex.f0_batch(clips)
    finally:
        ex.close()


def compute_f0_mouth(path, device="cuda") -> np.ndarray:
    """pitch/inference.py:compute_f0_mouth: the file read at 16 kHz, its padded Praat F0 (float64)."""
    from . import hubert_infer
    audio = hubert_infer.load_audio(path, SAMPLE_RATE)
    return f0_batch([audio], device)[0]
