"""Cutting the direct content out of raw recordings on the H100 path: the reference's
`prepare/preprocess_cdc.py:cut_direct_content` (the VCTK cleaning step: a 1024 / 256 Hann STFT, bins 0 and 1 set to
zero, the inverse STFT, written as int16), behind the C ABI (`svcb_cdc_ragged`, csrc/cdc_api.cu).  No CPU fallback: a
CUDA (sm_90a) device is required.

A clip of n samples gives 256 * (n // 256) output samples, as torch.istft without `length` does; it needs more than
512 samples, torch.stft's reflect padding.  The device evaluates the round trip in fp64, so against the reference's
float32 FFTs an output may differ by 1 LSB, on well under 0.2 % of samples (DESIGN.md §5)."""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .resample import scale_pcm

HOP = 256
PAD = 512   # torch.stft's reflect padding at each end; a clip needs more samples than this


def out_len(n: int) -> int:
    """Output samples of a clip of n: 256 * (n // 256)."""
    return HOP * (int(n) // HOP)


def load(path: str) -> Tuple[np.ndarray, int]:
    """(float32 samples, rate) of a mono .wav, decoded as torchaudio.load decodes it.  ValueError for a file with more
    than one channel (the reference would write its output transposed), of 512 samples or fewer (torch.stft's reflect
    pad fails) or with non-finite samples."""
    from scipy.io import wavfile
    rate, x = wavfile.read(path)
    if x.ndim != 1:
        raise ValueError(f"{x.shape[1]} channels; the cut takes mono audio")
    x = scale_pcm(x)
    if x.shape[0] <= PAD:
        raise ValueError(f"{x.shape[0]} samples; torch.stft's reflect padding of {PAD} needs more")
    if not np.isfinite(x).all():
        raise ValueError("non-finite samples")
    return x, int(rate)


@torch.no_grad()
def cdc_batch(clips: Sequence, device="cuda") -> List[np.ndarray]:
    """Float32 mono clips (ragged, each more than 512 samples) -> the int16 samples cut_direct_content writes for
    each, one device call; only the int16 samples are copied back."""
    dev = _lib.cuda_device(device)
    if not clips:
        return []
    flat, so = _lib.ragged(clips, dev)
    oo = _lib.offsets(out_len(so[b + 1] - so[b]) for b in range(len(so) - 1))
    out = torch.empty(max(oo[-1], 1), dtype=torch.int16, device=dev)
    _lib.call("cdc_ragged", flat.data_ptr(), so, len(clips), out.data_ptr(), device=dev)
    return _lib.split(out.cpu().numpy(), oo)
