"""Linear spectrograms of the training data on the H100 path: the reference's `vits/utils.py:load_wav_to_torch` with
the scaling of `prepare/preprocess_spec.py:compute_spec`, and `vits/spectrogram.py:spectrogram_torch` as that script
calls it (center=False), behind the C ABI (`svcb_linear_spec_ragged`, csrc/spec_api.cu).  No CPU fallback: a CUDA
(sm_90a) device is required.

The device path implements n_fft 1024, hop 320 and win 1024 (configs/base.yaml); a config with other values is
rejected.  A clip of n samples gives n // 320 frames; it needs more than 352 samples, the reflect padding."""
from __future__ import annotations

from typing import List, Sequence

import numpy as np
import torch

from . import _lib

N_FFT = 1024
HOP = 320
WIN = 1024
BINS = N_FFT // 2 + 1
PAD = (N_FFT - HOP) // 2   # reflect padding at each end; a clip needs more samples than this


def check_hparams(hp) -> None:
    """ValueError unless hp.data has the STFT geometry the device path implements."""
    d = hp.data
    got = (int(d.filter_length), int(d.hop_length), int(d.win_length))
    if got != (N_FFT, HOP, WIN):
        raise ValueError(f"unsupported spectrogram config: filter_length, hop_length, win_length = {got}; the device path "
                         f"implements {(N_FFT, HOP, WIN)}")


def frames(n_samples: int) -> int:
    """Frames of a clip of n_samples: (n + 2 * 352 - 1024) // 320 + 1 = n // 320."""
    return int(n_samples) // HOP


def load_wav(path: str, hp) -> np.ndarray:
    """load_wav_to_torch(path) / hp.data.max_wav_value, as float32 [n].  Rejects a file not at hp.data.sampling_rate
    (the reference asserts), a multi-channel file and a file of 352 samples or fewer (torch's reflect pad fails)."""
    from scipy.io.wavfile import read
    sr, data = read(path)
    if sr != hp.data.sampling_rate:
        raise ValueError(f"{sr} is not {hp.data.sampling_rate}")
    if data.ndim != 1:
        raise ValueError(f"{data.shape[1]} channels; the spectrogram takes mono audio")
    if data.shape[0] <= PAD:
        raise ValueError(f"{data.shape[0]} samples; the reflect padding needs more than {PAD}")
    return torch.from_numpy(data.astype(np.float32)).div(hp.data.max_wav_value).numpy()


def _range_notice(x: torch.Tensor) -> None:
    """spectrogram_torch's prints when the audio leaves [-1, 1]."""
    if torch.min(x) < -1.0:
        print("min value is ", torch.min(x))
    if torch.max(x) > 1.0:
        print("max value is ", torch.max(x))


@torch.no_grad()
def spec_batch(audios: Sequence, hp, device="cuda") -> List[torch.Tensor]:
    """Scaled clips (ragged) -> [513, n_b // 320] CPU float32 spectrograms, one device call.  The results are views of
    one buffer: clone one before keeping it apart from the others (torch.save of a view writes the whole buffer)."""
    check_hparams(hp)
    dev = _lib.cuda_device(device)
    clips = [torch.as_tensor(np.asarray(a, np.float32)).reshape(-1) for a in audios]
    if not clips:
        return []
    for x in clips:
        _range_notice(x)
    flat, so = _lib.ragged(clips, dev)
    fo = _lib.offsets(BINS * frames(x.numel()) for x in clips)
    out = torch.empty(max(fo[-1], 1), dtype=torch.float32, device=dev)
    _lib.call("linear_spec_ragged", flat.data_ptr(), so, len(clips), out.data_ptr(), None, 0, device=dev)
    return [s.view(BINS, s.numel() // BINS) for s in _lib.split(out.cpu(), fo)]
