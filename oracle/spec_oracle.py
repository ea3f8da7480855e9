"""Torch-CPU restatement of the linear spectrogram of prepare/preprocess_spec.py (TEST INFRASTRUCTURE).

`spectrogram` restates vits/spectrogram.py:spectrogram_torch(y, n_fft, sr, hop, win, center=False) op for op;
`load_wav` restates vits/utils.py:load_wav_to_torch with compute_spec's scaling.  `reference_spectrogram` imports the
live function from the reference tree (with a librosa stub: the module imports librosa's mel filters at the top, which
the linear spectrogram never calls), for the tests that pin the restatement where the reference exists.

    python oracle/spec_oracle.py    writes tests/golden/spec_synth.npz: seeded synthetic clips and their spectrograms
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
SR = 32000


def spectrogram(y: torch.Tensor, n_fft: int = 1024, hop: int = 320, win: int = 1024) -> torch.Tensor:
    """y [B, n] float32 -> [B, n_fft // 2 + 1, n // hop] (spectrogram_torch with center=False, without its prints)."""
    window = torch.hann_window(win).to(dtype=y.dtype, device=y.device)
    pad = int((n_fft - hop) / 2)
    y = torch.nn.functional.pad(y.unsqueeze(1), (pad, pad), mode="reflect").squeeze(1)
    spec = torch.stft(y, n_fft, hop_length=hop, win_length=win, window=window, center=False, pad_mode="reflect",
                      normalized=False, onesided=True, return_complex=False)
    return torch.sqrt(spec.pow(2).sum(-1) + 1e-6)


def load_wav(path: str, max_wav_value: float = 32768.0):
    """(load_wav_to_torch(path)[0] / max_wav_value, sampling rate)."""
    from scipy.io.wavfile import read
    sr, data = read(path)
    return torch.FloatTensor(data.astype(np.float32)) / max_wav_value, sr


def compute_spec(path: str, max_wav_value: float = 32768.0) -> torch.Tensor:
    """compute_spec's tensor for one file: [513, n // 320]."""
    audio, _ = load_wav(path, max_wav_value)
    return spectrogram(audio.unsqueeze(0))[0]


def reference_spectrogram():
    """The live vits.spectrogram.spectrogram_torch of the reference tree."""
    from oracle import ref_import
    ref_import._ensure_path()
    ref_import._stub("librosa")
    ref_import._stub("librosa.filters")
    sys.modules["librosa"].filters = sys.modules["librosa.filters"]
    if not hasattr(sys.modules["librosa.filters"], "mel"):
        def _no_mel(*a, **k):
            raise RuntimeError("librosa is not installed; the mel spectrogram is outside the oracle's scope")
        sys.modules["librosa.filters"].mel = _no_mel
    from vits import spectrogram as rs
    return rs.spectrogram_torch


# ---------------------------------------------------------------------------------------------------- fixture
def synth_clips(seed: int = 5) -> dict:
    """Seeded synthetic clips at 32 kHz, already scaled to [-1, 1]: name -> float32 [n].  Lengths include 353 (the
    shortest the reflect padding accepts), a multiple of 320 and 320 k + 17."""
    rng = np.random.default_rng(seed)
    n = 320 * 100 + 17
    t = np.arange(n) / SR
    sweep = 0.6 * np.sin(2 * np.pi * (50.0 * t + 0.5 * (15000.0 - 50.0) / t[-1] * t * t))   # 50 Hz -> 15 kHz
    m = 320 * 40
    square = np.where(np.sin(2 * np.pi * 441.0 * np.arange(m) / SR) >= 0, 1.0, -1.0)
    return {"sweep": sweep.astype(np.float32),
            "noise": np.clip(0.3 * rng.standard_normal(320 * 30 + 17), -1, 1).astype(np.float32),
            "short": np.clip(0.5 * rng.standard_normal(353), -1, 1).astype(np.float32),
            "silence": np.zeros(320 * 20, np.float32),
            "square": square.astype(np.float32)}


def load_golden() -> dict:
    """tests/golden/spec_synth.npz as {name: (clip, spectrogram)}."""
    z = np.load(os.path.join(GOLDEN, "spec_synth.npz"))
    return {k[:-5]: (z[k], z[k[:-5] + ".spec"]) for k in z.files if k.endswith(".clip")}


def main():
    out = {}
    for name, x in synth_clips().items():
        s = spectrogram(torch.from_numpy(x)[None])[0]
        assert s.shape == (513, x.shape[0] // 320)
        out[name + ".clip"], out[name + ".spec"] = x, s.numpy()
        print(name, x.shape[0], "samples ->", tuple(s.shape), "max %.3f" % float(s.max()))
    np.savez_compressed(os.path.join(GOLDEN, "spec_synth.npz"), **out)


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    main()
