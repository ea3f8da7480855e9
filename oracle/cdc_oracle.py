"""Torch-CPU restatement of prepare/preprocess_cdc.py:cut_direct_content (TEST INFRASTRUCTURE).

`decode` reads a .wav as torchaudio.load does (float32 [channels, n]: integer PCM divided by 2^(bits - 1), 8-bit as
(x - 128) / 128, float PCM as stored); `cdc` restates the function's steps 2-5 with the same torch calls: the 1024 / 256
Hann STFT, bins 0 and 1 set to zero, the inverse STFT, x 32768, clamp and `.short()`.  `reference_cut_direct_content`
imports the unmodified reference script behind a stub `torchaudio` whose `load` is `decode`, for the tests that pin
`cdc` and the written files to the reference where its tree exists.

    python oracle/cdc_oracle.py    writes tests/golden/cdc_synth.npz: seeded int16 clips and the oracle's outputs
"""
from __future__ import annotations

import importlib.util
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
MAX_WAV_VALUE = 32768.0


def decode(path: str):
    """torchaudio.load(path): (float32 tensor [channels, n], rate)."""
    from scipy.io import wavfile
    rate, x = wavfile.read(path)
    if x.dtype == np.uint8:
        x = (x.astype(np.float32) - 128.0) / 128.0
    elif x.dtype.kind in "iu":
        x = x.astype(np.float32) / float(np.iinfo(x.dtype).max + 1)
    x = torch.from_numpy(np.ascontiguousarray(x.astype(np.float32)))
    return (x.T.contiguous() if x.ndim > 1 else x[None]), int(rate)


def cdc(source) -> np.ndarray:
    """prepare/preprocess_cdc.py:18-26 for float32 source [channels, n] (or [n]): the int16 samples it writes."""
    source = torch.as_tensor(source, dtype=torch.float32)
    if source.ndim == 1:
        source = source[None]
    stft = torch.stft(source, 1024, 256, 1024, torch.hann_window(1024), return_complex=True)
    stft[:, 0, :] = 0
    stft[:, 1, :] = 0
    istft = torch.istft(stft, 1024, 256, 1024, torch.hann_window(1024))
    audio = istft.squeeze()
    audio = MAX_WAV_VALUE * audio
    audio = audio.clamp(min=-MAX_WAV_VALUE, max=MAX_WAV_VALUE - 1)
    audio = audio.short()
    return audio.data.cpu().detach().numpy()


def reference_cut_direct_content():
    """The live cut_direct_content of the reference's prepare/preprocess_cdc.py, its torchaudio replaced by a stub whose
    `load` is `decode`.  The stub is in sys.modules only while the script is imported, so an installed torchaudio is
    neither used nor changed.  The script is loaded from its file and imports nothing from the reference tree, so
    sys.path is left as it is (other suites depend on where the reference root sits in it)."""
    from oracle import ref_import
    if not ref_import.available():
        raise RuntimeError(f"reference tree not found at {ref_import.REF_ROOT}")
    stub = types.ModuleType("torchaudio")
    stub.load = decode
    saved = sys.modules.get("torchaudio")
    sys.modules["torchaudio"] = stub
    try:
        try:
            import tqdm  # noqa: F401  (the script imports it at the top; cut_direct_content does not use it)
        except ImportError:
            ref_import._stub("tqdm")
            sys.modules["tqdm"].tqdm = lambda it, **kw: it
        spec = importlib.util.spec_from_file_location("ref_preprocess_cdc",
                                                      os.path.join(ref_import.REF_ROOT, "prepare", "preprocess_cdc.py"))
        m = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(m)
    finally:
        if saved is None:
            del sys.modules["torchaudio"]
        else:
            sys.modules["torchaudio"] = saved
    return m.cut_direct_content


# ---------------------------------------------------------------------------------------------------- fixture
def synth_clips(seed: int = 7) -> dict:
    """Seeded int16 clips: name -> (rate, int16 [n]).  Harmonics, a DC offset, 30-50 Hz hum and noise, at lengths 513
    (the shortest the reflect padding accepts), 767 (255 mod 256), 1024 (0 mod 256), 48,000 and 3 x 48,000 + 129 at
    48 kHz, one clip at 22,050 Hz and one at 16 kHz; and a near-full-scale square-ish clip whose cut overshoots both
    int16 rails, so the clamp is hit at 32767 and -32768."""
    rng = np.random.default_rng(seed)

    def voice(sr, n, f0, dc, hum_hz):
        t = np.arange(n) / sr
        x = sum(0.3 / k * np.sin(2 * np.pi * k * f0 * t + rng.uniform(0, 2 * np.pi)) for k in (1, 2, 3, 4, 6))
        x = x + dc + 0.12 * np.sin(2 * np.pi * hum_hz * t + 0.3) + 0.02 * rng.standard_normal(n)
        return (np.clip(x, -1, 1) * 32767).astype(np.int16)

    clips = {}
    for i, n in enumerate((513, 767, 1024, 48000, 3 * 48000 + 129)):
        clips[f"v48k_{n}"] = (48000, voice(48000, n, 110.0 + 37 * i, 0.04 - 0.02 * i, 30.0 + 5 * i))
    clips["v22k_11102"] = (22050, voice(22050, 11102, 180.0, 0.06, 50.0))
    clips["v16k_8200"] = (16000, voice(16000, 8200, 140.0, -0.05, 35.0))
    # a 200 Hz pulse train high 90 % of each period, then 10 %: the cut moves each half's mean (about +-0.79) to 0,
    # so the short pulses land near -+1.77
    n = 9031
    t = np.arange(n)
    high = (t * 200 / 48000) % 1 < np.where(t < n // 2, 0.9, 0.1)
    sq = np.where(high, 0.985, -0.985) + 0.01 * rng.standard_normal(n)
    clips["square48k_9031"] = (48000, (np.clip(sq, -1, 1) * 32767).astype(np.int16))
    return clips


def load_golden() -> dict:
    """tests/golden/cdc_synth.npz as {name: (rate, int16 clip, int16 oracle output)}."""
    z = np.load(os.path.join(GOLDEN, "cdc_synth.npz"))
    return {k[:-5]: (int(z[k[:-5] + ".rate"]), z[k], z[k[:-5] + ".out"]) for k in z.files if k.endswith(".clip")}


def main():
    out = {}
    for name, (sr, x) in synth_clips().items():
        y = cdc(torch.from_numpy(x.astype(np.float32) / np.float32(MAX_WAV_VALUE)))
        assert y.shape == (256 * (x.shape[0] // 256),) and y.dtype == np.int16
        out[name + ".clip"], out[name + ".rate"], out[name + ".out"] = x, np.int64(sr), y
        print(name, sr, x.shape[0], "samples ->", y.shape[0], "rails hit:", int((y == 32767).sum()),
              int((y == -32768).sum()))
    np.savez_compressed(os.path.join(GOLDEN, "cdc_synth.npz"), **out)


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    main()
