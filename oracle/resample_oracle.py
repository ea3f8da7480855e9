"""CPU restatement of prepare/preprocess_a.py:resample_wave (TEST INFRASTRUCTURE).

`decode` reads a .wav as librosa does (integer PCM scaled to [-1, 1), channels averaged); `resample` is scipy's
`resample_poly` in float64, cast to float32 (the identity when the rates are equal); `pcm16` is the reference's float32
normalisation, step for step in numpy.  `reference_resample_wave` imports the unmodified reference script behind a
stub `librosa` whose `load(path, sr)` answers with `decode` and `resample`, for the tests that pin `pcm16` and the
written files to the reference where its tree exists.
"""
from __future__ import annotations

import importlib.util
import math
import os
import sys

import numpy as np


def decode(path: str):
    """(rate, float32 mono)."""
    from scipy.io import wavfile
    rate, x = wavfile.read(path)
    if x.dtype == np.uint8:
        x = (x.astype(np.float32) - 128.0) / 128.0
    elif x.dtype.kind in "iu":
        x = x.astype(np.float32) / float(np.iinfo(x.dtype).max + 1)
    x = x.astype(np.float32)
    return int(rate), (x.mean(axis=1) if x.ndim > 1 else x)


def resample(x: np.ndarray, sr_in: int, sr_out: int) -> np.ndarray:
    """resample_poly(x in float64, sr_out / sr_in reduced) as float32; x itself when the rates are equal."""
    from scipy.signal import resample_poly
    x = np.asarray(x, np.float32)
    if sr_in == sr_out:
        return x.copy()
    g = math.gcd(sr_in, sr_out)
    return resample_poly(x.astype(np.float64), sr_out // g, sr_in // g).astype(np.float32)


def pcm16(wav: np.ndarray) -> np.ndarray:
    """prepare/preprocess_a.py:12-14 without the write."""
    wav = wav / np.abs(wav).max() * 0.6
    wav = wav / max(0.01, np.max(np.abs(wav))) * 32767 * 0.6
    return wav.astype(np.int16)


def load(path: str, sr: int) -> np.ndarray:
    """librosa.load(path, sr=sr)[0] as the oracle states it."""
    rate, x = decode(path)
    return resample(x, rate, sr)


def reference_resample_wave():
    """The live resample_wave of the reference's prepare/preprocess_a.py, its librosa replaced by this oracle."""
    from oracle import ref_import
    ref_import._ensure_path()
    ref_import._stub("librosa")
    sys.modules["librosa"].load = lambda path, sr=22050, **kw: (load(path, sr), sr)
    try:
        import tqdm  # noqa: F401  (the script imports it at the top; resample_wave does not use it)
    except ImportError:
        ref_import._stub("tqdm")
        sys.modules["tqdm"].tqdm = lambda it, **kw: it
    spec = importlib.util.spec_from_file_location("ref_preprocess_a",
                                                  os.path.join(ref_import.REF_ROOT, "prepare", "preprocess_a.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m.resample_wave
