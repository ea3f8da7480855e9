"""Trimming silence out of raw recordings on the H100 path: the reference's `prepare/preprocess_trim.py:trim_silence`
(the second VCTK cleaning step: pydub's split_on_silence with min_silence_len=200, silence_thresh=-45 and
keep_silence=200, the chunks joined and exported as wav).  The silence decision of every 200 ms window runs on the
device (`svcb_trim_silence_ragged`, csrc/trim_api.cu); pydub's rules over those flags (detect_silence's ranges,
detect_nonsilent, split_on_silence's widening and midpoints) and the slicing stay on the host, with Python work
proportional to the number of ranges.  No CPU fallback for the flags: a CUDA (sm_90a) device is required.

Positions are pydub's milliseconds: a clip of n frames at `rate` is L = round(1000 n / rate) ms long, and ms m is
frame int(m * (rate / 1000.0)).  A slice that runs past frame n is zero-filled, as pydub pads it, and the padding
counts in a window's RMS (DESIGN.md §8 lists the rules and what of them is not pinned to pydub itself)."""
from __future__ import annotations

import wave
from ctypes import c_int32
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib

WIN = 200          # min_silence_len and keep_silence, ms
MAX_RATE = 192000  # the device's bound: a 200 ms sum of squares of int16 stays below 2^53


def length_ms(n: int, rate: int) -> int:
    """len(AudioSegment) of n frames: round(1000 * (n / rate)), a tie to even."""
    return round(1000 * (int(n) / rate))


def frame(m: int, rate: int) -> int:
    """The frame at ms m: int(m * (rate / 1000.0))."""
    return int(m * (rate / 1000.0))


def windows(n: int, rate: int) -> int:
    """Window starts 0 .. L - 200 of a clip of n frames (none under 200 ms): the flags svcb_trim_silence_ragged writes."""
    return max(length_ms(n, rate) - WIN + 1, 0)


def load(path: str) -> Tuple[np.ndarray, int]:
    """(int16 samples, rate) of a 16-bit PCM mono .wav.  ValueError for any other file the stdlib `wave` reader opens
    (more than one channel, another sample width, a compressed or float format) or a rate above 192 kHz."""
    try:
        with wave.open(path, "rb") as w:
            ch, width, rate = w.getnchannels(), w.getsampwidth(), w.getframerate()
            data = w.readframes(w.getnframes())
    except (wave.Error, EOFError) as e:
        raise ValueError(f"not a PCM wav: {e}") from e
    if ch != 1:
        raise ValueError(f"{ch} channels; the trim takes mono audio")
    if width != 2:
        raise ValueError(f"{8 * width}-bit samples; the trim takes 16-bit PCM")
    if not 1 <= rate <= MAX_RATE:
        raise ValueError(f"rate {rate}; the trim takes 1..{MAX_RATE} Hz")
    return np.frombuffer(data, "<i2").astype(np.int16), int(rate)


@torch.no_grad()
def trim_batch(clips: Sequence, rates: Sequence[int], device="cuda") -> List[np.ndarray]:
    """int16 mono clips (ragged) at their rates -> each clip's silence flags (uint8, one per window start 0 .. L - 200,
    1 = silent), one device call; only the flags are copied back."""
    dev = _lib.cuda_device(device)
    if not clips:
        return []
    xs = [np.asarray(c, np.int16).reshape(-1) for c in clips]
    so = _lib.offsets(x.shape[0] for x in xs)
    flat = torch.from_numpy(np.concatenate(xs + [np.zeros(1, np.int16)])).to(dev)
    oo = _lib.offsets(windows(x.shape[0], r) for x, r in zip(xs, rates))
    out = torch.empty(max(oo[-1], 1), dtype=torch.uint8, device=dev)
    _lib.call("trim_silence_ragged", flat.data_ptr(), so, (c_int32 * len(xs))(*rates), len(xs), out.data_ptr(),
              device=dev)
    return _lib.split(out.cpu().numpy(), oo)


def silent_ranges(flags) -> List[List[int]]:
    """detect_silence's ranges from the flags: a silent start opens a new range only when it is more than 200 ms after
    the previous one (which also makes it not the next ms); each range is [first start, last start + 200]."""
    s = np.flatnonzero(flags)
    if s.size == 0:
        return []
    cut = np.flatnonzero(np.diff(s) > WIN)
    return [[int(a), int(b) + WIN] for a, b in zip(s[np.r_[0, cut + 1]], s[np.r_[cut, s.size - 1]])]


def keep_ranges(flags, L: int) -> List[List[int]]:
    """split_on_silence's chunks, [start, end) in ms: detect_nonsilent's ranges widened by 200 on both sides, an overlap
    with the next range split at the midpoint, then clipped to [0, L]."""
    silent = silent_ranges(flags)
    if not silent:
        keep = [[0, L]]
    elif silent[0] == [0, L]:
        return []
    else:
        keep, prev = [], 0
        for a, b in silent:
            keep.append([prev, a])
            prev = b
        if prev != L:
            keep.append([prev, L])
        if keep[0] == [0, 0]:
            keep.pop(0)
    keep = [[a - WIN, b + WIN] for a, b in keep]
    for cur, nxt in zip(keep, keep[1:]):
        if nxt[0] < cur[1]:
            cur[1] = nxt[0] = (cur[1] + nxt[0]) // 2
    return [[max(a, 0), min(b, L)] for a, b in keep]


def cut(x: np.ndarray, rate: int, a: int, b: int) -> np.ndarray:
    """AudioSegment[a:b] of int16 samples x: frames [frame(a), frame(b)), zero-filled past the end (pydub pads with a
    copy of a zeroed first frame, so a slice that starts past the end stays empty)."""
    fa, fb = frame(a, rate), frame(b, rate)
    seg = x[fa:fb]
    if 0 < seg.shape[0] < fb - fa:
        seg = np.concatenate([seg, np.zeros(fb - fa - seg.shape[0], np.int16)])
    return seg


def trim(x: np.ndarray, rate: int, flags) -> Optional[np.ndarray]:
    """The int16 samples trim_silence writes for clip x given its flags, or None when every window is silent (the
    reference then fails on audio_chunks[0] and writes nothing)."""
    keep = keep_ranges(flags, length_ms(x.shape[0], rate))
    if not keep:
        return None
    return np.concatenate([cut(x, rate, a, b) for a, b in keep])


def write_wav(path: str, pcm: np.ndarray, rate: int) -> None:
    """AudioSegment.export(path, format="wav") of 16-bit mono samples: the stdlib wave writer, byte for byte."""
    with open(path, "wb") as f:
        w = wave.open(f, "wb")
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(rate)
        w.setnframes(int(pcm.shape[0]))
        w.writeframesraw(np.ascontiguousarray(pcm, "<i2").tobytes())
        w.close()
