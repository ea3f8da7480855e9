"""Restatement of prepare/preprocess_trim.py:trim_silence's pydub calls (TEST INFRASTRUCTURE).

pydub is not installed, so `AudioSegment` restates the parts of pydub 0.25.1's class the script touches for 16-bit mono
wavs: from_wav, __len__ (round(1000 * frames / rate) ms), slicing by ms (frame int(ms * (rate / 1000.0)), a slice that
runs past the end zero-filled), rms (as audioop.c computes it: the squares summed in double, over the frame count,
sqrt, truncated), `+` (append with crossfade 0: the bytes joined) and export to wav through the stdlib `wave` writer.
`split_on_silence`, `detect_nonsilent` and `detect_silence` restate pydub.silence's functions with their loops as
written: one 200 ms slice and one rms per ms.  Nothing here imports audioop, which Python 3.13 removes; the CPU suite pins
`rms` to audioop.rms where it exists.  These are restatements of pydub's rules, not pydub: DESIGN.md §8 says what that
leaves unpinned.

`reference_trim_silence` imports the unmodified reference script behind a stub `pydub` package built from this module,
for the tests that pin the written files to it where the reference tree exists.  `numpy_flags` is the same silence
decision as an int64 cumulative sum over the whole clip, the host arm of scripts/bench_trim.py.

    python oracle/trim_oracle.py    writes tests/golden/trim_synth.npz: seeded int16 clips and the oracle's flags
"""
from __future__ import annotations

import importlib.util
import itertools
import math
import os
import sys
import types
import wave

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


class TooManyMissingFrames(Exception):
    pass


def db_to_float(db, using_amplitude=True):
    db = float(db)
    return 10 ** (db / 20) if using_amplitude else 10 ** (db / 10)


class AudioSegment:
    def __init__(self, data: bytes, sample_width: int = 2, frame_rate: int = 16000, channels: int = 1):
        self._data, self.sample_width, self.frame_rate, self.channels = data, sample_width, frame_rate, channels
        self.frame_width = channels * sample_width

    @classmethod
    def from_wav(cls, path):
        with wave.open(path, "rb") as w:
            if w.getnchannels() != 1 or w.getsampwidth() != 2:
                raise ValueError("the restatement reads 16-bit mono wavs only")
            return cls(w.readframes(w.getnframes()), 2, w.getframerate(), 1)

    def _spawn(self, data):
        return AudioSegment(data, self.sample_width, self.frame_rate, self.channels)

    def frame_count(self, ms=None):
        if ms is not None:
            return ms * (self.frame_rate / 1000.0)
        return float(len(self._data) // self.frame_width)

    def __len__(self):
        return round(1000 * (self.frame_count() / self.frame_rate))

    @property
    def max_possible_amplitude(self):
        return (2 ** (self.sample_width * 8)) / 2

    def _parse_position(self, val):
        if val < 0:
            val = len(self) - abs(val)
        val = self.frame_count(ms=len(self)) if val == float("inf") else self.frame_count(ms=val)
        return int(val)

    def __getitem__(self, millisecond):
        if isinstance(millisecond, slice):
            start = millisecond.start if millisecond.start is not None else 0
            end = millisecond.stop if millisecond.stop is not None else len(self)
            start = min(start, len(self))
            end = min(end, len(self))
        else:
            start, end = millisecond, millisecond + 1
        start = self._parse_position(start) * self.frame_width
        end = self._parse_position(end) * self.frame_width
        data = self._data[start:end]
        missing_frames = (end - start - len(data)) // self.frame_width
        if missing_frames:
            if missing_frames > self.frame_count(ms=2):
                raise TooManyMissingFrames(f"You should never be filling in more than 2 ms with silence here, "
                                           f"missing frames: {missing_frames}")
            data += bytes(len(data[:self.frame_width])) * missing_frames   # audioop.mul(first frame, 0)
        return self._spawn(data)

    @property
    def rms(self):
        """audioop.rms(self._data, 2): the squares summed in a double, over the frame count, sqrt, truncated to an
        unsigned int.  Every partial sum is an integer below 2^53 (asserted), so the sum is exact in any order and
        numpy's equals audioop's sequential one."""
        if not self._data:
            return 0
        x = np.frombuffer(self._data, "<i2").astype(np.float64)
        s = float(np.dot(x, x))
        assert s < 2.0 ** 53
        return int(math.sqrt(s / float(x.shape[0])))

    def __add__(self, arg):
        return self._spawn(self._data + arg._data)

    def export(self, out_f, format="wav"):
        assert format == "wav"
        with open(out_f, "wb") as f:
            w = wave.open(f, "wb")
            w.setnchannels(self.channels)
            w.setsampwidth(self.sample_width)
            w.setframerate(self.frame_rate)
            w.setnframes(int(self.frame_count()))
            w.writeframesraw(self._data)
            w.close()
        return out_f


def detect_silence(audio_segment, min_silence_len=1000, silence_thresh=-16, seek_step=1):
    seg_len = len(audio_segment)
    if seg_len < min_silence_len:
        return []
    silence_thresh = db_to_float(silence_thresh) * audio_segment.max_possible_amplitude
    silence_starts = []
    last_slice_start = seg_len - min_silence_len
    slice_starts = range(0, last_slice_start + 1, seek_step)
    if last_slice_start % seek_step:
        slice_starts = itertools.chain(slice_starts, [last_slice_start])
    for i in slice_starts:
        if audio_segment[i:i + min_silence_len].rms <= silence_thresh:
            silence_starts.append(i)
    if not silence_starts:
        return []
    silent_ranges = []
    prev_i = silence_starts.pop(0)
    current_range_start = prev_i
    for silence_start_i in silence_starts:
        continuous = silence_start_i == prev_i + seek_step
        silence_has_gap = silence_start_i > prev_i + min_silence_len
        if not continuous and silence_has_gap:
            silent_ranges.append([current_range_start, prev_i + min_silence_len])
            current_range_start = silence_start_i
        prev_i = silence_start_i
    silent_ranges.append([current_range_start, prev_i + min_silence_len])
    return silent_ranges


def detect_nonsilent(audio_segment, min_silence_len=1000, silence_thresh=-16, seek_step=1):
    silent_ranges = detect_silence(audio_segment, min_silence_len, silence_thresh, seek_step)
    len_seg = len(audio_segment)
    if not silent_ranges:
        return [[0, len_seg]]
    if silent_ranges[0][0] == 0 and silent_ranges[0][1] == len_seg:
        return []
    prev_end_i = 0
    nonsilent_ranges = []
    for start_i, end_i in silent_ranges:
        nonsilent_ranges.append([prev_end_i, start_i])
        prev_end_i = end_i
    if end_i != len_seg:
        nonsilent_ranges.append([prev_end_i, len_seg])
    if nonsilent_ranges[0] == [0, 0]:
        nonsilent_ranges.pop(0)
    return nonsilent_ranges


def split_on_silence(audio_segment, min_silence_len=1000, silence_thresh=-16, keep_silence=100, seek_step=1):
    if isinstance(keep_silence, bool):
        keep_silence = len(audio_segment) if keep_silence else 0
    output_ranges = [[start - keep_silence, end + keep_silence]
                     for start, end in detect_nonsilent(audio_segment, min_silence_len, silence_thresh, seek_step)]
    a, b = itertools.tee(output_ranges)
    next(b, None)
    for range_i, range_ii in zip(a, b):
        last_end, next_start = range_i[1], range_ii[0]
        if next_start < last_end:
            range_i[1] = (last_end + next_start) // 2
            range_ii[0] = range_i[1]
    return [audio_segment[max(start, 0):min(end, len(audio_segment))] for start, end in output_ranges]


# ---------------------------------------------------------------------------------------------------- the script
def trim_chunks(x: np.ndarray, rate: int):
    """split_on_silence as trim_silence calls it, on int16 samples: the chunks (AudioSegments)."""
    seg = AudioSegment(np.ascontiguousarray(x, "<i2").tobytes(), 2, int(rate), 1)
    return split_on_silence(seg, min_silence_len=200, silence_thresh=-45, keep_silence=200)


def trim(x: np.ndarray, rate: int):
    """The int16 samples trim_silence writes for x, or None when it writes nothing (no chunks)."""
    chunks = trim_chunks(x, rate)
    if not chunks:
        return None
    out = chunks[0]
    for c in chunks[1:]:
        out += c
    return np.frombuffer(out._data, "<i2").copy()


def trim_silence(src, dst) -> bool:
    """trim_silence's body on this module's AudioSegment: read, split, join, export.  False, with nothing written, when
    there is no chunk (where the reference's audio_chunks[0] raises)."""
    chunks = split_on_silence(AudioSegment.from_wav(src), min_silence_len=200, silence_thresh=-45, keep_silence=200)
    if not chunks:
        return False
    out = chunks[0]
    for c in chunks[1:]:
        out += c
    out.export(dst, format="wav")
    return True


def window_flags(x: np.ndarray, rate: int) -> np.ndarray:
    """detect_silence's decision for every window start 0 .. L - 200, by its loop (one slice and one rms per ms)."""
    seg = AudioSegment(np.ascontiguousarray(x, "<i2").tobytes(), 2, int(rate), 1)
    thresh = db_to_float(-45) * seg.max_possible_amplitude
    return np.array([seg[i:i + 200].rms <= thresh for i in range(len(seg) - 199)], np.uint8)


def numpy_flags(x: np.ndarray, rate: int) -> np.ndarray:
    """window_flags as one int64 cumulative sum of squares over the clip: the window's frames [fs(i), fs(i + 200)),
    those past n zero, S / N and sqrt in fp64 (exact S, correctly rounded steps), truncated and compared."""
    n = x.shape[0]
    L = round(1000 * (n / rate))
    if L < 200:
        return np.zeros(0, np.uint8)
    q = np.concatenate([[0], np.cumsum(x.astype(np.int64) ** 2)])
    fs = (np.arange(L + 1, dtype=np.float64) * (rate / 1000.0)).astype(np.int64)
    i = np.arange(L - 199)
    S = q[np.minimum(fs[i + 200], n)] - q[np.minimum(fs[i], n)]
    N = fs[i + 200] - fs[i]
    with np.errstate(invalid="ignore", divide="ignore"):
        rms = np.where(N > 0, np.floor(np.sqrt(S.astype(np.float64) / N)), 0.0)
    return (rms <= db_to_float(-45) * 32768.0).astype(np.uint8)


def reference_trim_silence():
    """The live trim_silence of the reference's prepare/preprocess_trim.py behind a stub `pydub` package (pydub,
    pydub.silence, pydub.effects) built from this module.  The stub is in sys.modules only while the script is
    imported, and the script is loaded from its file, so sys.path is left as it is."""
    from oracle import ref_import
    if not ref_import.available():
        raise RuntimeError(f"reference tree not found at {ref_import.REF_ROOT}")
    pkg, silence, effects = (types.ModuleType(n) for n in ("pydub", "pydub.silence", "pydub.effects"))
    pkg.AudioSegment = AudioSegment
    silence.split_on_silence, silence.detect_nonsilent, silence.detect_silence = (split_on_silence, detect_nonsilent,
                                                                                  detect_silence)
    pkg.silence, pkg.effects = silence, effects
    names = ("pydub", "pydub.silence", "pydub.effects")
    saved = {k: sys.modules.get(k) for k in names}
    sys.modules.update(zip(names, (pkg, silence, effects)))
    try:
        spec = importlib.util.spec_from_file_location("ref_preprocess_trim",
                                                      os.path.join(ref_import.REF_ROOT, "prepare", "preprocess_trim.py"))
        m = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(m)
    finally:
        for k, v in saved.items():
            if v is None:
                del sys.modules[k]
            else:
                sys.modules[k] = v
    return m.trim_silence


# ---------------------------------------------------------------------------------------------------- fixture
def burst(rng, rate, ms, amp):
    """A speech-like burst: a few harmonics of a gliding pitch plus noise, under a 20 ms raised-cosine attack and
    release."""
    n = int(rate * ms / 1000)
    t = np.arange(n) / rate
    f0 = rng.uniform(100, 300)
    ph = 2 * np.pi * f0 * (t + 0.5 * rng.uniform(-0.2, 0.2) * t * t)
    x = sum(rng.uniform(0.2, 1.0) / k * np.sin(k * ph + rng.uniform(0, 2 * np.pi)) for k in (1, 2, 3, 5))
    x = x + 0.2 * rng.standard_normal(n)
    r = min(n // 2, int(0.02 * rate))
    env = np.ones(n)
    if r > 0:
        ramp = 0.5 - 0.5 * np.cos(np.pi * np.arange(r) / r)
        env[:r], env[n - r:] = ramp, ramp[::-1]
    return amp * x * env / max(np.abs(x).max(), 1e-9)


def quiet(rng, rate, ms, level):
    """Room noise of RMS about `level`."""
    return level * rng.standard_normal(int(rate * ms / 1000))


def square(rate, ms, mag):
    """A constant-magnitude stretch: +-mag alternating, RMS exactly mag over any whole number of its frames."""
    n = int(rate * ms / 1000)
    return mag * np.where(np.arange(n) % 2 == 0, 1.0, -1.0)


def compose(rng, rate, parts, n=None):
    """Join parts ('b', ms, amp) burst / ('q', ms, level) noise / ('s', ms, mag) square / ('z', ms) zeros into int16,
    cut or zero-extended to n frames when n is given."""
    xs = []
    for p in parts:
        if p[0] == "b":
            xs.append(burst(rng, rate, p[1], p[2]))
        elif p[0] == "q":
            xs.append(quiet(rng, rate, p[1], p[2]))
        elif p[0] == "s":
            xs.append(square(rate, p[1], p[2]))
        else:
            xs.append(np.zeros(int(rate * p[1] / 1000)))
    x = np.concatenate(xs)
    if n is not None:
        x = np.concatenate([x, np.zeros(max(0, n - x.shape[0]))])[:n]
    return np.clip(np.rint(x), -32768, 32767).astype(np.int16)


def synth_clips(seed: int = 11) -> dict:
    """Seeded int16 clips: name -> (rate, int16 [n]).
      gaps48k      leading and trailing silence; bursts apart by 150 ms (< 200: one range), 300 ms (200-400: the
                   widened ranges overlap, split at the midpoint) and 700 ms (> 400: two chunks with a gap)
      level48k     constant-magnitude stretches at RMS exactly 184 (silent: thresh = 184.27) and 185 (not) between
                   zeros and bursts; noise near the threshold
      pad44k       ends inside a burst at n = 132,323 (L = 3001 ms, frame(L) = 132,344): the last window and the last
                   chunk run 21 frames past the end and are zero-filled
      tail44k      44.1 kHz with long trailing noise, 100 ms bursts and 250 ms gaps
      level22k     the 184 / 185 stretches and bursts at 22.05 kHz
      tie16k_down  n = 16,008: 1000.5 ms, rounded to 1000 (ties to even)
      tie16k_up    n = 16,024: 1001.5 ms, rounded to 1002 (frame(1002) = 16,032: padded)
      silent16k    every window silent: no chunk, nothing written
      short16k     n = 2,590: 161.875 ms -> L = 162, under 200 ms: written whole, padded to 2,592 frames
      short48k     n = 7,000: L = 146, padded to 7,008"""
    rng = np.random.default_rng(seed)
    c = {}
    c["gaps48k"] = (48000, compose(rng, 48000, [("q", 300, 25), ("b", 400, 6000), ("q", 150, 30), ("b", 300, 4000),
                                                ("q", 300, 20), ("b", 250, 8000), ("q", 700, 35), ("b", 350, 5000),
                                                ("q", 500, 15)]))
    c["level48k"] = (48000, compose(rng, 48000, [("z", 300), ("s", 500, 184), ("z", 300), ("s", 500, 185), ("z", 250),
                                                 ("b", 200, 3000), ("s", 450, 185), ("q", 400, 120), ("s", 600, 184),
                                                 ("b", 150, 2500), ("z", 210)]))
    c["pad44k"] = (44100, compose(rng, 44100, [("q", 500, 40), ("b", 900, 7000), ("q", 350, 30), ("b", 1400, 6000)],
                                  n=132323))
    c["tail44k"] = (44100, compose(rng, 44100, [("b", 100, 9000), ("q", 250, 50), ("b", 100, 9000), ("q", 250, 50),
                                                ("b", 120, 3000), ("q", 900, 60)]))
    c["level22k"] = (22050, compose(rng, 22050, [("s", 400, 185), ("z", 220), ("s", 400, 184), ("b", 300, 5000),
                                                  ("q", 450, 100), ("s", 300, 185)]))
    c["tie16k_down"] = (16000, compose(rng, 16000, [("q", 200, 20), ("b", 500, 5000), ("q", 250, 20)], n=16008))
    c["tie16k_up"] = (16000, compose(rng, 16000, [("q", 210, 20), ("b", 450, 5000)], n=16024))
    c["silent16k"] = (16000, compose(rng, 16000, [("q", 1500, 40)]))
    c["short16k"] = (16000, compose(rng, 16000, [("b", 200, 3000)], n=2590))
    c["short48k"] = (48000, compose(rng, 48000, [("q", 150, 10)], n=7000))
    return c


def load_golden() -> dict:
    """tests/golden/trim_synth.npz as {name: (rate, int16 clip, uint8 flags)}."""
    z = np.load(os.path.join(GOLDEN, "trim_synth.npz"))
    return {k[:-5]: (int(z[k[:-5] + ".rate"]), z[k], z[k[:-5] + ".flags"]) for k in z.files if k.endswith(".clip")}


def main():
    out = {}
    for name, (sr, x) in synth_clips().items():
        f = window_flags(x, sr)
        y = trim(x, sr)
        out[name + ".clip"], out[name + ".rate"], out[name + ".flags"] = x, np.int64(sr), f
        print(name, sr, x.shape[0], "frames,", f.size, "windows,", int(f.sum()), "silent ->",
              "nothing" if y is None else f"{y.shape[0]} frames")
    np.savez_compressed(os.path.join(GOLDEN, "trim_synth.npz"), **out)


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    main()
