"""Restatement of prepare/preprocess_f0_mouth.py's parselmouth call in numpy fp64 (TEST INFRASTRUCTURE).

`praat_f0(x)` restates Praat's `Sound: To Pitch (ac)...` at the reference's arguments (time step 0.01 s, pitch floor
30 Hz, ceiling 1000 Hz, voicing threshold 0.5; the rest at Praat's defaults: 15 candidates, `very accurate` off, i.e. a
Hanning window of 3 periods, silence threshold 0.03, octave cost 0.01, octave-jump cost 0.35, voiced/unvoiced cost
0.14) followed by the reference's `np.pad(f0, [[6, 6]])`.  It was written from Boersma (1993), "Accurate short-term
analysis of the fundamental frequency and the harmonics-to-noise ratio of a sampled sound", IFA Proceedings 17, and
from the Praat manual's pages on `Sound: To Pitch (ac)...`; Praat's own code was not consulted.  The steps:

- Frames.  The window lasts 3 / 30 = 0.1 s, W = 1600 samples (the largest even count within it).  With dx = 1.0 / 16000
  and duration = n * dx, there are F = floor((duration - 0.1) / 0.01) + 1 frames, evaluated in that order in double
  precision; duration < 0.1 (n < 1600) or F < 1 is an error, as parselmouth raises one.  Lengths on the 160-sample
  grid sit on the floor's edge: 1760 samples give (0.11 - 0.1) / 0.01 = 0.9999999999999994, so one frame, not two.
  The frames are centred on the signal: t0 = (0.5 * duration - (0.5 * F) * 0.01) + 0.5 * 0.01 and t_i = t0 + i * 0.01,
  each operation rounded once in that order.  Sample k sits at (k + 0.5) dx; frame i's sample `left` is
  floor((t_i - 0.5 dx) / dx), the last sample at or before t_i, and its window holds samples left - 799 .. left + 800.
- Global peak: max |x - mean(x)| over the file.  All-zero audio gives all-unvoiced frames.
- Each frame: the local mean over one longest period on each side, P = floor(16000 / 30) = 533 samples, i.e. samples
  left - 532 .. left + 533; the local peak max |x - local mean| over the window; a[j] = (x - local mean) * w[j] with the
  Hanning window w[j] = 0.5 - 0.5 cos(2 pi (j + 1) / (W + 1)), j = 0 .. W - 1 (no zero end points); the
  autocorrelation r_a(k) = sum_j a[j] a[j + k] and the window's r_w(k) alike, and Boersma eq. (9):
  r(k) = (r_a(k) / r_a(0)) / (r_w(k) / r_w(0)).  A frame with r_a(0) = 0 has no voiced candidate.
  `frame_r` computes r by the direct sum (the form the device uses) or, with fft=True, through an FFT zero-padded to
  4096 >= 1.5 W points, as Praat does; 4096 exceeds W + the largest lag read, so no wrap-around reaches those lags.
- Lags: MIN_LAG = max(2, floor(16000 / 1000)) = 16 to MAX_LAG = floor(W / 3) + 2 = 535.
- Candidates.  Every lag k in [MIN_LAG, MAX_LAG] with r(k) > 0.5 * voicing threshold, r(k) > r(k - 1) and
  r(k) >= r(k + 1) is a local maximum.  It is refined first by the parabola through r(k - 1), r(k), r(k + 1), then by
  maximising the sinc interpolant of Boersma eq. (22) over the lags:
      r(t) = sum_{q = -D + 1}^{D} r(m + q) g(t - m - q),  m = floor(t),  g(d) = sinc(pi d) (0.5 + 0.5 cos(pi d / (D + 0.5)))
  with interpolation depth D = 70 (the depth Praat's manual gives for its sinc interpolation) and r(-k) = r(k).  The
  maximum is found by Newton's method on r'(t) = 0 with analytic derivatives, from the parabolic vertex, for at most 8
  steps: a step stops the search, without being taken, when r''(t) >= 0 or it would leave [k - 1, k + 1]; a step
  smaller than 1e-10 lags is the last one.  (Boersma maximises the same interpolant; the search method is not in the
  paper.  Newton's fixed point is insensitive to the summation order, which keeps the device within rounding.)
  The lags read are 0 .. MAX_LAG + D + 1 = 606.  A candidate at lag t (in samples) has the frequency 16000 / t and the
  strength r(t) - octave_cost * log2(floor * t / 16000); the interpolated r(t) is not capped at 1 and the frequency not
  capped at the ceiling (the refined lag may sit just below 16).
- At most 14 voiced candidates are kept: those of the 14 largest strengths, a tie going to the smaller lag, and they
  are kept in ascending lag order after the unvoiced candidate (index 0).  The unvoiced candidate's strength is
  voicing + max(0, 2 - (local peak / global peak) / (silence / (1 + voicing))), with local peak / global peak taken
  as 0 when the global peak is 0.
- Path finder (Viterbi).  delta_0(c) = strength_0(c); delta_i(c) = (max_p delta_{i-1}(p) - cost(p, c)) + strength_i(c),
  with cost 0 between two unvoiced candidates, voiced_unvoiced_cost when exactly one is voiced, and
  octave_jump_cost * |log2(f_p / f_c)| between two voiced ones, each times Praat's time-step correction 0.01 / dt
  (= 1 here).  A tie in a maximum (predecessor or last frame) goes to the lowest candidate index; the best path is
  traced back from the last frame.
- Output: the chosen candidate's frequency per frame, 0 if unvoiced, padded with 6 zeros on each side
  (lpad = rpad = 1024 // 160), float64, not rounded.

praat-parselmouth is not installed where this was written, so this restatement is not pinned to Praat there:
tests/test_praat_f0_cpu.py::test_pin_to_parselmouth pins it wherever parselmouth imports, and checks it against the
true F0 of synthetic tones everywhere (DESIGN.md §8).

    python oracle/praat_f0_oracle.py    writes tests/golden/praat_f0_synth.npz: seeded clips and the oracle's F0
"""
from __future__ import annotations

import math
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "praat_f0_synth.npz")

FS = 16000
DX = 1.0 / FS
DT = 160 / FS                      # time_step = 160 / sr, as the reference passes it
FLOOR = 30.0
CEILING = 1000.0
PERIODS = 3.0
MAX_CANDIDATES = 15
SILENCE = 0.03
VOICING = 0.5
OCTAVE_COST = 0.01
OCTAVE_JUMP_COST = 0.35
VUV_COST = 0.14
PAD = 1024 // 160                  # 6
WIN_DUR = PERIODS / FLOOR          # 0.1 s
W = 2 * (int(WIN_DUR * FS) // 2)   # 1600
HALF = W // 2
P = int(FS / FLOOR)                # 533: one longest period in samples
MIN_LAG = max(2, int(FS / CEILING))   # 16
MAX_LAG = W // 3 + 2               # 535
DEPTH = 70                         # sinc interpolation depth
NLAG = MAX_LAG + DEPTH + 2         # lags 0 .. 606 are read
NFFT = 4096
TSC = 0.01 / DT                    # time-step correction, 1.0
NEWTON_STEPS = 8


def n_frames(n: int) -> int:
    """Frames of n samples: floor((n dx - 0.1) / 0.01) + 1; 0 where Praat raises (n dx < 0.1)."""
    dur = n * DX
    if dur < WIN_DUR:
        return 0
    return max(0, math.floor((dur - WIN_DUR) / DT) + 1)


MIN_SAMPLES = next(n for n in range(1, 4 * W) if n_frames(n) >= 1)   # 1600


def frame_lefts(n: int) -> np.ndarray:
    """Sample `left` (the last sample at or before the frame centre) of each frame."""
    F = n_frames(n)
    if F < 1:
        raise ValueError(f"{n} samples: shorter than the 0.1 s window (at least {MIN_SAMPLES} samples)")
    dur = n * DX
    t0 = (0.5 * dur - (0.5 * F) * DT) + 0.5 * DT
    lefts = np.array([math.floor(((t0 + i * DT) - 0.5 * DX) / DX) for i in range(F)], np.int64)
    assert lefts[0] - HALF + 1 >= 0 and lefts[-1] + HALF < n, (n, lefts[0], lefts[-1])
    return lefts


def hanning() -> np.ndarray:
    j = np.arange(W, dtype=np.float64)
    return 0.5 - 0.5 * np.cos(2.0 * np.pi * (j + 1.0) / (W + 1.0))


def _direct_ac(a: np.ndarray) -> np.ndarray:
    """sum_j a[..., j] a[..., j + k] for k = 0 .. NLAG - 1, over the last axis."""
    return np.stack([np.einsum("...j,...j->...", a[..., :W - k], a[..., k:]) for k in range(NLAG)], axis=-1)


def _fft_ac(a: np.ndarray) -> np.ndarray:
    s = np.fft.rfft(a, NFFT, axis=-1)
    return np.fft.irfft(s.real * s.real + s.imag * s.imag, NFFT, axis=-1)[..., :NLAG]


def window_r() -> np.ndarray:
    """r_w(k) / r_w(0), k = 0 .. NLAG - 1 (direct sum)."""
    rw = _direct_ac(hanning())
    return rw / rw[0]


def frame_data(x: np.ndarray, fft: bool = False):
    """Per frame: r [F, NLAG] (zero rows where r_a(0) = 0), the local peaks, the global peak."""
    x = np.asarray(x, np.float64)
    lefts = frame_lefts(x.shape[0])
    gp = float(np.max(np.abs(x - x.sum() / x.shape[0])))
    idx = lefts[:, None] + np.arange(-HALF + 1, HALF + 1)[None, :]
    seg = x[idx]
    midx = lefts[:, None] + np.arange(-P + 1, P + 1)[None, :]
    lm = x[midx].sum(axis=1) / (2 * P)
    d = seg - lm[:, None]
    lp = np.abs(d).max(axis=1)
    a = d * hanning()[None, :]
    ra = _fft_ac(a) if fft else _direct_ac(a)
    rw = _fft_ac(hanning()) if fft else _direct_ac(hanning())
    rwn = rw / rw[0]
    r = np.zeros_like(ra)
    ok = ra[:, 0] != 0.0
    r[ok] = (ra[ok] / ra[ok, :1]) / rwn[None, :]
    return r, lp, gp


# ------------------------------------------------------------------------------------------ sinc interpolation
_B = math.pi / (DEPTH + 0.5)


def _g(d: np.ndarray, sp: float, cp: float, sign: np.ndarray):
    """g, g', g'' at d = u - q (u = t - m in [0, 1)); sp, cp = sin(pi u), cos(pi u); sign = (-1)^q."""
    pi = math.pi
    small = np.abs(d) < 1e-3
    ds = np.where(small, 1.0, d)
    s = sign * sp / (pi * ds)
    s1 = (sign * cp - s) / ds
    s2 = -pi * pi * s - 2.0 * s1 / ds
    p2 = (pi * d) ** 2
    s = np.where(small, 1.0 - p2 / 6.0 + p2 * p2 / 120.0, s)
    s1 = np.where(small, -pi * pi * d / 3.0 + pi ** 4 * d ** 3 / 30.0, s1)
    s2 = np.where(small, -pi * pi / 3.0 + pi ** 4 * d * d / 10.0, s2)
    c, sn = np.cos(_B * d), np.sin(_B * d)
    w, w1, w2 = 0.5 + 0.5 * c, -0.5 * _B * sn, -0.5 * _B * _B * c
    return s * w, s1 * w + s * w1, s2 * w + 2.0 * s1 * w1 + s * w2


def interp(r: np.ndarray, t: float):
    """The sinc interpolant of r (lags 0 .. NLAG - 1, mirrored below 0) and its first two derivatives at lag t."""
    m = math.floor(t)
    u = t - m
    q = np.arange(-DEPTH + 1, DEPTH + 1)
    sign = np.where(q % 2 == 0, 1.0, -1.0)
    g, g1, g2 = _g(u - q, math.sin(math.pi * u), math.cos(math.pi * u), sign)
    v = r[np.abs(m + q)]
    return float(np.sum(v * g)), float(np.sum(v * g1)), float(np.sum(v * g2))


def refine(r: np.ndarray, k: int):
    """(lag, r) of the maximum near the local maximum at integer lag k."""
    a, b, c = r[k - 1], r[k], r[k + 1]
    den = a - 2.0 * b + c
    t = k + 0.5 * (a - c) / den if den < 0.0 else float(k)
    if not (k - 1 <= t <= k + 1):
        t = float(k)
    for _ in range(NEWTON_STEPS):
        _, f1, f2 = interp(r, t)
        if not f2 < 0.0:
            break
        step = f1 / f2
        tn = t - step
        if not (k - 1 <= tn <= k + 1):
            break
        t = tn
        if abs(step) < 1e-10:
            break
    return t, interp(r, t)[0]


# ------------------------------------------------------------------------------------------ candidates
def frame_candidates(r: np.ndarray, lp: float, gp: float, margins: list | None = None):
    """(freqs, strengths) of one frame, the unvoiced candidate first, then at most 14 voiced in ascending lag."""
    ratio = lp / gp if gp > 0.0 else 0.0
    unv = VOICING + max(0.0, 2.0 - ratio / (SILENCE / (1.0 + VOICING)))
    cands = []
    if r[0] != 0.0:
        thr = 0.5 * VOICING
        for k in range(MIN_LAG, MAX_LAG + 1):
            if margins is not None and r[k] > thr - 1e-12:
                margins.append(min(abs(r[k] - thr), abs(r[k] - r[k - 1]), abs(r[k] - r[k + 1])))
            if r[k] > thr and r[k] > r[k - 1] and r[k] >= r[k + 1]:
                t, v = refine(r, k)
                cands.append((t, FS / t, v - OCTAVE_COST * math.log2(FLOOR * t / FS)))
    if len(cands) > MAX_CANDIDATES - 1:
        order = sorted(range(len(cands)), key=lambda i: (-cands[i][2], i))
        if margins is not None:
            margins.append(cands[order[MAX_CANDIDATES - 2]][2] - cands[order[MAX_CANDIDATES - 1]][2])
        keep = sorted(order[:MAX_CANDIDATES - 1])
        cands = [cands[i] for i in keep]
    return [0.0] + [c[1] for c in cands], [unv] + [c[2] for c in cands]


def candidates(x, margins: list | None = None):
    r, lp, gp = frame_data(x)
    out = [frame_candidates(r[i], float(lp[i]), gp, margins) for i in range(r.shape[0])]
    return [o[0] for o in out], [o[1] for o in out]


# ------------------------------------------------------------------------------------------ path finder
def transition(f1: float, f2: float) -> float:
    if f1 == 0.0 and f2 == 0.0:
        return 0.0
    if f1 == 0.0 or f2 == 0.0:
        return VUV_COST * TSC
    return OCTAVE_JUMP_COST * abs(math.log2(f1 / f2)) * TSC


def viterbi(freqs: list, strengths: list):
    """(best path as candidate indices, the smallest margin between the best and second-best choice it took)."""
    F = len(freqs)
    delta = list(strengths[0])
    back = []
    marg = []   # per frame and candidate: best - second best over the predecessors
    for i in range(1, F):
        nd, bp, mg = [], [], []
        for c, fc in enumerate(freqs[i]):
            vals = [delta[p] - transition(fp, fc) for p, fp in enumerate(freqs[i - 1])]
            best = max(range(len(vals)), key=lambda p: (vals[p], -p))
            second = max([v for p, v in enumerate(vals) if p != best], default=-math.inf)
            nd.append(vals[best] + strengths[i][c])
            bp.append(best)
            mg.append(vals[best] - second)
        delta, back, marg = nd, back + [bp], marg + [mg]
    last = max(range(len(delta)), key=lambda c: (delta[c], -c))
    margin = max([v for c, v in enumerate(delta) if c != last], default=-math.inf)
    margin = delta[last] - margin
    path = [last]
    for i in range(F - 1, 0, -1):
        margin = min(margin, marg[i - 1][path[-1]])
        path.append(back[i - 1][path[-1]])
    return path[::-1], margin


def path_score(freqs, strengths, path) -> float:
    s = strengths[0][path[0]]
    for i in range(1, len(path)):
        s = (s - transition(freqs[i - 1][path[i - 1]], freqs[i][path[i]])) + strengths[i][path[i]]
    return s


def praat_f0_unpadded(x, info: dict | None = None) -> np.ndarray:
    """One value per frame: what svcb_praat_f0_ragged computes."""
    margins = [] if info is not None else None
    freqs, strengths = candidates(x, margins)
    path, m = viterbi(freqs, strengths)
    if info is not None:
        info["path_margin"] = m
        info["candidate_margin"] = min(margins, default=math.inf)
    return np.array([freqs[i][c] for i, c in enumerate(path)], np.float64)


def praat_f0(x) -> np.ndarray:
    """parselmouth.Sound(x, 16000).to_pitch_ac(0.01, 30, ..., voicing 0.5, ceiling 1000) frequencies, padded 6 + 6."""
    return np.pad(praat_f0_unpadded(x), [[PAD, PAD]], mode="constant")


# ------------------------------------------------------------------------------------------ synthetic fixture
def tone(f0_track: np.ndarray, rng, amp=0.3, harmonics=(1.0, 0.5, 0.3, 0.2, 0.1)) -> np.ndarray:
    """A harmonic tone whose fundamental follows f0_track (Hz per sample; 0 = silence there)."""
    ph = 2.0 * np.pi * np.cumsum(f0_track) / FS + rng.uniform(0, 2 * np.pi)
    x = np.zeros_like(f0_track)
    for k, a in enumerate(harmonics, 1):
        x += a * np.sin(k * ph) * (k * f0_track < FS / 2)
    return amp * x * (f0_track > 0)


TONES = (40.0, 75.0, 130.0, 220.0, 370.0, 600.0, 950.0)
STRONG2 = (1.0, 1.6, 0.3, 0.15)     # second harmonic stronger than the fundamental: the octave-error trap
SHORT = (1600, 1601, 1759, 1760, 1761, 1919, 1921, 3200, 3361)   # one frame and the grid's edges


def _raw_items(seed: int):
    rng = np.random.default_rng(seed)
    t = lambda s: np.arange(int(s * FS)) / FS
    items = {}
    for f in TONES:
        n = int(0.45 * FS) + int(rng.integers(0, 160))
        items[f"tone_{int(f)}"] = (np.full(n, f), STRONG2)
    items["glide"] = (70.0 * (900.0 / 70.0) ** (t(1.6) / 1.6), None)
    tt = t(1.0)
    items["vibrato"] = (260.0 * 2.0 ** (0.6 / 12 * np.sin(2 * np.pi * 5.5 * tt)), None)
    tr = np.zeros(int(1.6 * FS) + 41)
    for a, b, f in ((0.15, 0.65, 140.0), (0.85, 1.45, 420.0)):
        tr[int(a * FS):int(b * FS)] = f
    items["onsets"] = (tr, None)
    out = {}
    for k, (tr, h) in items.items():
        out[k] = (tone(tr, rng) if h is None else tone(tr, rng, harmonics=h), tr)
    out["noise"] = (0.1 * rng.standard_normal(int(0.7 * FS) + 13), np.zeros(int(0.7 * FS) + 13))
    out["silence"] = (np.zeros(int(0.4 * FS) + 7), np.zeros(int(0.4 * FS) + 7))
    for n in SHORT:
        tr = np.full(n, float(rng.uniform(120, 500)))
        out[f"short_{n}"] = (tone(tr, rng) + 1e-3 * rng.standard_normal(n), tr)
    return {k: (x.astype(np.float32), tr) for k, (x, tr) in out.items()}


def synth_items(seed: int = 0) -> dict:
    """name -> (float32 audio at 16 kHz, true F0 per sample, 0 where unvoiced).  A clip whose best path or candidate
    choices sit within 1e-9 / 1e-12 of a tie is drawn again with the next seed, so no test rests on a rounding-equal
    choice."""
    out = {}
    names = list(_raw_items(seed))
    for name in names:
        s = seed
        while True:
            x, tr = _raw_items(s)[name]
            info = {}
            praat_f0_unpadded(x.astype(np.float64), info)
            if info["path_margin"] >= 1e-9 and info["candidate_margin"] >= 1e-12:
                break
            s += 1000
        out[name] = (x, tr)
    return out


def frame_truth(true_track: np.ndarray) -> tuple:
    """The true F0 at each frame centre (0 unvoiced) and the frames whose window lies 30 ms or more inside a voiced run."""
    n = true_track.shape[0]
    lefts = frame_lefts(n)
    f = true_track[lefts].copy()
    voiced = true_track > 0
    ok = np.zeros(lefts.shape[0], bool)
    for i, c in enumerate(lefts):
        a, b = c - HALF - 480, c + HALF + 480
        ok[i] = a >= 0 and b < n and voiced[a:b + 1].all()
    return f, ok


def make_golden(path: str = GOLDEN) -> None:
    items = synth_items()
    arrs = {}
    for k, (x, tr) in items.items():
        arrs[f"{k}/x"] = x
        arrs[f"{k}/f0"] = praat_f0_unpadded(x.astype(np.float64))
    np.savez_compressed(path, **arrs)


def load_golden(path: str = GOLDEN) -> dict:
    """name -> (audio, oracle F0 per frame, unpadded)."""
    z = np.load(path)
    names = sorted({k.split("/")[0] for k in z.files})
    return {k: (z[f"{k}/x"], z[f"{k}/f0"]) for k in names}


if __name__ == "__main__":
    make_golden()
    print("wrote", GOLDEN, os.path.getsize(GOLDEN), "bytes")
