"""Restatement of prepare/preprocess_f0.py's pyworld calls in numpy fp64 (TEST INFRASTRUCTURE).

`dio` restates WORLD's DIO (Morise, Kawahara and Katayose, "Fast and reliable F0 estimation method based on the period
extraction of vocal fold vibration of singing voice and speech", AES 35th conference, 2009) as pyworld 0.3.x bundles it,
at the settings the reference uses: fs 16 kHz, f0_floor 71, f0_ceil 900, two channels per octave (eight bands),
speed 1, allowed_range 0.1 and a 10 ms frame period.  `stonemask` restates StoneMask's instantaneous-frequency
refinement (Morise, Kawahara and Nishiura, "Rapid F0 estimation for high-SNR speech based on fundamental component
extraction", IEICE Trans. J93-D, 2010).  Both were written from the published algorithms; the steps are:

- the signal plus one trailing zero (y_length = n + 1), minus its mean, through a 641-tap zero-phase Hann low-cut
  filter (50 Hz) and then, per band, a Nuttall window of 4 h taps (h = round(fs / boundary / 2)) centred by a delay
  of 2 h.  WORLD filters by FFT with a transform long enough that nothing wraps, so this is linear convolution; here
  it is np.convolve.
- per band, the falling zero crossings of the band signal, of its negation, and of its first difference both ways:
  each gives intervals fs / (e[k+1] - e[k]) between linearly refined crossings e, placed at their midpoints.
- each family linearly interpolated onto the 10 ms grid (extrapolated from the end segments, as WORLD's interp1 with
  histc does), the candidate is the mean of the four, its score their standard deviation over the candidate; a
  candidate outside [boundary / 2, boundary] or [f0_floor, f0_ceil], or a band with fewer than three intervals in any
  family, is rejected.
- per frame, the candidate of the lowest score; then FixF0Contour's four steps.
- StoneMask per voiced frame: a Blackman window of 3 periods either side, its time derivative, and the
  instantaneous frequency of harmonics 1-2 and then 1-6, amplitude-weighted.

pyworld is not installed where this was written, so this restatement is not pinned to it there: tests/test_f0_cpu.py
pins it wherever pyworld imports, and checks it against the true F0 of synthetic tones everywhere (DESIGN.md §8).

One defined deviation: StoneMask's harmonic bins above fft_size / 2 lie outside WORLD's spectrum array, so their
reading there is undefined; here such a bin counts as zero power.  It can only happen when the 2-harmonic estimate is
near twice the DIO value, which the 20 % rule then rejects anyway.

    python oracle/f0_oracle.py    writes tests/golden/f0_synth.npz: seeded clips and the oracle's F0 before rounding
"""
from __future__ import annotations

import math
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "f0_synth.npz")

FS = 16000
FRAME_PERIOD = 10.0
F0_FLOOR = 71.0
F0_CEIL = 900.0
CHANNELS_IN_OCTAVE = 2.0
ALLOWED_RANGE = 0.1
CUTOFF = 50.0
SAFE = 1e-12            # world::kMySafeGuardMinimum
MAX_SCORE = 100000.0    # world::kMaximumValue
FLOOR_STONEMASK = 40.0  # world::kFloorF0StoneMask
LOG2 = 0.69314718055994529
HOP = 160               # samples per frame at 16 kHz and 10 ms
VOICE_RANGE_MIN = int(0.5 + 1000.0 / FRAME_PERIOD / F0_FLOOR) * 2 + 1   # 3
MIN_SAMPLES = HOP * VOICE_RANGE_MIN   # 480: fewer samples give at most 3 frames, and the contour fix writes nothing


def matlab_round(x: float) -> int:
    return int(x + 0.5) if x > 0 else int(x - 0.5)


def n_frames(n: int) -> int:
    """GetSamplesForDIO: int(1000 n / fs / frame_period) + 1 = n // 160 + 1."""
    return int(1000.0 * n / FS / FRAME_PERIOD) + 1


def n_bands() -> int:
    return 1 + int(math.log(F0_CEIL / F0_FLOOR) / LOG2 * CHANNELS_IN_OCTAVE)


def boundaries() -> list:
    return [F0_FLOOR * 2.0 ** ((i + 1) / CHANNELS_IN_OCTAVE) for i in range(n_bands())]


def half_lengths() -> list:
    """h of each band: its Nuttall low-pass has 4 h taps."""
    return [matlab_round(FS / b / 2.0) for b in boundaries()]


def lowcut_taps() -> np.ndarray:
    """The zero-phase low-cut filter, taps -320 .. 320 (DesignLowCutFilter): minus a normalised Hann, plus 1 at 0."""
    N = matlab_round(FS / CUTOFF) * 2 + 1
    h = np.array([0.5 - 0.5 * math.cos(i * 2.0 * math.pi / (N + 1)) for i in range(1, N + 1)])
    s = 0.0
    for v in h:                      # summed in order, as WORLD does
        s += v
    h = -h / s
    h[(N - 1) // 2] += 1.0
    return h


def nuttall(n: int) -> np.ndarray:
    t = np.arange(n) / (n - 1.0)
    return (0.355768 - 0.487396 * np.cos(2.0 * np.pi * t) + 0.144232 * np.cos(4.0 * np.pi * t)
            - 0.012604 * np.cos(6.0 * np.pi * t))


def band_signals(x: np.ndarray) -> list:
    """The eight band signals of y = [x, 0] - mean, each y_length = n + 1 long."""
    x = np.asarray(x, np.float64)
    y = np.concatenate([x, [0.0]])
    y = y - y.sum() / y.shape[0]
    lc = np.convolve(y, lowcut_taps())          # position j at index j + 320, j = -320 .. y_length + 319
    out = []
    for h in half_lengths():
        f = np.convolve(lc, nuttall(4 * h))     # sum_k w[k] lc(i + 2h - k) at index i + 2h + 320
        out.append(f[2 * h + 320: 2 * h + 320 + y.shape[0]])
    return out


def fine_edges(s: np.ndarray) -> np.ndarray:
    """ZeroCrossingEngine's refined falling crossings of s: e - s[e-1] / (s[e] - s[e-1]) where s[e-1] > 0 >= s[e]."""
    e = np.flatnonzero((s[:-1] > 0.0) & (s[1:] <= 0.0)) + 1
    return e - s[e - 1] / (s[e] - s[e - 1])


def event_families(f: np.ndarray) -> list:
    """(locations in s, intervals in Hz) of the negative-going, positive-going, peak and dip families."""
    d = f[1:] - f[:-1]
    out = []
    for s in (f, -f, d, -d):
        fe = fine_edges(s)
        if fe.shape[0] < 2:
            out.append((np.zeros(0), np.zeros(0)))
            continue
        out.append(((fe[:-1] + fe[1:]) / 2.0 / FS, FS / (fe[1:] - fe[:-1])))
    return out


def interp1(x: np.ndarray, y: np.ndarray, xi: np.ndarray) -> np.ndarray:
    """WORLD's interp1: linear, extrapolated from the first and last segments (histc's index clipped to 1 .. n-1)."""
    k = np.clip(np.searchsorted(x, xi, side="right"), 1, x.shape[0] - 1)
    s = (xi - x[k - 1]) / (x[k] - x[k - 1])
    return y[k - 1] + s * (y[k] - y[k - 1])


def temporal_positions(F: int) -> np.ndarray:
    return np.arange(F) * FRAME_PERIOD / 1000.0


def candidates(x: np.ndarray):
    """(raw candidates [bands, F], scores [bands, F]) of GetF0CandidatesAndScores."""
    F = n_frames(len(x))
    t = temporal_positions(F)
    cands, scores = [], []
    for b, f in zip(boundaries(), band_signals(x)):
        fam = event_families(f)
        if min(len(v[0]) for v in fam) < 3:
            c, sc = np.zeros(F), np.full(F, MAX_SCORE)
        else:
            a = [interp1(loc, iv, t) for loc, iv in fam]
            c = (a[0] + a[1] + a[2] + a[3]) / 4.0
            sc = np.sqrt(((a[0] - c) * (a[0] - c) + (a[1] - c) * (a[1] - c) + (a[2] - c) * (a[2] - c)
                          + (a[3] - c) * (a[3] - c)) / 3.0)
            bad = (c > b) | (c < b / 2.0) | (c > F0_CEIL) | (c < F0_FLOOR)
            c = np.where(bad, 0.0, c)
            sc = np.where(bad, MAX_SCORE, sc)
        cands.append(c)
        scores.append(sc / (c + SAFE))
    return np.array(cands), np.array(scores)


def best_contour(cands: np.ndarray, scores: np.ndarray) -> np.ndarray:
    best = cands[0].copy()
    tmp = scores[0].copy()
    for j in range(1, cands.shape[0]):
        m = tmp > scores[j]
        tmp = np.where(m, scores[j], tmp)
        best = np.where(m, cands[j], best)
    return best


def _select_best(cur, past, cands, j):
    ref = (cur * 3.0 - past) / 2.0
    col = cands[:, j]
    err = abs(ref - col[0])
    best = col[0]
    for i in range(1, col.shape[0]):
        e = abs(ref - col[i])
        if e < err:
            err, best = e, col[i]
    with np.errstate(divide="ignore", invalid="ignore"):
        r = abs(1.0 - np.float64(best) / np.float64(ref))
    return 0.0 if r > ALLOWED_RANGE else float(best)


def fix_contour(best: np.ndarray, cands: np.ndarray) -> np.ndarray:
    """FixF0Contour: jump removal, short-run removal, forward then backward extension from the candidates."""
    F, vrm = best.shape[0], VOICE_RANGE_MIN
    out = np.zeros(F)
    if F <= vrm:
        return out
    base = np.zeros(F)
    base[vrm:F - vrm] = best[vrm:F - vrm]
    s1 = np.zeros(F)
    for i in range(vrm, F):
        s1[i] = base[i] if abs((base[i] - base[i - 1]) / (SAFE + base[i])) < ALLOWED_RANGE else 0.0
    s2 = s1.copy()
    c = (vrm - 1) // 2
    for i in range(c, F - c):
        if np.any(s1[i - c:i + c + 1] == 0):
            s2[i] = 0.0
    neg = [i - 1 for i in range(1, F) if s2[i] == 0 and s2[i - 1] != 0]
    pos = [i for i in range(1, F) if s2[i - 1] == 0 and s2[i] != 0]
    s3 = s2.copy()
    for i in range(len(neg)):
        limit = F - 1 if i == len(neg) - 1 else neg[i + 1]
        for j in range(neg[i], limit):
            s3[j + 1] = _select_best(s3[j], s3[j - 1], cands, j + 1)
            if s3[j + 1] == 0:
                break
    s4 = s3.copy()
    for i in range(len(pos) - 1, -1, -1):
        limit = 1 if i == 0 else pos[i - 1]
        for j in range(pos[i], limit, -1):
            s4[j - 1] = _select_best(s4[j], s4[j + 1], cands, j - 1)
            if s4[j - 1] == 0:
                break
    return s4


def dio(x: np.ndarray) -> np.ndarray:
    """pyworld.dio(x, fs=16000, f0_ceil=900, frame_period=10)[0]."""
    x = np.asarray(x, np.float64)
    cands, scores = candidates(x)
    return fix_contour(best_contour(cands, scores), cands)


def _fix_f0(main: np.ndarray, diff: np.ndarray, fft_size: int, f0: float, nh: int) -> float:
    num = den = 0.0
    half = fft_size // 2
    for i in range(nh):
        k = matlab_round(f0 * fft_size / FS * (i + 1))
        if k > half:
            p = 0.0                               # outside WORLD's spectrum array (module docstring)
        else:
            p = main[k].real * main[k].real + main[k].imag * main[k].imag
        if p == 0.0:
            ifreq = 0.0
        else:
            ni = main[k].real * diff[k].imag - main[k].imag * diff[k].real
            ifreq = k * FS / fft_size + ni / p * FS / 2.0 / math.pi
        amp = math.sqrt(p)
        num += amp * ifreq
        den += amp * (i + 1.0)
    return num / (den + SAFE)


def refine_one(x: np.ndarray, pos: float, f0: float) -> float:
    """StoneMask's GetRefinedF0 for one frame."""
    if f0 <= FLOOR_STONEMASK or f0 > FS / 12.0:
        return 0.0
    hw = int(1.5 * FS / f0 + 1.0)
    L = 2 * hw + 1
    wlt = (2.0 * hw + 1.0) / FS
    fft_size = int(2.0 ** (2.0 + int(math.log(hw * 2.0 + 1.0) / LOG2)))
    base_time = (np.arange(L) - hw) / FS
    idx_raw = np.array([matlab_round(v) for v in (pos + base_time) * FS])
    tmp = (idx_raw - 1.0) / FS - pos
    win = 0.42 + 0.5 * np.cos(2.0 * np.pi * tmp / wlt) + 0.08 * np.cos(4.0 * np.pi * tmp / wlt)
    dwin = np.empty(L)
    dwin[0] = -win[1] / 2.0
    dwin[1:-1] = -(win[2:] - win[:-2]) / 2.0
    dwin[-1] = win[-2] / 2.0
    seg = x[np.clip(idx_raw - 1, 0, x.shape[0] - 1)]
    main = np.fft.rfft(seg * win, fft_size)
    diff = np.fft.rfft(seg * dwin, fft_size)
    t = _fix_f0(main, diff, fft_size, f0, 2)
    if t <= 0.0 or t > f0 * 2:
        mean = 0.0
    else:
        mean = _fix_f0(main, diff, fft_size, t, 6)
    return f0 if abs(mean - f0) > f0 * 0.2 else mean


def stonemask(x: np.ndarray, f0: np.ndarray) -> np.ndarray:
    """pyworld.stonemask(x, f0, t, fs=16000) with t the 10 ms grid."""
    x = np.asarray(x, np.float64)
    t = temporal_positions(f0.shape[0])
    return np.array([refine_one(x, t[i], f0[i]) for i in range(f0.shape[0])])


def world_f0(x) -> np.ndarray:
    """dio + stonemask, before the 0.1 rounding: what svcb_world_f0_ragged computes."""
    x = np.asarray(x, np.float64)
    return stonemask(x, dio(x))


def round1(f0) -> np.ndarray:
    """Each value as Python's round(v, 1), the reference's rounding (correctly rounded, ties to even)."""
    return np.array([round(float(v), 1) for v in np.asarray(f0, np.float64).reshape(-1)], np.float64)


# ------------------------------------------------------------------------------------------ synthetic fixture
def tone(f0_track: np.ndarray, rng, amp=0.3, harmonics=(1.0, 0.5, 0.3, 0.2, 0.1)) -> np.ndarray:
    """A harmonic tone whose fundamental follows f0_track (Hz per sample; 0 = silence there)."""
    ph = 2.0 * np.pi * np.cumsum(f0_track) / FS + rng.uniform(0, 2 * np.pi)
    x = np.zeros_like(f0_track)
    for k, a in enumerate(harmonics, 1):
        x += a * np.sin(k * ph) * (k * f0_track < FS / 2)
    return amp * x * (f0_track > 0)


def synth_items(seed: int = 0) -> dict:
    """name -> (float32 audio at 16 kHz, as the loader gives it; true F0 per sample, 0 where unvoiced)."""
    rng = np.random.default_rng(seed)
    t = lambda s: np.arange(int(s * FS)) / FS
    items = {}
    tr = 80.0 * (800.0 / 80.0) ** (t(2.5) / 2.5)
    items["glide_up"] = tr
    tr = np.interp(t(2.0), [0, 1.0, 2.0], [420.0, 150.0, 240.0])
    items["glide_down"] = tr
    tt = t(1.5)
    items["vibrato"] = 220.0 * 2.0 ** (0.5 / 12 * np.sin(2 * np.pi * 5.5 * tt))
    tr = np.zeros(int(3.2 * FS))
    for k, (a, b, f) in enumerate(((0.2, 0.8, 130.0), (1.1, 1.7, 310.0), (2.0, 2.9, 610.0))):
        tr[int(a * FS):int(b * FS)] = f
    items["voiced_unvoiced"] = tr
    items["steady_100"] = np.full(int(1.0 * FS) + 77, 100.0)
    out = {k: (tone(v, rng), v) for k, v in items.items()}
    # a recording's pauses are never digital zeros: there the band signals would be rounding noise, whose crossings
    # differ between any two summation orders
    x, v = out["voiced_unvoiced"]
    out["voiced_unvoiced"] = (x + 1e-3 * rng.standard_normal(x.shape[0]), v)
    out["silence"] = (np.zeros(int(0.8 * FS) + 33), np.zeros(int(0.8 * FS) + 33))
    out["noise"] = (0.1 * rng.standard_normal(2 * FS + 101), np.zeros(2 * FS + 101))
    n = 1000                                    # seven frames
    out["short"] = (tone(np.full(n, 200.0), rng), np.full(n, 200.0))
    return {k: (x.astype(np.float32), tr) for k, (x, tr) in out.items()}


def frame_truth(true_track: np.ndarray) -> np.ndarray:
    """The true F0 at each frame centre (0 unvoiced) and the frames at least 30 ms after an onset and before an end."""
    F = n_frames(true_track.shape[0])
    idx = np.minimum(np.arange(F) * HOP, true_track.shape[0] - 1)
    f = true_track[idx].copy()
    voiced = true_track > 0
    ok = np.zeros(F, bool)
    for i in range(F):
        a, b = idx[i] - 480, idx[i] + 480
        ok[i] = a >= 0 and b < true_track.shape[0] and voiced[a:b + 1].all()
    return f, ok


def make_golden(path: str = GOLDEN) -> None:
    items = synth_items()
    arrs = {}
    for k, (x, _) in items.items():
        arrs[f"{k}/x"] = x
        arrs[f"{k}/f0"] = world_f0(x)
    np.savez_compressed(path, **arrs)


def load_golden(path: str = GOLDEN) -> dict:
    """name -> (audio, oracle F0 before rounding)."""
    z = np.load(path)
    names = sorted({k.split("/")[0] for k in z.files})
    return {k: (z[f"{k}/x"], z[f"{k}/f0"]) for k in names}


if __name__ == "__main__":
    make_golden()
    print("wrote", GOLDEN)
