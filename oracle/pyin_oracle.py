"""pYIN F0 (libf0's `pyin()` of pitch/core/pyin.py at Fs=16000, N=2048, H=160, F_min=50, F_max=1000, defaults
otherwise), restated in numpy (TEST INFRASTRUCTURE).  The wrapper and its parameters are this project's choice
(whisper-vits-svc_b200/pyin_f0.py): no command of the reference calls pyin.

The steps, each as the reference computes it and as the device (csrc/pyin_f0_api.cu) restates it:
1. Frames: 1024 zeros on each side of the signal, M = n // 160 + 1 frames of 2048 samples; one sample gives one frame.
2. CMNDF per frame (yin.py:cumulative_mean_normalized_difference_function), 321 values: cmndf[0] = 1; for tau = 1 ..
   320 the difference d(tau) = sum_j (x_j - x_{j+tau})^2 over 2048 - tau samples, each square rounded and added in
   ascending j (numba's np.sum); the mean updated as m = m (tau - 1) / tau + d / tau; cmndf = d / (m + eps64).  The
   frame's RMS is sqrt(sum x^2 / 2048), summed in the same order.
3. Probabilistic thresholding (pyin.py:probabilistic_thresholding) with p_min = 16, p_max = 320:
   - cmndf[:16] and cmndf[320:] = inf; local minima are strict, in 1 .. 319.
   - Every minimum is interpolated parabolically and the value written back, the ones at 16 and 319 included: the
     reference's `delete_numba(arr, np.argwhere(arr == v))` compares the elements with the *position* p of v and
     then drops the element at the row index of the match, which is always 0.  So it drops nothing when v = 16
     (p = 0, and no lag is 0), and drops the *first* minimum when v = 319 (p = k - 1, k minima) and some minimum
     lies at lag k - 1.  Next to an inf the parabola gives NaN, so an interpolated minimum at 16 or 319 becomes NaN:
     it is never under a threshold, and argmin / min of the frame return it (the first NaN) when no minimum is.
   - The corrections p_corr follow the interpolated list, with a 0 in front when a minimum sits at 16 and a 0 at the
     end when one sits at 319.  The lag of a threshold is the first minimum under it plus p_corr[0]: always the first
     entry, the reference's np.argmin(min_idxs_thr) being 0.  With no minimum under it: argmin(cmndf), weight 0.01.
     With no minima at all: a zero column, lags 16, values 1.  Lags are clamped to [16, 319].
   - The bin is the first argmin of |1200 log2(F_axis / (16000 / lag))|; O[bin] += weight * beta[i] in threshold order.
4. O[:518] *= 0.5; O[518:] = 0.5 (1 - sum of the voiced half, ascending) / 518.
5. Viterbi (pyin.py:viterbi_log_likelihood) on log(A + tiny), log(1 / 1036 + tiny) and log(O + tiny), tiny the
   smallest normal double.  `viterbi_banded` restates the dense recursion exactly: a column's predecessors with A > 0
   (the band and the voiced / unvoiced cross entry), plus, when it lies outside them, g: the first k whose rounded
   log(tiny) + D[k] equals log(tiny) + max D.  Every other predecessor scores log(tiny) + D[k], and rounding is
   monotone, so none of them scores above g's sum and those that tie with it come later.  g is not always the argmax
   of D: adding -708 absorbs differences in the last bits of D.  An in-band g scores about 700 nats above that sum, so
   then no other predecessor can win.  Ties go to the lowest index, as np.argmax.
6. f0 = F_axis extended by zeros at the path; f0[0] = 0; f0[rms < 0.01] = 0; conf = O[path, m] / max O[:, m]; then
   refine_estimates_yin: a voiced frame takes, among the thresholds' float lags within 10 cents of f0, the one with
   the smallest CMNDF value (first on ties, first NaN first), else keeps f0.

The logarithms of the Viterbi tables and the quantisation run through `math` (the C library's log and log2, which
numba calls too), so the tables are bitwise the reference's.

`python oracle/pyin_oracle.py` writes tests/golden/pyin_synth.npz.
"""
from __future__ import annotations

import functools
import math
import operator
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "pyin_synth.npz")

FS = 16000
N = 2048
HOP = 160
F_MIN = 50.0
F_MAX = 1000.0
R = 10
BETA_PARAMS = (1, 18)
ABS_MIN_PROB = 0.01
VOICING_PROB = 0.5
MAX_STEP = int(50 / R)                                   # 5
B = int(np.log2(F_MAX / F_MIN) * (1200 / R))             # 518 pitch bins
S = 2 * B                                                # 1036 HMM states
P_MIN = max(int(np.ceil(FS / F_MAX)), 1)                 # 16
P_MAX = int(np.ceil(FS / F_MIN))                         # 320
LAGS = P_MAX + 1                                         # 321 CMNDF values
NTHR = 99
BAND = 12                                                # predecessors with A > 0 per column, at most
TINY = np.finfo(0.).tiny
EPS = np.finfo(np.float64).eps
_log = np.frompyfunc(math.log, 1, 1)


def n_frames(n: int) -> int:
    return int(n) // HOP + 1


def thresholds() -> np.ndarray:
    return np.arange(0.01, 1, 0.01)


def beta_distr() -> np.ndarray:
    from scipy.special import beta, comb
    thr = thresholds()
    i = np.arange(len(thr))
    a, b = BETA_PARAMS
    return comb(len(thr), i) * beta(i + a, len(thr) - i + b) / beta(a, b)


def f_axis() -> np.ndarray:
    return F_MIN * np.power(2, np.arange(B) * R / 1200)


def triang_distr() -> np.ndarray:
    from scipy.stats import triang
    return triang.pdf(np.arange(-MAX_STEP, MAX_STEP + 1), 0.5, scale=2 * MAX_STEP, loc=-MAX_STEP)


def transition_matrix() -> np.ndarray:
    """The HMM's transitions (pyin.py:compute_transition_matrix with the 11-tap triangle), A[k, j] from state k to j.
    Within each half a state k moves to j = k - 5 .. k + 5 with weight 0.99 t[j - k + 5]; a row that the edge of its
    half cuts short is divided by the sum of the taps it keeps, added in ascending order (numba's np.sum).  Each voiced
    state moves to its unvoiced twin with 1 - 0.99, and back."""
    t = triang_distr()
    A = np.zeros((S, S))
    for half in (0, B):
        for k in range(B):
            lo, hi = max(0, k - MAX_STEP), min(B, k + MAX_STEP + 1)
            taps = t[lo - k + MAX_STEP:hi - k + MAX_STEP]
            row = 0.99 * taps
            if hi - lo < 2 * MAX_STEP + 1:
                row = row / functools.reduce(operator.add, taps.tolist(), 0.0)
            A[half + k, half + lo:half + hi] = row
    k = np.arange(B)
    A[k, k + B] = 1 - 0.99
    A[k + B, k] = 1 - 0.99
    return A


def band(A: np.ndarray | None = None) -> tuple:
    """([S, BAND] predecessor index, -1 past the end; [S, BAND] log(A + tiny), -inf past the end): each column's
    predecessors with A > 0, ascending."""
    A = transition_matrix() if A is None else A
    idx = np.full((S, BAND), -1, np.int64)
    val = np.full((S, BAND), -np.inf)
    for i in range(S):
        k = np.flatnonzero(A[:, i] > 0)
        assert k.shape[0] <= BAND
        idx[i, :k.shape[0]] = k
        val[i, :k.shape[0]] = _log(A[k, i] + TINY).astype(np.float64)
    return idx, val


def log_init() -> float:
    return math.log(1.0 / S + TINY)


def log_tiny() -> float:
    return math.log(TINY)


def frames(x) -> np.ndarray:
    """[M, 2048] float64 frames of the zero-padded signal."""
    x = np.asarray(x).reshape(-1)
    if x.shape[0] < 1:
        raise ValueError("no samples")
    xp = np.concatenate((np.zeros(N // 2), x, np.zeros(N // 2)))
    M = n_frames(x.shape[0])
    return xp[np.arange(M)[:, None] * HOP + np.arange(N)[None, :]]


def _seqsum(v: np.ndarray) -> np.ndarray:
    """Sum over the last axis, one accumulator in ascending order, as numba sums a difference of squares."""
    return np.cumsum(v, axis=-1)[..., -1]


def cmndf(fr: np.ndarray) -> tuple:
    """([M, 321] CMNDF, [M] RMS) of frames."""
    M = fr.shape[0]
    c = np.zeros((M, LAGS))
    c[:, 0] = 1
    mean = np.zeros(M)
    for tau in range(1, LAGS):
        d = fr[:, :-tau] - fr[:, tau:]
        diff = _seqsum(d * d)
        mean = mean * (tau - 1) / tau + diff / tau
        c[:, tau] = diff / (mean + EPS)
    rms = np.sqrt(_seqsum(fr * fr) / N)
    return c, rms


def quantise(lag: float, fa: np.ndarray) -> tuple:
    """(first argmin of |1200 log2(F_axis / (16000 / lag))|, gap between the two smallest distances).  The distance
    falls then rises along the axis, so the minimum lies within two bins of the nearest log-frequency bin."""
    f = FS / lag
    b0 = int(round(120 * math.log2(f / F_MIN)))
    lo, hi = max(0, b0 - 3), min(B, b0 + 4)
    dist = np.array([abs(1200 * math.log2(fa[b] / f)) for b in range(lo, hi)])
    j = int(np.argmin(dist))
    s = np.sort(dist)
    return lo + j, float(gap(s[1], s[0])) if s.shape[0] > 1 else np.inf


def parabolic(y1, y2, y3):
    """(offset of the vertex from the middle sample, value there) of the parabola through three equally spaced
    samples, its curvature nudged by eps64 as yin.py does."""
    curv = (y1 + y3 - 2 * y2) / 2 + EPS
    slope = (y3 - y1) / 2
    return -slope / (2 * curv), y2 - slope * slope / (4 * curv)


def gap(a, b):
    """The decision margin's unit: |a - b| over max(1, |a|, |b|), for any two values a decision compares."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b) / np.maximum(1.0, np.maximum(np.abs(a), np.abs(b)))


def threshold_frame(c: np.ndarray, thr, beta, fa) -> tuple:
    """pyin.py:probabilistic_thresholding of one frame's CMNDF (a copy is modified) -> (O column [S] before the
    normalisation, float lags [99], values [99], decision margin, the CMNDF after the write-back)."""
    c = c.copy()
    c[:P_MIN] = np.inf
    c[P_MAX:] = np.inf
    margin = np.inf
    fin = np.isfinite(c[:-1]) & np.isfinite(c[1:])
    if fin.any():
        margin = float(gap(c[1:][fin], c[:-1][fin]).min())
    with np.errstate(invalid="ignore"):
        mins = np.flatnonzero((c[1:-1] < c[:-2]) & (c[1:-1] < c[2:])) + 1
    O = np.zeros(S)
    if mins.size == 0:
        return O, np.full(NTHR, float(P_MIN)), np.ones(NTHR), margin, c
    k = mins.shape[0]
    interp = mins
    if mins[-1] == P_MAX - 1 and (mins == k - 1).any():   # delete_numba's quirk: see the module's docstring
        interp = mins[1:]
    with np.errstate(invalid="ignore", divide="ignore"):
        p_corr, c[interp] = parabolic(c[interp - 1], c[interp], c[interp + 1])
    if mins[0] == P_MIN:
        p_corr = np.concatenate(([0.0], p_corr))
    if mins[-1] == P_MAX - 1:
        p_corr = np.concatenate((p_corr, [0.0]))
    lags = np.zeros(NTHR)
    vals = np.zeros(NTHR)
    cm = c[mins]
    fin = np.isfinite(c)
    srt = np.sort(c[fin])
    for i, t in enumerate(thr):
        under = mins[cm < t]
        with np.errstate(invalid="ignore"):
            d = gap(cm, t)
        if np.isfinite(d).any():
            margin = min(margin, float(np.nanmin(d)))
        if under.size == 0:
            lag = float(np.argmin(c))
            am = ABS_MIN_PROB
            val = np.min(c)
            if srt.shape[0] > 1 and not np.isnan(c).any():
                margin = min(margin, float(gap(srt[1], srt[0])))
        else:
            am = 1
            lag = float(under[0]) + p_corr[0]
            val = c[under[0]]
        if lag < P_MIN:
            lag = P_MIN
        elif lag >= P_MAX:
            lag = P_MAX - 1
        lags[i], vals[i] = lag, val
        idx, qgap = quantise(lag, fa)
        margin = min(margin, qgap)
        O[idx] += am * beta[i]
    return O, lags, vals, margin, c


def observations(x, info: dict | None = None) -> tuple:
    """(O [S, M], rms [M], lags [99, M], values [99, M]) of float audio at 16 kHz; info gets the CMNDF [M, 321] and
    each frame's decision margin."""
    fr = frames(x)
    C, rms = cmndf(fr)
    M = fr.shape[0]
    thr, beta, fa = thresholds(), beta_distr(), f_axis()
    O = np.zeros((S, M))
    lags = np.zeros((NTHR, M))
    vals = np.zeros((NTHR, M))
    margin = np.zeros(M)
    for m in range(M):
        O[:, m], lags[:, m], vals[:, m], margin[m], _ = threshold_frame(C[m], thr, beta, fa)
        margin[m] = min(margin[m], float(gap(rms[m], 0.01)))
    O[0:B, :] *= VOICING_PROB
    O[B:, :] = (1 - VOICING_PROB) * (1 - np.cumsum(O[0:B, :], axis=0)[-1]) / B     # summed in ascending bins
    if info is not None:
        info["cmndf"], info["margin"] = C, margin
    return O, rms, lags, vals


def viterbi_banded(O: np.ndarray, tabs: tuple | None = None) -> np.ndarray:
    """The dense Viterbi's path (int64 [M]) by the banded-exact recursion."""
    idx, val = band() if tabs is None else tabs
    lt = log_tiny()
    Ol = _log(O + TINY).astype(np.float64)
    M = O.shape[1]
    valid = idx >= 0
    safe = np.where(valid, idx, 0)
    D = log_init() + Ol[:, 0]
    E = np.zeros((max(M - 1, 0), S), np.int64)
    rows = np.arange(S)
    for n in range(1, M):
        cand = np.where(valid, val + D[safe], -np.inf)
        j = np.argmax(cand, axis=1)
        best, arg = cand[rows, j], safe[rows, j]
        vg = lt + np.max(D)
        g = int(np.flatnonzero(lt + D == vg)[0])        # the first k whose off-band term rounds to the largest
        off = ~(idx == g).any(axis=1)
        take = off & ((vg > best) | ((vg == best) & (g < arg)))
        best = np.where(take, vg, best)
        arg = np.where(take, g, arg)
        E[n - 1] = arg
        D = best + Ol[:, n]
    path = np.zeros(M, np.int64)
    path[-1] = int(np.argmax(D))
    for n in range(M - 2, -1, -1):
        path[n] = E[n, path[n + 1]]
    return path


def refine(f0, lags, vals, info_margin: np.ndarray | None = None) -> np.ndarray:
    """pyin.py:refine_estimates_yin with tol = 10 cents."""
    out = np.zeros_like(f0)
    for m in np.flatnonzero(f0 > 0):
        fo = FS / lags[:, m]
        dc = np.array([abs(1200 * math.log2(v / f0[m])) for v in fo])
        if info_margin is not None:
            info_margin[m] = min(info_margin[m], float(gap(dc, R).min()))
        cand = np.flatnonzero(dc < R)
        out[m] = f0[m] if cand.size == 0 else fo[cand[np.argmin(vals[cand, m])]]
    return out


def pyin(x, info: dict | None = None) -> tuple:
    """(f0, conf) as float64 [n // 160 + 1]; info gets cmndf, O, path and margin."""
    info = {} if info is None else info
    O, rms, lags, vals = observations(x, info)
    path = viterbi_banded(O)
    f0 = np.concatenate((f_axis(), np.zeros(B)))[path]
    f0[0] = 0
    f0[rms < 0.01] = 0
    conf = (O / np.max(O, axis=0))[path, np.arange(O.shape[1])]
    f0 = refine(f0, lags, vals, info["margin"])
    info["O"], info["path"] = O, path
    return f0, conf


# ------------------------------------------------------------------------------------------ synthetic fixture
def tone(f0_track: np.ndarray, rng, amp=0.3, harmonics=(1.0, 0.6, 0.4, 0.25, 0.15, 0.1)) -> np.ndarray:
    """A harmonic tone whose fundamental follows f0_track (Hz per sample; 0 = silence there)."""
    ph = 2.0 * np.pi * np.cumsum(f0_track) / FS + rng.uniform(0, 2 * np.pi)
    x = np.zeros_like(f0_track)
    for k, a in enumerate(harmonics, 1):
        x += a * np.sin(k * ph) * (k * f0_track < FS / 2)
    return amp * x * (f0_track > 0)


TONES = (90.0, 220.0, 600.0)
EDGES = (1, 159, 160, 161, 2048)


def synth_items(seed: int = 0) -> dict:
    """name -> (float32 audio at 16 kHz, true F0 per sample, 0 where unvoiced)."""
    rng = np.random.default_rng(seed)
    t = lambda s: np.arange(int(s * FS)) / FS
    items = {}
    for f in TONES:
        items[f"tone_{int(f)}"] = np.full(int(0.3 * FS) + int(rng.integers(0, 160)), f)
    items["glide"] = 200.0 * 1.3 ** (t(0.8) / 0.8)
    items["vibrato"] = 300.0 * 2.0 ** (0.5 / 12 * np.sin(2 * np.pi * 5.5 * t(0.6)))
    out = {k: (tone(tr, rng), tr) for k, tr in items.items()}
    tr = np.full(int(0.3 * FS) + 31, 180.0)
    out["second_harmonic"] = (tone(tr, rng, harmonics=(0.3, 1.0, 0.2)), tr)
    n = int(0.2 * FS) + 13
    out["noise"] = (0.3 * rng.standard_normal(n), np.zeros(n))
    out["silence"] = (np.zeros(int(0.1 * FS) + 7), np.zeros(int(0.1 * FS) + 7))
    tr = np.full(int(0.3 * FS) + 57, 250.0)
    out["quiet"] = (tone(tr, rng, amp=0.004), np.zeros_like(tr))     # RMS under 0.01: every frame unvoiced
    for n in EDGES:
        tr = np.full(n, 300.0)
        out[f"edge_{n}"] = (tone(tr, rng) + 1e-3 * rng.standard_normal(n), np.zeros(n))
    return {k: (x.astype(np.float32), tr) for k, (x, tr) in out.items()}


def frame_truth(true_track: np.ndarray, inside_s: float = 0.03) -> tuple:
    """The true F0 at each frame centre and the frames whose centre lies at least `inside_s` inside a voiced run of
    the track, counted from the clip's edges too."""
    n = true_track.shape[0]
    c = np.arange(n_frames(n)) * HOP
    voiced = true_track > 0
    m = int(inside_s * FS)
    ok = np.array([i - m >= 0 and i + m < n and voiced[i - m:i + m + 1].all() for i in c])
    return true_track[np.minimum(c, n - 1)], ok


FIELDS = ("cmndf", "O", "path", "f0", "conf", "margin")


def make_golden(path: str = GOLDEN) -> None:
    arrs = {}
    for k, (x, _) in synth_items().items():
        info = {}
        f0, conf = pyin(x, info)
        arrs[f"{k}/x"] = x
        arrs[f"{k}/cmndf"] = info["cmndf"].T.copy()          # [321, M]
        arrs[f"{k}/O"] = info["O"]
        arrs[f"{k}/path"] = info["path"].astype(np.int32)
        arrs[f"{k}/f0"], arrs[f"{k}/conf"], arrs[f"{k}/margin"] = f0, conf, info["margin"]
    np.savez_compressed(path, **arrs)


# margin: per frame, the smallest gap(a, b) = |a - b| / max(1, |a|, |b|) over the values its decisions compare:
# neighbouring CMNDF values (the strict minima), each minimum and threshold, the two smallest CMNDF values where the
# absolute minimum is taken, the two nearest quantisation distances (cents), each refinement distance and the 10-cent
# tolerance, the RMS and 0.01.  One unit for all of them: relative above 1, absolute below.


def load_golden(path: str = GOLDEN) -> dict:
    """name -> {"x": audio, "cmndf": [321, M], "O": [1036, M], "path", "f0", "conf", "margin": [M]}."""
    z = np.load(path)
    out = {}
    for key in z.files:
        name, field = key.split("/")
        out.setdefault(name, {})[field] = z[key]
    return out


if __name__ == "__main__":
    make_golden()
    print("wrote", GOLDEN, os.path.getsize(GOLDEN), "bytes")
