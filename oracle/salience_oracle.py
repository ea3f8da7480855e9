"""Salience-based F0 (the reference's pitch/inference.py:compute_f0_salience: libf0's `salience()` at Fs=16000, N=2048,
H=320, F_min=45, F_max=1760, defaults otherwise), restated in numpy.

`dtype` picks the precision of the STFT the rest of the analysis reads:
* np.float32 reproduces the reference: librosa's stft of float32 audio returns complex64, so the phase angles and the
  power |X|^2 are float32 there; everything after them is float64 (the reference's arithmetic).
* np.float64 is the device's contract (csrc/salience_f0_api.cu): every value in fp64.

The steps, each as the device computes it:
1. STFT: centred, 1024 zeros on each side, periodic Hann of 2048 (scipy's get_window), n // 320 + 1 frames.
2. Instantaneous frequency per bin k and frame t >= 1 from the phase advance since frame t - 1, heterodyned by the bin
   centre and wrapped to [-pi, pi] with round-half-to-even; frame 0 takes frame 1's values.  Bins whose frequency is in
   [45, 1760) add |X|^2 into log-frequency bin floor(120 log2(f / 45) + 0.5), in ascending k order.  636 bins.
3. Smoothing along frequency with np.hanning(11), zeros outside.
4. Threshold: an element is kept while v / max + eps32 < 1, max over the whole item (gamma = 0: 20 log10(.) < 0).  This
   clears the item's largest element; a silent item gives 0 / 0 and clears everything.
5. Harmonic summation: Z[i] = sum_j w[j] Y[i + j - 4] over the 641-tap weighting vector, which holds a cos^2 window of
   11 taps scaled by 0.9^idx at offset round(120 log2 h), h = 1 .. 10.  The -4 is scipy's correlate1d at the
   reference's origin, -641 // 2 + 5: the window centred at offset + 5 reads bin i + offset + 1.  Then step 4 on Z.
6. DP: D[b, n] = max_b' (T[b, b'] + D[b', n - 1]) + log(Z[b, n] + eps32), T = log(1 + eps32) within 5 bins and
   log(0.01 + eps32) beyond; the first index of the maximum; backtracking from the first argmax of the last column.
7. F0 = 45 * 2 ** (b * 10 / 1200) of the path's bins.

compute_f0_salience adds np.repeat(f0, 2) and a centred moving average over 3 (np.convolve, 'same').

`python oracle/salience_oracle.py` writes tests/golden/salience_synth.npz.
"""
from __future__ import annotations

import os

import numpy as np
import scipy.signal

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "salience_synth.npz")

FS = 16000
N_FFT = 2048
HOP = 320
F_MIN = 45.0
F_MAX = 1760.0
R = 10.0
NUM_HARM = 10
SMOOTH_LEN = 11
ALPHA = 0.9
TOL = 5
SCORE_LOW = 0.01
SCORE_HIGH = 1.0
EPS32 = float(np.finfo(np.float32).eps)
B = int(np.floor(1200 / R * np.log2(F_MAX / F_MIN) + 0.5)) + 1      # 636
MIN_SAMPLES = HOP                                                   # two frames: the phase advance needs a pair
HARM_OFFSETS = np.round(np.log2(np.arange(1, NUM_HARM + 1)) * 1200 / R).astype(int)
CORR_SHIFT = -4                                                     # Z[i] reads Y[i + j + CORR_SHIFT]


def n_frames(n: int) -> int:
    return int(n) // HOP + 1


def bin_hz() -> np.ndarray:
    """The centre frequency of each of the B bins."""
    return F_MIN * np.power(2, np.arange(B) * R / 1200)


def window() -> np.ndarray:
    return scipy.signal.get_window("hann", N_FFT, fftbins=True)


def stft(x, dtype=np.float64) -> np.ndarray:
    """[1025, n // 320 + 1] spectrum of float audio; complex128, or rounded to complex64 for dtype=np.float32."""
    x = np.asarray(x, np.float64).reshape(-1)
    xp = np.concatenate([np.zeros(N_FFT // 2), x, np.zeros(N_FFT // 2)])
    F = n_frames(x.shape[0])
    idx = np.arange(F)[:, None] * HOP + np.arange(N_FFT)[None, :]
    X = np.fft.rfft(xp[idx] * window()[None, :], axis=1).T
    return X.astype(np.complex64) if dtype == np.float32 else X


def inst_freq(X: np.ndarray) -> np.ndarray:
    """[K, F] instantaneous frequency in Hz (float64) of each bin and frame; frame 0 repeats frame 1."""
    k = np.arange(X.shape[0], dtype=np.float64)[:, None]
    omega = 2 * np.pi * k / N_FFT
    ang = np.angle(X)
    dphi = (ang[:, 1:] - ang[:, :-1]) - omega * HOP      # float32 angle differences stay float32 until here
    dphi = dphi - 2 * np.pi * (np.around(dphi / (2 * np.pi) + 1) - 1)
    f = (omega + dphi / HOP) * FS / (2 * np.pi)
    return np.concatenate([f[:, :1], f], axis=1)


def bin_index(f: np.ndarray) -> np.ndarray:
    """Log-frequency bin of each frequency, B where it lies outside [45, 1760)."""
    f = np.asarray(f, np.float64)
    inside = (f >= F_MIN) & (f < F_MAX)
    with np.errstate(divide="ignore", invalid="ignore"):
        b = np.floor(1200 / R * np.log2(np.where(inside, f, F_MIN) / F_MIN) + 0.5).astype(np.int64)
    return np.where(inside, b, B)


def binned(X: np.ndarray, info: dict | None = None) -> np.ndarray:
    """[B, F] float64 log-frequency spectrogram: |X|^2 added into the bins of the instantaneous frequencies, per frame
    in ascending bin-k order."""
    f = inst_freq(X)
    bins = bin_index(f)
    P = np.abs(X) ** 2
    Y = np.zeros((B + 1, X.shape[1]))
    for t in range(X.shape[1]):
        np.add.at(Y[:, t], bins[:, t], P[:, t])
    if info is not None:
        info["inst_f"] = f
    return Y[:B]


def smooth(Y: np.ndarray) -> np.ndarray:
    """Along frequency with np.hanning(11), zeros outside."""
    h = np.hanning(SMOOTH_LEN)
    c = SMOOTH_LEN // 2
    Yp = np.pad(Y, ((c, c), (0, 0)))
    out = np.zeros_like(Y)
    for j in range(SMOOTH_LEN):
        out += h[j] * Yp[j:j + Y.shape[0]]
    return out


def threshold(V: np.ndarray) -> np.ndarray:
    """V with every element whose ratio to the whole array's maximum reaches 1 - eps32 cleared (all of it when the
    maximum is 0)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        keep = (V / np.max(V) + EPS32) < 1.0
    return np.where(keep, V, 0.0)


def harmonic_taps() -> np.ndarray:
    """The 641-tap weighting vector of the harmonic summation."""
    half = SMOOTH_LEN // 2
    win = np.cos(np.linspace(-1, 1, 2 * half + 1) * np.pi / 2) ** 2
    w = np.zeros(B + half)
    for idx, h in enumerate(HARM_OFFSETS):
        w[h:h + SMOOTH_LEN] += win * ALPHA ** idx
    return w


def correlate(Y: np.ndarray) -> np.ndarray:
    """Z[i] = sum_j w[j] Y[i + j - 4], zeros outside, j ascending over the non-zero taps."""
    w = harmonic_taps()
    n = Y.shape[0]
    Z = np.zeros_like(Y)
    for j in np.flatnonzero(w):
        s = j + CORR_SHIFT
        lo, hi = max(0, -s), min(n, n - s)
        if lo < hi:
            Z[lo:hi] += w[j] * Y[lo + s:hi + s]
    return Z


def salience_rep(x, dtype=np.float64, info: dict | None = None) -> np.ndarray:
    """[B, F] salience Z of float audio at 16 kHz."""
    Y = binned(stft(x, dtype), info)
    if info is not None:
        info["Y"] = Y
    return threshold(correlate(threshold(smooth(Y))))


def transition_log() -> np.ndarray:
    d = np.abs(np.arange(B)[:, None] - np.arange(B)[None, :])
    return np.log(np.where(d <= TOL, SCORE_HIGH, SCORE_LOW) + EPS32)


def dp(Z: np.ndarray, info: dict | None = None) -> np.ndarray:
    """The path's bin per frame (int64).  info gets each path decision's margin: for frame n < F - 1 the gap between
    the best and the second-best predecessor of the path's bin at n + 1, for the last frame that of the final argmax;
    relative to the best value."""
    T = transition_log()
    Zl = np.log(Z + EPS32)
    nb, F = Z.shape
    D = Zl[:, 0].copy()
    E = np.zeros((F, nb), np.int64)
    S_keep = []
    for n in range(1, F):
        S = T + D[None, :]
        E[n - 1] = np.argmax(S, axis=1)
        D = S[np.arange(nb), E[n - 1]] + Zl[:, n]
        if info is not None:
            S_keep.append(S)
    eta = np.zeros(F, np.int64)
    eta[-1] = int(np.argmax(D))
    for n in range(F - 2, -1, -1):
        eta[n] = E[n, eta[n + 1]]
    if info is not None:
        margin = np.zeros(F)
        margin[-1] = _margin(D)
        for n in range(F - 1):
            margin[n] = _margin(S_keep[n][eta[n + 1]])
        info["margin"] = margin
    return eta


def _margin(v: np.ndarray) -> float:
    top = np.sort(v)[::-1]
    if top.shape[0] < 2:
        return np.inf
    return float((top[0] - top[1]) / max(abs(top[0]), 1e-300))


def path_score(Z: np.ndarray, eta: np.ndarray) -> float:
    """Sum of log(Z + eps32) along the path and the transitions between its bins."""
    T = transition_log()
    Zl = np.log(Z + EPS32)
    s = Zl[eta[0], 0]
    for n in range(1, eta.shape[0]):
        s = s + T[eta[n], eta[n - 1]] + Zl[eta[n], n]
    return float(s)


def salience_f0(x, dtype=np.float64, info: dict | None = None) -> np.ndarray:
    """Unrepeated float64 F0 per 20 ms frame (n // 320 + 1 values) of float audio at 16 kHz, at least 320 samples."""
    x = np.asarray(x).reshape(-1)
    if x.shape[0] < MIN_SAMPLES:
        raise ValueError(f"{x.shape[0]} samples: fewer than {MIN_SAMPLES}, one hop")
    Z = salience_rep(x, dtype, info)
    eta = dp(Z, info)
    if info is not None:
        info["Z"], info["eta"] = Z, eta
    return bin_hz()[eta]


def finish(f0: np.ndarray) -> np.ndarray:
    """compute_f0_salience's host tail: every value twice (20 ms -> 10 ms), then a centred moving average over 3."""
    f0 = np.repeat(f0, 2, -1)
    return np.convolve(f0, np.ones((3,)) / 3, mode="same")


def compute_f0_salience(x, dtype=np.float64) -> np.ndarray:
    return finish(salience_f0(x, dtype))


# ------------------------------------------------------------------------------------------ synthetic fixture
def tone(f0_track: np.ndarray, rng, amp=0.3, harmonics=(1.0, 0.6, 0.4, 0.25, 0.15, 0.1)) -> np.ndarray:
    """A harmonic tone whose fundamental follows f0_track (Hz per sample; 0 = silence there)."""
    ph = 2.0 * np.pi * np.cumsum(f0_track) / FS + rng.uniform(0, 2 * np.pi)
    x = np.zeros_like(f0_track)
    for k, a in enumerate(harmonics, 1):
        x += a * np.sin(k * ph) * (k * f0_track < FS / 2)
    return amp * x * (f0_track > 0)


TONES = (80.0, 130.0, 220.0, 370.0, 600.0, 1000.0)
EDGES = (319, 320, 321)


def synth_items(seed: int = 0) -> dict:
    """name -> (float32 audio at 16 kHz, true F0 per sample, 0 where unvoiced)."""
    rng = np.random.default_rng(seed)
    t = lambda s: np.arange(int(s * FS)) / FS
    items = {}
    for f in TONES:
        n = int(0.5 * FS) + int(rng.integers(0, 320))
        items[f"tone_{int(f)}"] = np.full(n, f)
    items["glide"] = 200.0 * 1.5 ** (t(2.0) / 2.0)
    items["vibrato"] = 300.0 * 2.0 ** (0.5 / 12 * np.sin(2 * np.pi * 5.5 * t(1.2)))
    out = {k: (tone(tr, rng), tr) for k, tr in items.items()}
    n = int(1.0 * FS) + 77
    melody = np.full(n, 440.0)
    chord = sum(tone(np.full(n, f), rng, amp=0.5, harmonics=(1.0, 0.3)) for f in (130.8, 164.8, 196.0))
    out["under_chord"] = (tone(melody, rng, amp=0.25) + chord, melody)
    out["noise"] = (0.1 * rng.standard_normal(int(0.6 * FS) + 13), np.zeros(int(0.6 * FS) + 13))
    out["silence"] = (np.zeros(int(0.3 * FS) + 7), np.zeros(int(0.3 * FS) + 7))
    for n in EDGES:
        tr = np.full(n, 300.0)
        out[f"edge_{n}"] = (tone(tr, rng) + 1e-3 * rng.standard_normal(n), tr)
    return {k: (x.astype(np.float32), tr) for k, (x, tr) in out.items()}


def frame_truth(true_track: np.ndarray, inside_s: float = 0.04) -> tuple:
    """The true F0 at each frame centre and the frames whose centre lies at least `inside_s` inside a voiced run of
    the track, counted from the clip's edges too."""
    n = true_track.shape[0]
    c = np.arange(n_frames(n)) * HOP
    voiced = true_track > 0
    m = int(inside_s * FS)
    ok = np.array([i - m >= 0 and i + m < n and voiced[i - m:i + m + 1].all() for i in c])
    return true_track[np.minimum(c, n - 1)], ok


def make_golden(path: str = GOLDEN) -> None:
    arrs = {}
    for k, (x, _) in synth_items().items():
        arrs[f"{k}/x"] = x
        if x.shape[0] < MIN_SAMPLES:
            continue
        for name, dt in (("eta64", np.float64), ("eta32", np.float32)):
            info = {}
            salience_f0(x, dt, info)
            arrs[f"{k}/{name}"] = info["eta"].astype(np.int16)
    np.savez_compressed(path, **arrs)


def load_golden(path: str = GOLDEN) -> dict:
    """name -> {"x": audio, "eta64": path of the fp64 oracle, "eta32": of the float32 one} (no paths below 320
    samples)."""
    z = np.load(path)
    out = {}
    for key in z.files:
        name, field = key.split("/")
        out.setdefault(name, {})[field] = z[key]
    return out


if __name__ == "__main__":
    make_golden()
    print("wrote", GOLDEN, os.path.getsize(GOLDEN), "bytes")
