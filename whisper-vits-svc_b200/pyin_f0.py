"""pYIN F0 on the H100 path: libf0's probabilistic YIN tracker (`pitch/core/pyin.py:pyin`) at 16 kHz, a 2048-sample
window, a 160-sample hop and 50-1000 Hz, its other parameters at libf0's defaults.  The wrapper `compute_f0_pyin` and
these parameters are this project's choice: no command of the reference calls pyin.  The 160-sample hop gives the
n // 160 + 1 values at 10 ms that WORLD writes and a pitch CSV holds, and 50-1000 Hz is the CREPE wrappers' range.

The CMNDF, the probabilistic thresholding, the HMM's Viterbi and the refinement run on the device in fp64
(`svcb_pyin_f0_ragged`, csrc/pyin_f0_api.cu).  The host computes the tables they read (thresholds, Beta weights,
F_axis, the transition band) with the reference's own numpy and scipy expressions, once per Extractor.  The output is
float64, 0 for unvoiced frames, not rounded.  No CPU fallback: a CUDA (sm_90a) device is required.

Audio is read as `praat_f0.py` reads it: `hubert_infer.load_audio(path, 16000)`, .wav only, resampled with
`resample_poly` where the file is not at 16 kHz."""
from __future__ import annotations

import functools
import math
import operator
from typing import List, Sequence

import numpy as np
import torch

from . import _lib

SAMPLE_RATE = 16000
HOP = 160
F_MIN = 50.0
F_MAX = 1000.0
BINS = 518                 # int(log2(1000 / 50) * 1200 / 10)
STATES = 2 * BINS          # voiced, then unvoiced
LAGS = 321                 # CMNDF values per frame (lags 0 .. ceil(16000 / 50))
MIN_SAMPLES = 1
BAND = 12
TAB_THR, TAB_BETA, TAB_FAXIS, TAB_BIDX, TAB_BLOG, TAB_DOUBLES = 0, 99, 198, 716, 13148, 25580   # svcb.h SVCB_PYIN_TAB_*


def frames_of(n: int) -> int:
    """Frames of n samples: n // 160 + 1."""
    return int(n) // HOP + 1


def f_axis() -> np.ndarray:
    return F_MIN * np.power(2, np.arange(BINS) * 10 / 1200)


def tables() -> np.ndarray:
    """The device table (svcb.h SVCB_PYIN_TAB_*), float64, each entry as pyin() computes it."""
    from scipy.special import beta, comb
    from scipy.stats import triang
    thr = np.arange(0.01, 1, 0.01)
    i = np.arange(len(thr))
    bd = comb(len(thr), i) * beta(i + 1, len(thr) - i + 18) / beta(1, 18)
    ms = 5
    tri = triang.pdf(np.arange(-ms, ms + 1), 0.5, scale=2 * ms, loc=-ms)
    # compute_transition_matrix: within each half, state k moves to k - 5 .. k + 5 with 0.99 tri; a row the half's edge
    # cuts short is divided by the sum of the taps it keeps, which numba adds with one accumulator in ascending order
    A = np.zeros((STATES, STATES))
    for half in (0, BINS):
        for k in range(BINS):
            lo, hi = max(0, k - ms), min(BINS, k + ms + 1)
            taps = tri[lo - k + ms:hi - k + ms]
            row = 0.99 * taps
            if hi - lo < 2 * ms + 1:
                row = row / functools.reduce(operator.add, taps.tolist(), 0.0)
            A[half + k, half + lo:half + hi] = row
    k = np.arange(BINS)
    A[k, k + BINS] = 1 - 0.99                 # voiced <-> unvoiced twin
    A[k + BINS, k] = 1 - 0.99
    tiny = np.finfo(0.).tiny
    idx = np.full((STATES, BAND), -1.0)
    lg = np.full((STATES, BAND), -np.inf)
    for s in range(STATES):
        k = np.flatnonzero(A[:, s] > 0)       # the triangle's zero end points are off the band: log(tiny) either way
        idx[s, :k.shape[0]] = k
        lg[s, :k.shape[0]] = [math.log(a + tiny) for a in A[k, s]]   # the C library's log, as numba's
    tab = np.concatenate([thr, bd, f_axis(), idx.reshape(-1), lg.reshape(-1)])
    assert tab.shape == (TAB_DOUBLES,)
    return tab


class Extractor:
    """One device, the uploaded table and a grow-only workspace for `svcb_pyin_f0_ragged`.  `close()` frees both."""

    def __init__(self, device="cuda"):
        self.device = _lib.cuda_device(device)
        self.tab = torch.from_numpy(tables()).to(self.device)
        self._ws = None

    def workspace(self, nbytes: int) -> torch.Tensor:
        if self._ws is None or self._ws.numel() < nbytes:
            self._ws = None
            self._ws = torch.empty(int(nbytes), dtype=torch.uint8, device=self.device)
        return self._ws

    def close(self) -> None:
        self._ws = None
        self.tab = None

    @torch.no_grad()
    def raw(self, clips: Sequence, taps: bool = False):
        """Float clips at 16 kHz (each >= 1 sample) -> each one's (f0, conf), float64 per 10 ms frame on the device.
        With taps, also each one's CMNDF [321, frames], observations [1036, frames] (float64) and path (int32)."""
        if not clips:
            return []
        flat, so = _lib.ragged(clips, self.device)
        lens = [so[b + 1] - so[b] for b in range(len(so) - 1)]
        fo = _lib.offsets(frames_of(n) for n in lens)
        f0 = torch.empty(fo[-1], dtype=torch.float64, device=self.device)
        conf = torch.empty_like(f0)
        cm = obs = path = None
        if taps:
            cm = torch.empty(LAGS * fo[-1], dtype=torch.float64, device=self.device)
            obs = torch.empty(STATES * fo[-1], dtype=torch.float64, device=self.device)
            path = torch.empty(fo[-1], dtype=torch.int32, device=self.device)
        ptr = lambda t: t.data_ptr() if t is not None else None
        ws = self.workspace(_lib.load().svcb_pyin_f0_workspace_bytes(so[-1] - so[0], len(lens)))
        _lib.call("pyin_f0_ragged", flat.data_ptr(), so, len(lens), self.tab.data_ptr(), f0.data_ptr(),
                  conf.data_ptr(), ptr(cm), ptr(obs), ptr(path), ws.data_ptr(), ws.numel(), device=self.device)
        f, c = _lib.split(f0, fo), _lib.split(conf, fo)
        if not taps:
            return list(zip(f, c))
        F = [fo[b + 1] - fo[b] for b in range(len(lens))]
        return [(f[b], c[b], cm[LAGS * fo[b]:LAGS * fo[b + 1]].view(LAGS, F[b]),
                 obs[STATES * fo[b]:STATES * fo[b + 1]].view(STATES, F[b]), path[fo[b]:fo[b + 1]])
                for b in range(len(lens))]

    def f0_batch(self, clips: Sequence) -> List[np.ndarray]:
        """Float clips at 16 kHz -> each one's float64 pYIN F0 (n // 160 + 1 values, 0 where unvoiced)."""
        return [f.cpu().numpy() for f, _ in self.raw(clips)]


def f0_batch(clips: Sequence, device="cuda") -> List[np.ndarray]:
    """Float clips at 16 kHz -> the float64 pYIN F0 of each; one device call."""
    ex = Extractor(device)
    try:
        return ex.f0_batch(clips)
    finally:
        ex.close()


def pyin(x, device="cuda"):
    """libf0's pyin(x, Fs=16000, N=2048, H=160, F_min=50, F_max=1000) on the device -> (f0, t, conf) as numpy."""
    ex = Extractor(device)
    try:
        f, c = ex.raw([x])[0]
    finally:
        ex.close()
    f = f.cpu().numpy()
    return f, np.arange(f.shape[0]) * HOP / SAMPLE_RATE, c.cpu().numpy()


def dp_paths(obs: Sequence, device="cuda") -> List[np.ndarray]:
    """The device's Viterbi and trace back alone on given observations ([1036, frames] float64 each) -> each one's
    path (int32 states)."""
    dev = _lib.cuda_device(device)
    if not obs:
        return []
    fo = _lib.offsets(o.shape[1] for o in obs)
    flat = torch.cat([torch.as_tensor(o, dtype=torch.float64).reshape(-1) for o in obs]).to(dev)
    tab = torch.from_numpy(tables()).to(dev)
    path = torch.empty(fo[-1], dtype=torch.int32, device=dev)
    ws = torch.empty(max(1, _lib.load().svcb_pyin_dp_workspace_bytes(fo[-1])), dtype=torch.uint8, device=dev)
    _lib.call("pyin_dp_ragged", flat.data_ptr(), fo, len(obs), tab.data_ptr(), path.data_ptr(), ws.data_ptr(),
              ws.numel(), device=dev)
    return [p.cpu().numpy() for p in _lib.split(path, fo)]


def compute_f0_pyin(path, device="cuda") -> np.ndarray:
    """The file read at 16 kHz (`hubert_infer.load_audio`) -> the `f0` of pyin(audio, Fs=16000, N=2048, H=160,
    F_min=50.0, F_max=1000.0), float64."""
    from . import hubert_infer
    audio = hubert_infer.load_audio(path, SAMPLE_RATE)
    return f0_batch([audio], device)[0]
