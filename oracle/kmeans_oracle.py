"""IVF training oracle (TEST INFRASTRUCTURE): a numpy restatement of what faiss 1.7.4 does for the reference's
`svc_train_retrieval.py` (`IVF{nlist},Flat` train + add through feature_retrieval/index.py:122-154), which cannot
run here because faiss is not installed.

* `assign`: faiss's fp32 BLAS distance |x|^2 + |c|^2 - 2 x.c clamped at 0, arg-min to the first (lowest) centroid.
* `kmeans_step`: assign, then each centroid as the fp32 sum of its rows in ascending row order (`np.add.at` in float32)
  times float32 1 / count; empty clusters keep their centroid.
* `kmeans` / `train_ivf_flat`: faiss's Clustering::train (sample, initial rows, niter steps, split_clusters) and
  IndexIVF::add, drawing from the same `numpy.random.default_rng(seed)` stream as whisper_vits_svc_b200.retrieval_train,
  so both start from the same rows and take the same split decisions where their counts agree.
* `import_train_retrieval`: the UNMODIFIED reference `svc_train_retrieval.py` and `feature_retrieval/` behind a stub
  `faiss` that records the `index_factory` string, the `train` and `add` matrices and the `write_index` path, and a
  stub `MiniBatchKMeans` that records its arguments.
"""
from __future__ import annotations

import importlib
import sys

import numpy as np

from oracle.retrieval_oracle import METRIC_L2, _module

F32 = np.float32
UP, DOWN = F32(1 + 1 / 1024), F32(1 - 1 / 1024)


def assign(x: np.ndarray, c: np.ndarray, block: int = 4096):
    """-> (assign [n] int64, dist [n] float32) with faiss's formula in fp32.  Equal centroids (duplicate initial rows)
    get equal distances, so a tie goes to the first of them."""
    x = np.asarray(x, F32)
    c, inv = np.unique(np.asarray(c, F32), axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    cn = (c * c).sum(1, dtype=F32)
    a = np.empty(len(x), np.int64)
    dist = np.empty(len(x), F32)
    for r in range(0, len(x), block):
        xb = x[r:r + block]
        dis = (xb * xb).sum(1, dtype=F32)[:, None] + cn[None, :] - F32(2) * (xb @ c.T)
        dis = np.maximum(dis, F32(0))[:, inv]
        a[r:r + block] = np.argmin(dis, 1)
        dist[r:r + block] = dis[np.arange(len(xb)), a[r:r + block]]
    return a, dist


def centroids_from(x: np.ndarray, a: np.ndarray, c: np.ndarray):
    """faiss compute_centroids: -> (centroids [k, d], counts [k]); empty clusters keep c's row."""
    k = c.shape[0]
    sums = np.zeros(c.shape, F32)
    np.add.at(sums, a, np.asarray(x, F32))       # row by row in ascending order, fp32
    counts = np.bincount(a, minlength=k)
    out = np.array(c, F32, copy=True)
    nz = counts > 0
    out[nz] = sums[nz] * (F32(1) / counts[nz].astype(F32))[:, None]
    return out, counts


def kmeans_step(x, c):
    """-> (assign, dist, new centroids, counts)."""
    a, dist = assign(x, c)
    new, counts = centroids_from(x, a, c)
    return a, dist, new, counts


def split_plan(hassign: np.ndarray, n: int, rng):
    """faiss split_clusters' choice on float32 counts (updated in place), one float32 draw per candidate, a cycle of k
    at a time (the stream retrieval_train.split_plan draws)."""
    k = hassign.shape[0]
    pairs = []
    for ci in np.flatnonzero(hassign == 0):
        while True:
            p = ((hassign.astype(np.float64) - 1.0) / np.float64(F32(n - k))).astype(F32)
            hit = np.flatnonzero(rng.random(k, dtype=F32) < p)
            if hit.size:
                cj = int(hit[0])
                break
        pairs.append((int(ci), cj))
        hassign[ci] = hassign[cj] / F32(2)
        hassign[cj] -= hassign[ci]
    return pairs


def apply_splits(c: np.ndarray, pairs) -> None:
    even = np.arange(c.shape[1]) % 2 == 0
    for ci, cj in pairs:
        v = c[cj].copy()
        c[ci] = np.where(even, v * UP, v * DOWN)
        c[cj] = np.where(even, v * DOWN, v * UP)


def kmeans(x, k: int, niter: int = 10, seed: int = 1234, max_points_per_centroid: int | None = 256):
    """faiss Clustering::train -> (centroids, {"obj": [...], "nsplit": [...]})."""
    x = np.asarray(x, F32)
    n = len(x)
    rng = np.random.default_rng(seed)
    if max_points_per_centroid and n > max_points_per_centroid * k:
        x = x[rng.permutation(n)[:max_points_per_centroid * k]]
        n = len(x)
    stats = {"obj": [], "nsplit": []}
    if n == k:
        return x.copy(), stats
    c = x[rng.permutation(n)[:k]].copy()
    for _ in range(niter):
        a, dist, c, counts = kmeans_step(x, c)
        stats["obj"].append(float(dist.astype(np.float64).sum()))
        pairs = split_plan(counts.astype(F32), n, rng)
        apply_splits(c, pairs)
        stats["nsplit"].append(len(pairs))
    return c, stats


def train_ivf_flat(x, nlist: int, niter: int = 10, seed: int = 1234):
    """-> retrieval.IVFFlat: the trained centroids, row i added to its nearest list with id i (lists ascending)."""
    from oracle.retrieval_oracle import from_parts
    x = np.asarray(x, F32)
    c, _ = kmeans(x, nlist, niter, seed)
    a, _ = assign(x, c)
    lists = []
    for lst in range(nlist):
        ids = np.flatnonzero(a == lst)
        lists.append((x[ids], ids.astype(np.int64)))
    return from_parts(c, lists)


# ------------------------------------------------------------------------------------------------ the reference
def import_train_retrieval(monkeypatch):
    """Import the reference's svc_train_retrieval.py and feature_retrieval/ with stubs; pytest's monkeypatch removes
    them (and the imported modules) from sys.modules after the test.  -> (svc_train_retrieval module, record) where
    record holds lists "factory" ((d, string, metric)), "train", "add" (matrices), "write" (paths) and "mbk"
    (MiniBatchKMeans keyword arguments).  The stub MiniBatchKMeans returns the first n_clusters rows as its centres."""
    from oracle import ref_import
    ref_import._ensure_path()
    rec = {"factory": [], "train": [], "add": [], "write": [], "mbk": []}
    faiss = _module("faiss")

    class Index:
        pass

    class IndexIVF(Index):
        def __init__(self, d, nlist, metric):
            self.d, self.nlist, self.metric_type, self.nprobe, self.is_trained = d, nlist, metric, 1, False

        def train(self, x):
            rec["train"].append(np.array(x, copy=True))
            self.is_trained = True

        def add(self, x):
            rec["add"].append(np.array(x, copy=True))

    def index_factory(d, s, metric=METRIC_L2):
        rec["factory"].append((d, s, metric))
        return IndexIVF(d, int(s[3:s.index(",")]), metric)

    def write_index(index, path):
        rec["write"].append(str(path))
        with open(path, "wb") as f:
            f.write(b"stub")

    faiss.METRIC_L2, faiss.METRIC_INNER_PRODUCT = METRIC_L2, 0
    faiss.Index, faiss.IndexIVF = Index, IndexIVF
    faiss.index_factory, faiss.extract_index_ivf, faiss.write_index = index_factory, (lambda ix: ix), write_index
    monkeypatch.setitem(sys.modules, "faiss", faiss)
    tq = _module("tqdm")
    tq.tqdm = lambda it, total=None: it
    monkeypatch.setitem(sys.modules, "tqdm", tq)
    try:
        import sklearn.cluster  # noqa: F401
    except ImportError:
        for name in ("sklearn", "sklearn.cluster"):
            m = _module(name)
            m.MiniBatchKMeans = None
            monkeypatch.setitem(sys.modules, name, m)
    mods = lambda: [n for n in sys.modules if n == "svc_train_retrieval" or n == "feature_retrieval" or  # noqa: E731
                    n.startswith("feature_retrieval.")]
    for name in mods():
        monkeypatch.delitem(sys.modules, name)   # bound to an earlier stub
    stm = importlib.import_module("svc_train_retrieval")
    for name in mods():
        monkeypatch.setitem(sys.modules, name, sys.modules[name])

    class MiniBatchKMeans:
        def __init__(self, **kw):
            rec["mbk"].append(dict(kw))
            self.n_clusters = kw["n_clusters"]

        def fit(self, x):
            self.cluster_centers_ = np.array(x[:self.n_clusters], copy=True)
            return self

    monkeypatch.setattr(sys.modules["feature_retrieval.transform"], "MiniBatchKMeans", MiniBatchKMeans)
    return stm, rec
