"""Feature retrieval oracle (TEST INFRASTRUCTURE): a numpy restatement of what the reference's
`FaissRVCRetrievableFeatureIndex.retriv` (feature_retrieval/index.py:57-62,75-94) computes on an `IVF{nlist},Flat`
L2 index through faiss, which is not installed here.

* `search`: faiss's IVF-Flat search — coarse search over the IndexFlatL2 quantizer with faiss's fp32 BLAS formula
  |x|^2 + |c|^2 - 2 x.c (clamped at 0), then the probed lists scanned in stored order with the exact fp32
  sum (x - v)^2, keeping the k smallest (ties: the vector scanned first), `search_and_reconstruct`'s NaN vector
  and label -1 where fewer than k were found.
* `blend_reference`: index.py:80-88 + :61 verbatim in numpy float32 (NaN rows included).
* `blend_defined`: the same, with the degenerate rows the device path defines (zero distances share the weight;
  the blend runs over the neighbours found; none found -> the row unchanged).
* `write_ivf_flat`: emits the faiss 1.7.4 `IndexIVFFlat` byte layout (`full` or `sprs` list sizes) for tests.
* `import_feature_retrieval`: the UNMODIFIED reference classes behind a stub `faiss` whose index answers
  `search_and_reconstruct` from `search` — so the blend half of the goldens is the reference's own code.
* `retrieval_case` / `python -m oracle.retrieval_oracle`: writes tests/golden/retrieval_*.npz (needs the reference).
"""
from __future__ import annotations

import importlib.machinery
import os
import struct
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
METRIC_L2 = 1


# ------------------------------------------------------------------------------------------------ search
def coarse_search(x: np.ndarray, centroids: np.ndarray, nprobe: int) -> np.ndarray:
    """-> [M, min(nprobe, nlist)] list ids, ascending by faiss's fp32 distance, ties to the lower list."""
    x = np.asarray(x, np.float32)
    c = np.asarray(centroids, np.float32)
    xn = (x * x).sum(1, dtype=np.float32)
    cn = (c * c).sum(1, dtype=np.float32)
    dis = xn[:, None] + cn[None, :] - np.float32(2) * (x @ c.T)
    dis = np.maximum(dis, np.float32(0))
    return np.argsort(dis, axis=1, kind="stable")[:, :min(nprobe, c.shape[0])]


def search(ix, x: np.ndarray, k: int, nprobe: int | None = None):
    """-> (dist [M,k] f32, ids [M,k] i64, pos [M,k] row in ix.vectors or -1, vectors [M,k,d] f32 NaN-filled)."""
    x = np.asarray(x, np.float32)
    M, d = x.shape
    probes = coarse_search(x, ix.centroids, ix.nprobe if nprobe is None else nprobe)
    dist = np.full((M, k), np.inf, np.float32)
    ids = np.full((M, k), -1, np.int64)
    pos = np.full((M, k), -1, np.int64)
    vecs = np.full((M, k, d), np.nan, np.float32)
    off = ix.list_offsets
    for m in range(M):
        cand = np.concatenate([np.arange(off[lst], off[lst + 1]) for lst in probes[m]]) if len(probes[m]) else np.zeros(0, np.int64)
        if cand.size == 0:
            continue
        diff = x[m][None, :] - ix.vectors[cand]
        dd = (diff * diff).sum(1, dtype=np.float32)
        sel = np.argsort(dd, kind="stable")[:k]   # stable: scan order breaks ties
        n = sel.size
        dist[m, :n], pos[m, :n] = dd[sel], cand[sel]
        ids[m, :n] = ix.ids[cand[sel]]
        vecs[m, :n] = ix.vectors[cand[sel]]
    return dist, ids, pos, vecs


def knn_float64(ix, x: np.ndarray, k: int):
    """Brute-force kNN in float64 over every vector (ties in stored order): -> (dist, ids)."""
    x = np.asarray(x, np.float64)
    v = ix.vectors.astype(np.float64)
    dd = ((x[:, None, :] - v[None, :, :]) ** 2).sum(-1)
    sel = np.argsort(dd, axis=1, kind="stable")[:, :k]
    return np.take_along_axis(dd, sel, 1), ix.ids[sel]


# ------------------------------------------------------------------------------------------------ blend
def blend_reference(x: np.ndarray, scores: np.ndarray, nearest: np.ndarray, ratio: float) -> np.ndarray:
    """index.py:85-88 and :61, float32 throughout (NaN where the reference produces NaN)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        weight = np.square(1 / scores)
        weight /= weight.sum(axis=1, keepdims=True)
        weight = np.expand_dims(weight, axis=2)
        weighted = np.sum(nearest * weight, axis=1)
        return (1 - ratio) * np.asarray(x, np.float32) + ratio * weighted


def blend_defined(x: np.ndarray, scores: np.ndarray, nearest: np.ndarray, ratio: float) -> np.ndarray:
    """blend_reference with the device path's degenerate rows: zero-distance neighbours share the weight equally,
    otherwise the blend runs over the neighbours found (finite distance), none found -> out = x."""
    x = np.asarray(x, np.float32)
    found = np.isfinite(scores)
    zero = found & (scores == 0)
    with np.errstate(divide="ignore", invalid="ignore"):
        w = np.where(found, np.square(np.float32(1) / np.where(found, scores, np.float32(1))), np.float32(0)).astype(np.float32)
    w = np.where(zero.any(1, keepdims=True), zero.astype(np.float32), w)
    s = np.zeros(x.shape[0], np.float32)
    for j in range(scores.shape[1]):   # the device sums the k weights in rank order
        s = s + w[:, j]
    with np.errstate(divide="ignore", invalid="ignore"):
        w = w / s[:, None]
    blend = np.zeros_like(x)
    for j in range(scores.shape[1]):
        use = (w[:, j] != 0)[:, None]
        blend = np.where(use, blend + w[:, j, None] * np.where(use, nearest[:, j], np.float32(0)), blend)
    out = (1 - ratio) * x + ratio * blend
    return np.where(found.any(1, keepdims=True), out, x).astype(np.float32)


# ------------------------------------------------------------------------------------------------ file writer
def _header(d: int, ntotal: int, metric: int = METRIC_L2) -> bytes:
    return struct.pack("<iqqqBi", d, ntotal, 1 << 20, 1 << 20, 1, metric) + (struct.pack("<f", 0.0) if metric > 1 else b"")


def write_ivf_flat(path, centroids: np.ndarray, lists, nprobe: int = 1, sparse: bool = False, metric: int = METRIC_L2) -> None:
    """faiss 1.7.4 write_index(IndexIVFFlat): lists = [(vectors [n_l, d] f32, ids [n_l] i64)] per centroid."""
    c = np.asarray(centroids, np.float32)
    nlist, d = c.shape
    assert len(lists) == nlist
    ntotal = sum(len(v) for v, _ in lists)
    b = bytearray(b"IwFl" + _header(d, ntotal, metric) + struct.pack("<QQ", nlist, nprobe))
    b += b"IxF2" + _header(d, nlist, metric) + struct.pack("<Q", nlist * d) + c.astype("<f4").tobytes()
    b += struct.pack("<BQ", 0, 0)                                  # direct map: none
    b += b"ilar" + struct.pack("<QQ", nlist, 4 * d)
    sizes = [len(v) for v, _ in lists]
    if sparse:
        pairs = [(i, n) for i, n in enumerate(sizes) if n]
        b += b"sprs" + struct.pack("<Q", 2 * len(pairs)) + b"".join(struct.pack("<QQ", i, n) for i, n in pairs)
    else:
        b += b"full" + struct.pack("<Q", nlist) + struct.pack(f"<{nlist}Q", *sizes)
    for v, ids in lists:
        if len(v):
            b += np.asarray(v, "<f4").tobytes() + np.asarray(ids, "<i8").tobytes()
    with open(path, "wb") as f:
        f.write(bytes(b))


def clustered_index(seed: int, d: int, nlist: int, sizes=None, spread: float = 0.35):
    """A small clustered IVF-Flat index as (centroids, lists): vectors = centroid + noise, ids shuffled."""
    rng = np.random.default_rng(seed)
    cen = rng.standard_normal((nlist, d)).astype(np.float32)
    if sizes is None:
        sizes = rng.integers(3, 14, nlist)
    ntotal = int(np.sum(sizes))
    idp = rng.permutation(ntotal).astype(np.int64)
    lists, o = [], 0
    for lst, n in enumerate(sizes):
        v = (cen[lst] + spread * rng.standard_normal((int(n), d))).astype(np.float32)
        lists.append((v, idp[o:o + int(n)]))
        o += int(n)
    return cen, lists


def from_parts(centroids, lists, nprobe: int = 1):
    """(centroids, lists) -> the reader's IVFFlat, without a file."""
    from whisper_vits_svc_b200.retrieval import IVFFlat
    sizes = [len(v) for v, _ in lists]
    off = np.zeros(len(lists) + 1, np.int64)
    off[1:] = np.cumsum(sizes)
    d = centroids.shape[1]
    vec = np.concatenate([np.asarray(v, np.float32).reshape(-1, d) for v, _ in lists]) if off[-1] else np.zeros((0, d), np.float32)
    ids = np.concatenate([np.asarray(i, np.int64) for _, i in lists]) if off[-1] else np.zeros(0, np.int64)
    return IVFFlat(d=d, nlist=len(lists), nprobe=nprobe, metric=METRIC_L2, centroids=np.asarray(centroids, np.float32),
                   list_offsets=off, vectors=vec, ids=ids)


# ------------------------------------------------------------------------------------------------ the reference
def _module(name):
    m = types.ModuleType(name)
    m.__spec__ = importlib.machinery.ModuleSpec(name, loader=None)
    return m


def import_feature_retrieval(ix_by_path: dict, monkeypatch=None):
    """Import the reference's feature_retrieval/ with a stub `faiss` in sys.modules.  `faiss.read_index(path)` returns an
    index over ix_by_path[path] (an IVFFlat) whose `search_and_reconstruct` is `search` above.  Pass pytest's
    `monkeypatch` so the stubs and the imported modules leave sys.modules after the test.
    -> (feature_retrieval.index, feature_retrieval.retrieval)."""
    from oracle import ref_import
    ref_import._ensure_path()
    put = monkeypatch.setitem if monkeypatch else (lambda mp, k, v: mp.__setitem__(k, v))
    drop = monkeypatch.delitem if monkeypatch else (lambda mp, k: mp.__delitem__(k))
    faiss = _module("faiss")

    class Index:
        pass

    class IndexIVF(Index):
        pass

    class _StubIVFFlat(IndexIVF):
        def __init__(self, ix):
            self.ix, self.metric_type, self.d, self.nprobe = ix, ix.metric, ix.d, ix.nprobe

        def search_and_reconstruct(self, x, k):
            dist, ids, _, vecs = search(self.ix, x, k)
            return dist, ids, vecs

    faiss.METRIC_L2 = METRIC_L2
    faiss.METRIC_INNER_PRODUCT = 0
    faiss.Index, faiss.IndexIVF = Index, IndexIVF
    faiss.read_index = lambda p: _StubIVFFlat(ix_by_path[str(p)])
    put(sys.modules, "faiss", faiss)
    for name in ("sklearn", "sklearn.cluster", "tqdm"):   # imported by transform.py / index.py; unused by retriv
        try:
            __import__(name)
        except ImportError:
            m = _module(name)
            m.MiniBatchKMeans = m.tqdm = None
            put(sys.modules, name, m)
    for name in [n for n in sys.modules if n == "feature_retrieval" or n.startswith("feature_retrieval.")]:
        drop(sys.modules, name)   # bound to an earlier stub
    import importlib
    fr_index = importlib.import_module("feature_retrieval.index")
    fr_retrieval = importlib.import_module("feature_retrieval.retrieval")
    for name in [n for n in sys.modules if n == "feature_retrieval" or n.startswith("feature_retrieval.")]:
        put(sys.modules, name, sys.modules[name])   # so monkeypatch removes them again
    return fr_index, fr_retrieval


# ------------------------------------------------------------------------------------------------ goldens
RETRIEVAL_CASES = {   # name: (seed, d, nlist, queries)
    "retrieval_d256_n37": (41, 256, 37, 128),
    "retrieval_d1280_n11": (42, 1280, 11, 32),
}
GOLDEN_RATIO, GOLDEN_K = 0.5, 3


def _grid(a):
    """Round to multiples of 1/64: the stored index and queries then compress to a fraction of their float32 size
    (the blended output, a weighted sum, does not, so it bounds the number of queries kept)."""
    return (np.round(np.asarray(a, np.float64) * 64) / 64).astype(np.float32)


def golden_parts(name):
    """The case's index and queries: some lists shorter than k, one empty; queries near random lists, some equal to an
    index vector (distance 0), some at a centroid, a few next to the empty list's centroid (nothing found)."""
    seed, d, nlist, M = RETRIEVAL_CASES[name]
    rng = np.random.default_rng(seed + 1000)
    sizes = rng.integers(3, 8, nlist)
    sizes[[1, 4, 7]] = [1, 2, 0]        # two lists shorter than k = 3, list 7 empty
    cen, lists = clustered_index(seed, d, nlist, sizes)
    cen, lists = _grid(cen), [(_grid(v), i) for v, i in lists]
    ix = from_parts(cen, lists)
    q = cen[rng.integers(0, nlist, M)] + 0.4 * rng.standard_normal((M, d))
    q[:8] = ix.vectors[rng.integers(0, ix.ntotal, 8)]             # exact duplicates
    q[8:10] = cen[[2, 3]]                                         # at a centroid
    q[10:13] = cen[7] + 0.05 * rng.standard_normal((3, d))        # probes only the empty list
    q[13:16] = cen[[1, 4, 4]] + 0.05 * rng.standard_normal((3, d))   # short lists
    return ix, _grid(q)


def retrieval_case(name):
    import tempfile
    ix, q = golden_parts(name)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "x.index")
        fr_index, _ = import_feature_retrieval({path: ix})
        ref = fr_index.load_retrieve_index(filepath=path, ratio=GOLDEN_RATIO, n_nearest_vectors=GOLDEN_K)
        out_ref = ref.retriv(q)
    dist, ids, _, vecs = search(ix, q, GOLDEN_K)
    own = blend_reference(q, dist, vecs, GOLDEN_RATIO)
    assert np.array_equal(np.isnan(own), np.isnan(out_ref)) and np.array_equal(own[~np.isnan(own)], out_ref[~np.isnan(out_ref)])
    np.savez_compressed(os.path.join(GOLDEN, name + ".npz"), centroids=ix.centroids, list_offsets=ix.list_offsets,
                        vectors=ix.vectors, ids=ix.ids, queries=q, ratio=np.float32(GOLDEN_RATIO), k=np.int64(GOLDEN_K),
                        search_dist=dist, search_ids=ids, retriv=out_ref.astype(np.float32))
    print(name, "rows", q.shape[0], "NaN rows in the reference", int(np.isnan(out_ref).any(1).sum()))


def load_golden(name):
    """-> (IVFFlat, npz dict) of a stored case."""
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    from whisper_vits_svc_b200.retrieval import IVFFlat
    ix = IVFFlat(d=g["centroids"].shape[1], nlist=g["centroids"].shape[0], nprobe=1, metric=METRIC_L2,
                 centroids=g["centroids"], list_offsets=g["list_offsets"], vectors=g["vectors"], ids=g["ids"])
    return ix, g


if __name__ == "__main__":
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    for case in RETRIEVAL_CASES:
        retrieval_case(case)
