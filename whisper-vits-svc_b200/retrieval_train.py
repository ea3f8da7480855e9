"""Building IVF-Flat retrieval indexes on the H100 — mirror of the reference's `svc_train_retrieval.py` and
`feature_retrieval/train.py`, `transform.py` and `index.py:122-154`, without faiss or scikit-learn, behind the C ABI
(`svcb_kmeans_*`, csrc/kmeans_api.cu).

The index is what faiss 1.7.4 builds for `IVF{nlist},Flat` with `train` then `add`: Lloyd k-means with faiss's
procedure (sample 256 nlist rows when there are more, nlist distinct random rows as the start, ten iterations of
assign / fp32 ascending-order means / empty-cluster splits), then every row added to the list of its nearest centroid,
with ids 0..n-1 in ascending order inside each list.  The assignment runs on the tensor cores exactly as the search of
`retrieval.py` does, and the final one uses the image and norms `retrieval.pack_ivf` builds for the written index, so a
stored vector is found in the list its own search probes.

Deliberate deviations from the reference:
* random draws (the training sample, the initial rows, the split walk) come from numpy's `default_rng(seed)`, not
  faiss's mt19937, so the centroids are not faiss's bit for bit;
* feature sets above `--compress-features-after` rows are compressed by device Lloyd k-means (`compress_features`) in
  place of scikit-learn's `MiniBatchKMeans`: the same output shape, [n_clusters, d];
* the `*.npy` files are read in sorted path order rather than `rglob` order, so the index is reproducible."""
from __future__ import annotations

import logging
import struct
import time
from pathlib import Path
from typing import Dict, List, Tuple

import numpy as np
import torch

from . import _lib
from .retrieval import METRIC_L2, IVFFlat, pack_centroids

logger = logging.getLogger(__name__)

MIN_POINTS_PER_LIST = 39            # index.py:148: nlist = min(16 sqrt(n), n // 39)
MAX_POINTS_PER_CENTROID = 256       # faiss ClusteringParameters.max_points_per_centroid
SEED = 1234                         # faiss ClusteringParameters.seed


def default_nlist(n: int) -> int:
    """index.py:148: `min(int(16 * np.sqrt(num_vectors)), num_vectors // 39)`."""
    return min(int(16 * np.sqrt(n)), n // MIN_POINTS_PER_LIST)


# ------------------------------------------------------------------------------------------------ device steps
def _workspace(n: int, d: int, k: int, chunk: int, dev) -> torch.Tensor:
    need = int(_lib.load().svcb_kmeans_workspace_bytes(n, d, k, chunk))
    if need == 0:
        raise ValueError(f"k-means shape not supported: n={n} d={d} k={k} (need d % 64 == 0, 64 <= d <= 2048, k >= 1)")
    return torch.empty(need, dtype=torch.uint8, device=dev)


def pack_device(centroids: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """centroids [k, d] fp32 on the device -> (wimg, cnorm) in pack_centroids' layout, built on the device."""
    k, d = centroids.shape
    npad = (k + 255) // 256 * 256
    wimg = torch.empty(npad * 3 * d // 2, dtype=torch.float32, device=centroids.device)
    cnorm = torch.empty(npad, dtype=torch.float32, device=centroids.device)
    _lib.call("kmeans_pack", centroids.data_ptr(), wimg.data_ptr(), cnorm.data_ptr(), k, d, device=centroids.device)
    return wimg, cnorm


def assign(x: torch.Tensor, centroids: torch.Tensor, wimg: torch.Tensor, cnorm: torch.Tensor, chunk: int = 0, ws=None):
    """x [n, d] fp32 on the device -> (assign [n] int32, dist [n] fp32): the nearest of the centroids [k, d] (fp32 on the
    device) through their packed image (wimg, cnorm), and faiss's distance max(|x|^2 + |c|^2 - 2 x.c, 0).
    chunk: rows per pass (0 = the library's default)."""
    k = centroids.shape[0]
    n, d = x.shape
    dev = x.device
    a = torch.empty(n, dtype=torch.int32, device=dev)
    dist = torch.empty(n, dtype=torch.float32, device=dev)
    if ws is None:
        ws = _workspace(n, d, k, chunk, dev)
    _lib.call("kmeans_assign", x.data_ptr(), centroids.data_ptr(), wimg.data_ptr(), cnorm.data_ptr(), a.data_ptr(),
              dist.data_ptr(), n, d, k, chunk, ws.data_ptr(), ws.numel(), device=dev)
    return a, dist


def update(x: torch.Tensor, a: torch.Tensor, k: int, centroids: torch.Tensor | None = None, ws=None):
    """Stable counting sort of the rows by a -> (counts [k], offsets [k + 1], order [n]) int32 on the device; with
    centroids ([k, d], updated in place) each non-empty one becomes the fp32 mean of its rows in ascending order."""
    n, d = x.shape
    dev = x.device
    counts = torch.empty(k, dtype=torch.int32, device=dev)
    offsets = torch.empty(k + 1, dtype=torch.int32, device=dev)
    order = torch.empty(n, dtype=torch.int32, device=dev)
    if ws is None:
        ws = _workspace(n, d, k, 0, dev)
    cptr = None if centroids is None else centroids.data_ptr()
    _lib.call("kmeans_update", x.data_ptr(), a.data_ptr(), cptr, counts.data_ptr(), offsets.data_ptr(),
              order.data_ptr(), n, d, k, ws.data_ptr(), ws.numel(), device=dev)
    return counts, offsets, order


def split(centroids: torch.Tensor, pairs: List[Tuple[int, int]]) -> None:
    """Apply split_plan's (empty, split) pairs to the device centroids in place, in order."""
    if not pairs:
        return
    p = torch.tensor(pairs, dtype=torch.int32).to(centroids.device)
    _lib.call("kmeans_split", centroids.data_ptr(), p.data_ptr(), len(pairs), centroids.shape[1], device=centroids.device)


def split_plan(hassign: np.ndarray, n: int, rng: np.random.Generator) -> List[Tuple[int, int]]:
    """faiss split_clusters' choice, on float32 counts updated in place: for each empty ci in order, walk cj = 0, 1, ...
    cyclically and take the first with r < (count[cj] - 1) / (n - k); then count[ci] = count[cj] / 2 and
    count[cj] -= count[ci].  The walk draws one float32 per candidate a whole cycle at a time."""
    k = hassign.shape[0]
    pairs = []
    for ci in np.flatnonzero(hassign == 0):
        while True:
            p = ((hassign.astype(np.float64) - 1.0) / np.float64(np.float32(n - k))).astype(np.float32)
            hit = np.flatnonzero(rng.random(k, dtype=np.float32) < p)
            if hit.size:
                cj = int(hit[0])
                break
        pairs.append((int(ci), cj))
        hassign[ci] = hassign[cj] / np.float32(2)
        hassign[cj] -= hassign[ci]
    return pairs


def kmeans_step(x: torch.Tensor, centroids: torch.Tensor, chunk: int = 0):
    """One Lloyd iteration on the device from centroids [k, d] (not modified) ->
    (assign, dist, new centroids, counts); empty clusters keep their centroid (the split step replaces them)."""
    k = centroids.shape[0]
    wimg, cnorm = pack_device(centroids)
    a, dist = assign(x, centroids, wimg, cnorm, chunk)
    c = centroids.clone()
    counts, _, _ = update(x, a, k, c)
    return a, dist, c, counts


# ------------------------------------------------------------------------------------------------ training
def _device_rows(x, device) -> torch.Tensor:
    dev = _lib.cuda_device(device)
    t = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32))
    return t.to(dev, torch.float32).contiguous()


def _check_dim(d: int) -> None:
    if d % 64 or not 64 <= d <= 2048:
        raise ValueError(f"feature width {d} is not supported: the index reader needs a multiple of 64 in [64, 2048]")


def kmeans(x, k: int, niter: int = 10, seed: int = SEED, max_points_per_centroid: int | None = MAX_POINTS_PER_CENTROID,
           device="cuda", chunk: int = 0) -> Tuple[np.ndarray, Dict[str, list]]:
    """faiss Clustering::train on the device -> (centroids [k, d] float32, stats).  stats["obj"][i] is the sum of the
    distances of iteration i's assignment, stats["nsplit"][i] the number of empty clusters it split."""
    xd = _device_rows(x, device)
    n, d = xd.shape
    _check_dim(d)
    if not 1 <= k <= n:
        raise ValueError(f"k-means with {k} clusters needs 1 <= k <= the number of rows ({n})")
    rng = np.random.default_rng(seed)
    if max_points_per_centroid and n > max_points_per_centroid * k:
        sel = rng.permutation(n)[:max_points_per_centroid * k]
        logger.debug("k-means: sampling %s of %s rows", sel.size, n)
        xd = xd[torch.from_numpy(sel).to(xd.device)].contiguous()
        n = sel.size
    stats: Dict[str, list] = {"obj": [], "nsplit": []}
    if n == k:   # faiss copies the points
        return xd.cpu().numpy(), stats
    c = xd[torch.from_numpy(rng.permutation(n)[:k]).to(xd.device)].contiguous()
    ws = _workspace(n, d, k, chunk, xd.device)
    for _ in range(niter):
        wimg, cnorm = pack_device(c)
        a, dist = assign(xd, c, wimg, cnorm, chunk, ws)
        counts, _, _ = update(xd, a, k, c, ws)
        hassign = counts.cpu().numpy().astype(np.float32)
        stats["obj"].append(float(dist.cpu().numpy().astype(np.float64).sum()))
        pairs = split_plan(hassign, n, rng)
        split(c, pairs)
        stats["nsplit"].append(len(pairs))
    return c.cpu().numpy(), stats


def train_ivf_flat(x, nlist: int | None = None, niter: int = 10, nprobe: int = 1, device="cuda", seed: int = SEED) -> IVFFlat:
    """`IVF{nlist},Flat` trained and filled as index.py:122-139 does -> retrieval.IVFFlat with ids 0..n-1, each list in
    ascending id order.  nlist defaults to index.py:148's rule."""
    xd = _device_rows(x, device)
    n, d = xd.shape
    _check_dim(d)
    nlist = default_nlist(n) if nlist is None else int(nlist)
    if nlist < 1:
        raise ValueError(f"{n} feature rows give nlist = min(16 sqrt(n), n // 39) = {nlist}: need at least 39 rows")
    centroids, _ = kmeans(xd, nlist, niter, seed, device=xd.device)
    wimg, cnorm = (t.to(xd.device) for t in pack_centroids(centroids))   # exactly the written index's search image
    a, _ = assign(xd, torch.from_numpy(centroids).to(xd.device), wimg, cnorm)
    _, offsets, order = update(xd, a, nlist)
    offsets = offsets.cpu().numpy().astype(np.int64)
    if offsets[-1] != n:
        raise ValueError(f"{n - int(offsets[-1])} rows could not be assigned to a list (non-finite values?)")
    order_d = order.long()
    return IVFFlat(d=d, nlist=nlist, nprobe=nprobe, metric=METRIC_L2, centroids=centroids, list_offsets=offsets,
                   vectors=xd[order_d].cpu().numpy(), ids=order_d.cpu().numpy())


def _check_clusters(n: int, n_clusters: int) -> None:
    if not 1 <= n_clusters <= n:
        raise ValueError(f"cannot compress {n} feature rows to {n_clusters} clusters: n_clusters must be <= the rows "
                         "and >= 1")


def compress_features(x, n_clusters: int, niter: int = 25, device="cuda", seed: int = SEED) -> np.ndarray:
    """In place of transform.py:29-53's MiniBatchKMeans(n_clusters).cluster_centers_: Lloyd k-means over every row on
    the device -> [n_clusters, d] float32."""
    _check_clusters(int(x.shape[0]), n_clusters)
    return kmeans(x, n_clusters, niter, seed, max_points_per_centroid=None, device=device)[0]


# ------------------------------------------------------------------------------------------------ files
def _header(d: int, ntotal: int) -> bytes:
    """write_index_header: d, ntotal, two dummies 1 << 20, is_trained, metric_type."""
    return struct.pack("<iqqqBi", d, ntotal, 1 << 20, 1 << 20, 1, METRIC_L2)


def write_ivf_flat(path, ix: IVFFlat, rewrite: bool = False) -> None:
    """faiss 1.7.4 write_index(IndexIVFFlat): `IwFl`, an `IxF2` quantizer, no direct map, `ilar` lists whose sizes are
    written `full` when more than nlist / 2 lists are non-empty and `sprs` otherwise.  index.py:26-29: an existing file
    raises FileExistsError unless rewrite."""
    path = Path(path)
    if path.exists() and not rewrite:
        raise FileExistsError(f"index already exists by path {path}")
    d, nlist = ix.d, ix.nlist
    sizes = np.diff(ix.list_offsets).astype(np.int64)
    with open(path, "wb") as f:
        f.write(b"IwFl" + _header(d, ix.ntotal) + struct.pack("<QQ", nlist, ix.nprobe))
        f.write(b"IxF2" + _header(d, nlist) + struct.pack("<Q", nlist * d))
        f.write(np.ascontiguousarray(ix.centroids, "<f4").tobytes())
        f.write(struct.pack("<BQ", 0, 0) + b"ilar" + struct.pack("<QQ", nlist, 4 * d))
        nz = np.flatnonzero(sizes)
        if nz.size > nlist // 2:
            f.write(b"full" + struct.pack("<Q", nlist) + sizes.astype("<u8").tobytes())
        else:
            pairs = np.stack([nz, sizes[nz]], 1).astype("<u8")
            f.write(b"sprs" + struct.pack("<Q", pairs.size) + pairs.tobytes())
        for lst in nz:
            o0, o1 = int(ix.list_offsets[lst]), int(ix.list_offsets[lst + 1])
            f.write(np.ascontiguousarray(ix.vectors[o0:o1], "<f4").tobytes())
            f.write(np.ascontiguousarray(ix.ids[o0:o1], "<i8").tobytes())


def get_feature_matrix(features_dir) -> np.ndarray:
    """train.py:35-38 over the `*.npy` files under features_dir in sorted path order -> [n, d] float32."""
    features_dir = Path(features_dir)
    files = sorted(features_dir.rglob("*.npy"))
    if not files:
        raise ValueError(f"no *.npy feature files under {features_dir}")
    mats = []
    for p in files:
        m = np.load(str(p))
        if m.ndim != 2:
            raise ValueError(f"{p}: features must be a [frames, width] matrix, got shape {m.shape}")
        if mats and m.shape[1] != mats[0].shape[1]:
            raise ValueError(f"{p}: feature width {m.shape[1]} differs from {mats[0].shape[1]} of {files[0]}")
        mats.append(m)
    x = np.ascontiguousarray(np.concatenate(mats, axis=0), dtype=np.float32)   # faiss trains on float32
    if not np.isfinite(x).all():
        raise ValueError(f"{features_dir}: the features hold non-finite values")
    return x


def train_index(features_dir, out_path, compress_after: int = 200_000, n_clusters: int = 10_000, device="cuda") -> IVFFlat:
    """train.py:11-32 with the transform of svc_train_retrieval.py:55-59: compress when n > compress_after, then
    `IVF{nlist},Flat` train + add, saved to out_path (FileExistsError if it exists)."""
    features_dir, out_path = Path(features_dir), Path(out_path)
    if out_path.exists():
        raise FileExistsError(f"index already exists by path {out_path}")
    logger.info("start getting feature vectors from %s", features_dir.absolute())
    x = get_feature_matrix(features_dir)
    logger.debug("fetched %s features", x.shape[0])
    _check_dim(x.shape[1])
    logger.info("apply transform to feature matrix")
    if x.shape[0] > compress_after:
        logger.info("pass condition. Transform by rule LloydKmeansFeatureTransform")
        _check_clusters(x.shape[0], n_clusters)
        x = compress_features(x, n_clusters, device=device)
    else:
        logger.info("condition is not passed. Transform by rule DummyFeatureTransform")
    n = x.shape[0]
    logger.debug("features transformed. Current features %s", n)
    if default_nlist(n) < 1:
        raise ValueError(f"{n} feature rows give nlist = 0: an IVF index needs at least {MIN_POINTS_PER_LIST} rows")
    logger.info("adding features to index with training")
    start = time.monotonic()
    ix = train_ivf_flat(x, device=device)
    logger.info("index is trained and filled. Took %.2f seconds", time.monotonic() - start)
    write_ivf_flat(out_path, ix)
    logger.info("index saved to %s", out_path.absolute())
    return ix
