"""Feature retrieval on the H100 path — mirror of the reference's `feature_retrieval/` (`load_retrieve_index`,
`FaissRVCRetrievableFeatureIndex.retriv`, `DummyRetrieval`, `FaissIndexRetrieval`) and of `create_retrival` in its
`svc_inference.py:19-58`, behind the C ABI (`svcb_ivf_*`, csrc/retrieval_api.cu).

faiss is not needed: `read_ivf_flat` parses the `IndexIVFFlat` files faiss 1.7.4 writes (`faiss/impl/index_write.cpp`),
and the search, the RVC weighting and the blend run on the device.  Rows whose reference output is NaN (a query equal to
an index vector, or probed lists holding fewer than k vectors) are defined here instead: zero-distance neighbours share
the weight equally, otherwise the blend runs over the neighbours found, and a row with none passes through unchanged."""
from __future__ import annotations

import logging
import struct
from dataclasses import dataclass
from pathlib import Path
from typing import List, Tuple

import numpy as np
import torch

from . import _lib, pack
from .whisper_infer import _bf16_as_f32

logger = logging.getLogger(__name__)

METRIC_L2 = 1
MAX_K, MAX_NPROBE = 32, 8


class IndexFormatError(ValueError):
    pass


@dataclass
class IVFFlat:
    d: int
    nlist: int
    nprobe: int
    metric: int
    centroids: np.ndarray      # [nlist, d] float32
    list_offsets: np.ndarray   # [nlist + 1] int64: list l holds vectors[list_offsets[l]:list_offsets[l + 1]]
    vectors: np.ndarray        # [ntotal, d] float32, in list order
    ids: np.ndarray            # [ntotal] int64

    @property
    def ntotal(self) -> int:
        return int(self.vectors.shape[0])


class _Reader:
    def __init__(self, buf: bytes, path):
        self.buf, self.pos, self.path = buf, 0, path

    def take(self, n: int) -> bytes:
        if n < 0 or self.pos + n > len(self.buf):
            raise IndexFormatError(f"{self.path}: truncated index file (need {n} bytes at offset {self.pos}, "
                                   f"file has {len(self.buf)})")
        b = self.buf[self.pos:self.pos + n]
        self.pos += n
        return b

    def unpack(self, fmt: str):
        return struct.unpack("<" + fmt, self.take(struct.calcsize("<" + fmt)))

    def array(self, dtype, count: int) -> np.ndarray:
        dt = np.dtype(dtype).newbyteorder("<")
        return np.frombuffer(self.take(count * dt.itemsize), dtype=dt).astype(dtype)

    def header(self):
        """read_index_header: d, ntotal, two dummies, is_trained, metric_type (+ metric_arg when > 1)."""
        d, ntotal, _, _, _is_trained, metric = self.unpack("iqqqBi")
        if metric > 1:
            self.unpack("f")
        return d, ntotal, metric


def read_ivf_flat(path) -> IVFFlat:
    """Parse an `IndexIVFFlat` written by faiss.write_index (fourcc `IwFl`, L2 metric, `ilar` inverted lists)."""
    buf = Path(path).read_bytes()
    r = _Reader(buf, path)
    fourcc = r.take(4)
    if fourcc != b"IwFl":
        raise IndexFormatError(f"{path}: index type {fourcc!r} is not supported: only IVF-Flat (IwFl) indexes are")
    d, ntotal, metric = r.header()
    if metric != METRIC_L2:
        raise IndexFormatError(f"{path}: index metric type {metric} is unsupported; only METRIC_L2 ({METRIC_L2}) is")
    nlist, nprobe = r.unpack("QQ")
    if d < 1 or nlist < 1 or ntotal < 0:
        raise IndexFormatError(f"{path}: bad IVF header d={d} nlist={nlist} ntotal={ntotal}")
    q = r.take(4)
    if q != b"IxF2":
        raise IndexFormatError(f"{path}: coarse quantizer {q!r} is not supported: only IndexFlatL2 (IxF2) is")
    qd, qn, qmetric = r.header()
    if qd != d or qn != nlist or qmetric != METRIC_L2:
        raise IndexFormatError(f"{path}: quantizer (d={qd}, ntotal={qn}, metric={qmetric}) does not match the IVF "
                               f"index (d={d}, nlist={nlist}, L2)")
    (n,) = r.unpack("Q")
    if n != nlist * d:
        raise IndexFormatError(f"{path}: quantizer holds {n} floats, expected nlist * d = {nlist * d}")
    centroids = r.array(np.float32, n).reshape(nlist, d)
    dm_type, dm_count = r.unpack("BQ")
    if dm_type == 2:
        raise IndexFormatError(f"{path}: direct map of type hashtable is not supported")
    if dm_type not in (0, 1):
        raise IndexFormatError(f"{path}: unknown direct map type {dm_type}")
    r.take(8 * dm_count)
    il = r.take(4)
    if il != b"ilar":
        raise IndexFormatError(f"{path}: inverted lists {il!r} are not supported: only ArrayInvertedLists (ilar) are")
    il_nlist, code_size = r.unpack("QQ")
    if il_nlist != nlist or code_size != 4 * d:
        raise IndexFormatError(f"{path}: inverted lists (nlist={il_nlist}, code_size={code_size}) do not match "
                               f"nlist={nlist}, 4 d={4 * d}")
    kind = r.take(4)
    sizes = np.zeros(nlist, dtype=np.int64)
    if kind == b"full":
        (cnt,) = r.unpack("Q")
        if cnt != nlist:
            raise IndexFormatError(f"{path}: {cnt} list sizes for {nlist} lists")
        sizes[:] = r.array(np.uint64, nlist).astype(np.int64)
    elif kind == b"sprs":
        (cnt,) = r.unpack("Q")
        if cnt % 2:
            raise IndexFormatError(f"{path}: odd sparse list-size count {cnt}")
        pairs = r.array(np.uint64, cnt).reshape(-1, 2).astype(np.int64)
        for lst, sz in pairs:
            if not 0 <= lst < nlist:
                raise IndexFormatError(f"{path}: sparse list id {lst} out of range")
            sizes[lst] = sz
    else:
        raise IndexFormatError(f"{path}: list-size encoding {kind!r} is unknown")
    if sizes.sum() != ntotal:
        raise IndexFormatError(f"{path}: lists hold {int(sizes.sum())} vectors, header says ntotal={ntotal}")
    vectors = np.empty((ntotal, d), dtype=np.float32)
    ids = np.empty(ntotal, dtype=np.int64)
    offsets = np.zeros(nlist + 1, dtype=np.int64)
    offsets[1:] = np.cumsum(sizes)
    for lst in range(nlist):
        sz = int(sizes[lst])
        if sz == 0:
            continue
        o = int(offsets[lst])
        vectors[o:o + sz] = r.array(np.float32, sz * d).reshape(sz, d)
        ids[o:o + sz] = r.array(np.int64, sz)
    if r.pos != len(buf):
        raise IndexFormatError(f"{path}: {len(buf) - r.pos} trailing bytes after the index")
    return IVFFlat(d=d, nlist=nlist, nprobe=nprobe, metric=metric, centroids=centroids, list_offsets=offsets,
                   vectors=vectors, ids=ids)


def pack_centroids(centroids: np.ndarray) -> Tuple[torch.Tensor, torch.Tensor]:
    """centroids [nlist, d] -> ("ivf.wimg", "ivf.cnorm"): the coarse search's bf16 tile image of [-2 c_hi | -2 c_hi | -2 c_lo]
    and |c|^2 summed in float64 (+inf on the rows padding nlist to whole 256-column tiles), both CPU float32 tensors."""
    nlist, d = centroids.shape
    npad = (nlist + 255) // 256 * 256
    c = torch.zeros(npad, d, dtype=torch.float32)
    c[:nlist] = torch.from_numpy(np.ascontiguousarray(centroids, dtype=np.float32))
    m2 = -2.0 * c                                        # exact: a power-of-two scale
    hi = m2.bfloat16()
    lo = (m2 - hi.float()).bfloat16()
    wimg = _bf16_as_f32(torch.cat([hi, hi, lo], dim=1).float())   # pairs with the query image [x_hi | x_lo | x_hi]
    cnorm = torch.full((npad,), float("inf"), dtype=torch.float32)
    cnorm[:nlist] = torch.from_numpy((centroids.astype(np.float64) ** 2).sum(1).astype(np.float32))
    return wimg, cnorm


def pack_ivf(ix: IVFFlat) -> Tuple[List[Tuple[str, torch.Tensor]], _lib.IvfConfig]:
    """-> ([(name, fp32-typed tensor)], svcb_ivf_config).  Names consumed by csrc/retrieval_api.cu (include/svcb.h)."""
    if ix.d % 64 or not 64 <= ix.d <= 2048:
        raise IndexFormatError(f"index dimension {ix.d} is not supported: need a multiple of 64 in [64, 2048]")
    if not 1 <= ix.nprobe <= MAX_NPROBE:
        raise IndexFormatError(f"index nprobe {ix.nprobe} is not supported: need 1 <= nprobe <= {MAX_NPROBE}")
    d, nlist = ix.d, ix.nlist
    wimg, cnorm = pack_centroids(ix.centroids)
    items = [
        ("ivf.wimg", wimg),
        ("ivf.cnorm", cnorm),
        ("ivf.vectors", torch.from_numpy(np.ascontiguousarray(ix.vectors, dtype=np.float32)).reshape(-1)),
        ("ivf.offsets", torch.from_numpy(ix.list_offsets.astype(np.int32)).view(torch.float32)),
        ("ivf.ids", torch.from_numpy(np.ascontiguousarray(ix.ids, dtype=np.int64)).view(torch.float32)),
    ]
    cfg = _lib.IvfConfig(d=d, nlist=nlist, nprobe=ix.nprobe, pad_=0, ntotal=ix.ntotal)
    return items, cfg


class DeviceIVFIndex:
    """`FaissRVCRetrievableFeatureIndex` of the reference on the device: `retriv(x)` and `search(x, k)`."""

    def __init__(self, ix: IVFFlat, ratio: float, n_nearest_vectors: int, device="cuda"):
        if ix.metric != METRIC_L2:                                   # index.py:37-38
            raise ValueError(f"index metric type {ix.metric} is unsupported, supported distance {METRIC_L2}")
        if 1 > n_nearest_vectors:                                    # index.py:40-41
            raise ValueError("n-retrieval-vectors must be gte 1")
        if n_nearest_vectors > MAX_K:
            raise ValueError(f"n-retrieval-vectors must be <= {MAX_K}")
        # index.py:44's `0 > ratio > 1` never holds, so the reference accepts any ratio; so does this class
        self.ratio, self.k, self.d, self.nlist = float(ratio), int(n_nearest_vectors), ix.d, ix.nlist
        self.device = _lib.cuda_device(device)
        items, cfg = pack_ivf(ix)
        blob_cpu, table = pack.build_blob(items)
        self._handle = _lib.Handle("ivf", table, blob_cpu.to(self.device), cfg)

    def _run(self, x: torch.Tensor, k: int, ratio: float, want_out: bool, want_search: bool):
        if x.dim() != 2 or x.shape[1] != self.d:
            raise ValueError(f"features must be [M, {self.d}], got {tuple(x.shape)}")
        xd = x.to(self.device, torch.float32).contiguous()
        M = xd.shape[0]
        out = torch.empty_like(xd) if want_out else None
        dist = torch.empty(M, k, device=self.device, dtype=torch.float32) if want_search else None
        ids = torch.empty(M, k, device=self.device, dtype=torch.int64) if want_search else None
        if M:
            ws = self._handle.workspace(_lib.load().svcb_ivf_workspace_bytes(self._handle, M, k))
            ptr = lambda t: None if t is None else t.data_ptr()   # noqa: E731
            self._handle.call("ivf_retrieve", xd.data_ptr(), ptr(out), ptr(dist), ptr(ids), M, k, float(np.float32(ratio)),
                              ws.data_ptr(), ws.numel())
        return out, dist, ids

    @torch.no_grad()
    def search(self, x: torch.Tensor, k: int | None = None):
        """-> (distances [M, k] float32 ascending, ids [M, k] int64) on the device; +inf / -1 where fewer than k were found."""
        _, dist, ids = self._run(x, int(k or self.k), 0.0, False, True)
        return dist, ids

    @torch.no_grad()
    def retriv(self, x: torch.Tensor) -> torch.Tensor:
        """index.py:57-62: (1 - ratio) x + ratio * blend of the k nearest vectors, on x's device."""
        out, _, _ = self._run(x, self.k, self.ratio, True, False)
        return out.to(x.device)


def load_retrieve_index(filepath, ratio: float, n_nearest_vectors: int, device="cuda", expected_dim: int | None = None):
    """index.py:157-160.  expected_dim: the feature width the index must have (hp.vits.ppg_dim / vec_dim)."""
    ix = read_ivf_flat(filepath)
    if expected_dim is not None and ix.d != int(expected_dim):
        raise IndexFormatError(f"{filepath}: index dimension {ix.d} does not match the model's feature width {expected_dim}")
    return DeviceIVFIndex(ix, ratio, n_nearest_vectors, device)


class DummyRetrieval:
    """retrieval.py:21-28: features pass through (the reference also moves them to the CPU)."""

    def retriv_whisper(self, vec: torch.Tensor) -> torch.Tensor:
        logger.debug("start dummy retriv whisper")
        return vec.clone().to(torch.device("cpu"))

    def retriv_hubert(self, vec: torch.Tensor) -> torch.Tensor:
        logger.debug("start dummy retriv hubert")
        return vec.clone().to(torch.device("cpu"))


class IndexRetrieval:
    """FaissIndexRetrieval (retrieval.py:31-44) over device indexes."""

    def __init__(self, hubert_index: DeviceIVFIndex, whisper_index: DeviceIVFIndex):
        self._hubert_index = hubert_index
        self._whisper_index = whisper_index

    def retriv_whisper(self, vec: torch.Tensor) -> torch.Tensor:
        logger.debug("start retriv whisper")
        return self._whisper_index.retriv(vec)

    def retriv_hubert(self, vec: torch.Tensor) -> torch.Tensor:
        logger.debug("start retriv hubert")
        return self._hubert_index.retriv(vec)


def get_speaker_name_from_path(speaker_path) -> str:
    """svc_inference.py:19-22 as written: `str.rstrip` strips a character SET, so `sunny.npy` gives `su`."""
    speaker_path = Path(speaker_path)
    suffixes = "".join(speaker_path.suffixes)
    return speaker_path.name.rstrip(suffixes)


def index_paths(spk, prefix: str = "", hubert_index_path=None, whisper_index_path=None, root=".") -> Tuple[Path, Path]:
    """svc_inference.py:31-45: (hubert, whisper) index files, by default ./data_svc/indexes/<speaker>/<prefix>{hubert,whisper}.index."""
    base = Path(root).absolute() / "data_svc" / "indexes" / get_speaker_name_from_path(spk)
    hub = Path(hubert_index_path) if hubert_index_path else base / f"{prefix}hubert.index"
    whi = Path(whisper_index_path) if whisper_index_path else base / f"{prefix}whisper.index"
    return hub, whi


def create_retrival(args, hp, device="cuda"):
    """svc_inference.py:25-58, with each index's dimension checked against hp.vits.vec_dim / ppg_dim."""
    if not args.enable_retrieval:
        logger.info("infer without retrival")
        return DummyRetrieval()
    logger.info("load index retrival model")
    hub, whi = index_paths(args.spk, args.retrieval_index_prefix, args.hubert_index_path, args.whisper_index_path)
    return IndexRetrieval(
        hubert_index=load_retrieve_index(hub, args.retrieval_ratio, args.n_retrieval_vectors, device, int(hp.vits.vec_dim)),
        whisper_index=load_retrieve_index(whi, args.retrieval_ratio, args.n_retrieval_vectors, device, int(hp.vits.ppg_dim)),
    )
