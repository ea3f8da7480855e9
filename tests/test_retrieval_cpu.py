"""Feature retrieval, host side: the faiss IVF-Flat reader, the oracle against the unmodified reference and the
goldens, and the CLI's index-path rules (no GPU)."""
import os
import struct
from argparse import Namespace
from pathlib import Path

import numpy as np
import pytest

from oracle import ref_import
from oracle import retrieval_oracle as RO
from whisper_vits_svc_b200 import retrieval as R


def _hdr(d, ntotal, metric=1):
    return struct.pack("<i", d) + struct.pack("<q", ntotal) + struct.pack("<qq", 0, 0) + struct.pack("<B", 1) + \
        struct.pack("<i", metric) + (struct.pack("<f", 0.5) if metric > 1 else b"")


def _hand_file(d=64, sparse=False, fourcc=b"IwFl", metric=1, dm_type=0, qfourcc=b"IxF2"):
    """An IndexIVFFlat file assembled field by field (independent of oracle.write_ivf_flat): 3 lists of sizes 2, 0, 1."""
    rng = np.random.default_rng(5)
    cen = rng.standard_normal((3, d)).astype(np.float32)
    v0 = rng.standard_normal((2, d)).astype(np.float32)
    v2 = rng.standard_normal((1, d)).astype(np.float32)
    b = fourcc + _hdr(d, 3, metric) + struct.pack("<Q", 3) + struct.pack("<Q", 2)
    b += qfourcc + _hdr(d, 3, metric) + struct.pack("<Q", 3 * d) + cen.tobytes()
    b += struct.pack("<B", dm_type) + struct.pack("<Q", 0)
    b += b"ilar" + struct.pack("<Q", 3) + struct.pack("<Q", 4 * d)
    if sparse:
        b += b"sprs" + struct.pack("<Q", 4) + struct.pack("<QQ", 0, 2) + struct.pack("<QQ", 2, 1)
    else:
        b += b"full" + struct.pack("<Q", 3) + struct.pack("<QQQ", 2, 0, 1)
    b += v0.tobytes() + struct.pack("<qq", 11, 7)
    b += v2.tobytes() + struct.pack("<q", 42)
    return b, cen, np.concatenate([v0, v2]), np.array([11, 7, 42])


@pytest.mark.parametrize("sparse", [False, True])
def test_reader_hand_assembled(tmp_path, sparse):
    b, cen, vec, ids = _hand_file(sparse=sparse)
    p = tmp_path / "x.index"
    p.write_bytes(b)
    ix = R.read_ivf_flat(p)
    assert (ix.d, ix.nlist, ix.nprobe, ix.metric, ix.ntotal) == (64, 3, 2, 1, 3)
    assert np.array_equal(ix.centroids, cen)
    assert ix.list_offsets.tolist() == [0, 2, 2, 3]
    assert np.array_equal(ix.vectors, vec) and ix.ids.tolist() == ids.tolist()


@pytest.mark.parametrize("kind,match", [
    (dict(fourcc=b"IvFl"), "not supported"),
    (dict(fourcc=b"IxFI"), "not supported"),
    (dict(qfourcc=b"IxFI"), "quantizer"),
    (dict(metric=0), "metric"),
    (dict(dm_type=2), "hashtable"),
])
def test_reader_rejects(tmp_path, kind, match):
    b, *_ = _hand_file(**kind)
    p = tmp_path / "x.index"
    p.write_bytes(b)
    with pytest.raises(R.IndexFormatError, match=match):
        R.read_ivf_flat(p)


def test_reader_rejects_truncated_and_trailing(tmp_path):
    b, *_ = _hand_file()
    p = tmp_path / "x.index"
    for cut in (3, 40, len(b) // 2, len(b) - 1):
        p.write_bytes(b[:cut])
        with pytest.raises(R.IndexFormatError, match="truncated"):
            R.read_ivf_flat(p)
    p.write_bytes(b + b"\0")
    with pytest.raises(R.IndexFormatError, match="trailing"):
        R.read_ivf_flat(p)


def test_reader_rejects_bad_dimension(tmp_path):
    cen, lists = RO.clustered_index(3, 96, 4)
    p = tmp_path / "x.index"
    RO.write_ivf_flat(p, cen, lists)
    with pytest.raises(R.IndexFormatError, match="multiple of 64"):
        R.pack_ivf(R.read_ivf_flat(p))
    cen, lists = RO.clustered_index(3, 128, 4)
    RO.write_ivf_flat(p, cen, lists)
    with pytest.raises(R.IndexFormatError, match="does not match"):
        R.load_retrieve_index(p, 0.5, 3, "cpu", expected_dim=256)


@pytest.mark.parametrize("sparse", [False, True])
def test_writer_reader_round_trip(tmp_path, sparse):
    cen, lists = RO.clustered_index(4, 128, 9, sizes=[3, 0, 5, 1, 2, 0, 7, 4, 1])
    p = tmp_path / "x.index"
    RO.write_ivf_flat(p, cen, lists, nprobe=3, sparse=sparse)
    ix = R.read_ivf_flat(p)
    ref = RO.from_parts(cen, lists, nprobe=3)
    assert (ix.d, ix.nlist, ix.nprobe) == (128, 9, 3)
    for f in ("centroids", "list_offsets", "vectors", "ids"):
        assert np.array_equal(getattr(ix, f), getattr(ref, f)), f


def test_pack_ivf_layout():
    cen, lists = RO.clustered_index(6, 128, 7)
    ix = RO.from_parts(cen, lists)
    items, cfg = R.pack_ivf(ix)
    t = dict(items)
    assert (cfg.d, cfg.nlist, cfg.nprobe, cfg.ntotal) == (128, 7, 1, ix.ntotal)
    assert t["ivf.wimg"].numel() == 256 * 3 * 128 // 2
    cn = t["ivf.cnorm"].numpy()
    assert np.isinf(cn[7:]).all() and np.allclose(cn[:7], (cen.astype(np.float64) ** 2).sum(1), rtol=1e-7)
    assert np.array_equal(t["ivf.offsets"].numpy().view(np.int32), ix.list_offsets.astype(np.int32))
    assert np.array_equal(t["ivf.ids"].numpy().view(np.int64), ix.ids)
    # the image decodes to [-2 c_hi | -2 c_hi | -2 c_lo] with hi + lo = -2 c to bf16x2 precision
    import torch
    img = t["ivf.wimg"].view(torch.bfloat16).view(1, 3 * 128 // 64, 8, 256, 8).permute(0, 3, 1, 2, 4).reshape(256, 3 * 128).float()
    hi, hi2, lo = img[:, :128], img[:, 128:256], img[:, 256:]
    assert torch.equal(hi, hi2)
    assert float((hi + lo - torch.from_numpy(-2 * np.pad(cen, ((0, 249), (0, 0))))).abs().max()) <= 2e-5 * 2 * np.abs(cen).max()


def test_oracle_search_all_lists_is_exact_knn():
    cen, lists = RO.clustered_index(8, 64, 6)
    ix = RO.from_parts(cen, lists)
    q = (cen[np.arange(40) % 6] + 0.5 * np.random.default_rng(9).standard_normal((40, 64))).astype(np.float32)
    dist, ids, _, _ = RO.search(ix, q, 5, nprobe=6)
    d64, i64 = RO.knn_float64(ix, q, 5)
    assert np.array_equal(ids, i64)
    assert np.allclose(dist, d64, rtol=1e-5)


def _golden_names():
    return list(RO.RETRIEVAL_CASES)


@pytest.mark.parametrize("name", _golden_names())
def test_oracle_matches_golden(name):
    ix, g = RO.load_golden(name)
    dist, ids, _, vecs = RO.search(ix, g["queries"], int(g["k"]))
    assert np.array_equal(ids, g["search_ids"]) and np.array_equal(dist, g["search_dist"])
    out = RO.blend_reference(g["queries"], dist, vecs, float(g["ratio"]))
    assert np.array_equal(np.isnan(out), np.isnan(g["retriv"]))
    fin = ~np.isnan(g["retriv"])
    assert np.array_equal(out[fin], g["retriv"][fin])
    # the defined form equals the reference wherever the reference is finite, and is finite everywhere
    dfn = RO.blend_defined(g["queries"], dist, vecs, float(g["ratio"]))
    assert np.isfinite(dfn).all()
    rows = fin.all(1)
    assert np.abs(dfn[rows] - g["retriv"][rows]).max() <= 1e-6 * max(1.0, np.abs(g["queries"]).max())


needs_ref = pytest.mark.skipif(not ref_import.available(), reason="reference tree not present")


@needs_ref
@pytest.mark.parametrize("ratio,k", [(0.5, 3), (0.25, 1), (1.0, 5)])
def test_oracle_blend_equals_live_reference(monkeypatch, tmp_path, ratio, k):
    ix, q = RO.golden_parts("retrieval_d256_n37")
    path = str(tmp_path / "h.index")
    fr_index, fr_retrieval = RO.import_feature_retrieval({path: ix}, monkeypatch)
    ref = fr_index.load_retrieve_index(filepath=path, ratio=ratio, n_nearest_vectors=k)
    with np.errstate(divide="ignore", invalid="ignore"):
        out_ref = ref.retriv(q)
    dist, _, _, vecs = RO.search(ix, q, k)
    out = RO.blend_reference(q, dist, vecs, ratio)
    fin = np.isfinite(out_ref)
    assert np.array_equal(fin, np.isfinite(out)) and np.array_equal(out[fin], out_ref[fin])
    dfn = RO.blend_defined(q, dist, vecs, ratio)
    nan_rows = ~fin.all(1)
    assert nan_rows.any() and np.isfinite(dfn[nan_rows]).all()   # NaN in the reference, finite in the defined form
    rows = fin.all(1)
    assert rows.any() and np.abs(dfn[rows] - out_ref[rows]).max() <= 1e-6 * max(1.0, np.abs(q).max())
    # FaissIndexRetrieval: the torch wrapper of the same blend
    import torch
    fir = fr_retrieval.FaissIndexRetrieval(hubert_index=ref, whisper_index=ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        t = fir.retriv_hubert(torch.from_numpy(q)).numpy()
    assert np.array_equal(t[fin], out_ref[fin])


@needs_ref
def test_reference_rejections(monkeypatch, tmp_path):
    ix, _ = RO.golden_parts("retrieval_d256_n37")
    path = str(tmp_path / "h.index")
    fr_index, _ = RO.import_feature_retrieval({path: ix}, monkeypatch)
    with pytest.raises(ValueError):
        fr_index.load_retrieve_index(filepath=path, ratio=0.5, n_nearest_vectors=0)
    fr_index.load_retrieve_index(filepath=path, ratio=7.0, n_nearest_vectors=1)   # any ratio is accepted


def test_device_index_rejections_match_reference():
    cen, lists = RO.clustered_index(3, 64, 2)
    ix = RO.from_parts(cen, lists)
    with pytest.raises(ValueError, match="gte 1"):
        R.DeviceIVFIndex(ix, 0.5, 0, "cpu")
    ix.metric = 0
    with pytest.raises(ValueError, match="metric"):
        R.DeviceIVFIndex(ix, 0.5, 3, "cpu")


def test_speaker_name_and_index_paths(tmp_path):
    assert R.get_speaker_name_from_path(Path("sunny.npy")) == "su"
    assert R.get_speaker_name_from_path(Path("data/spk/alice.spk.npy")) == "alice"
    assert R.get_speaker_name_from_path("x/bob.npy") == "bob"
    hub, whi = R.index_paths("spk/sunny.npy", "", None, None, root=tmp_path)
    assert hub == tmp_path / "data_svc" / "indexes" / "su" / "hubert.index"
    assert whi == tmp_path / "data_svc" / "indexes" / "su" / "whisper.index"
    hub, whi = R.index_paths("a.npy", "p_", None, None, root=tmp_path)
    assert (hub.name, whi.name) == ("p_hubert.index", "p_whisper.index")
    hub, whi = R.index_paths("a.npy", "p_", "/x/h.index", "/y/w.index", root=tmp_path)
    assert (str(hub), str(whi)) == ("/x/h.index", "/y/w.index")


def test_create_retrival_disabled_is_dummy():
    import torch
    args = Namespace(enable_retrieval=False)
    r = R.create_retrival(args, None)
    assert isinstance(r, R.DummyRetrieval)
    x = torch.randn(4, 8)
    assert torch.equal(r.retriv_whisper(x), x) and torch.equal(r.retriv_hubert(x), x)


def test_chunked_retrieval_equals_whole_utterance():
    """svc_inference.py:117-118 retrieves per 2500-frame chunk (+-10 frames); the rows are the same when the whole
    utterance is retrieved once (what hostio.svc_infer does)."""
    from whisper_vits_svc_b200 import hostio
    ix, _ = RO.golden_parts("retrieval_d256_n37")
    n = 2600
    rng = np.random.default_rng(3)
    x = (ix.centroids[rng.integers(0, ix.nlist, n)] + 0.4 * rng.standard_normal((n, ix.d))).astype(np.float32)

    def retriv(rows):
        dist, _, _, vecs = RO.search(ix, rows, 3)
        return RO.blend_defined(rows, dist, vecs, 0.5)

    whole = retriv(x)
    for cs, ce, _, _ in hostio.chunk_plan(n, 320):
        assert np.array_equal(retriv(x[cs:ce]), whole[cs:ce])
