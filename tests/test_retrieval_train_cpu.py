"""Building retrieval indexes, host side: the unmodified reference's svc_train_retrieval.py behind stubs against
retrieval_train's choices, the faiss IVF-Flat writer, the input checks, and the oracle's Lloyd compression against
scikit-learn's MiniBatchKMeans (no GPU)."""
import importlib.util
import multiprocessing
import os

import numpy as np
import pytest

from oracle import kmeans_oracle as KO
from oracle import ref_import
from oracle import retrieval_oracle as RO
from tests.util import ROOT
from whisper_vits_svc_b200 import retrieval as R
from whisper_vits_svc_b200 import retrieval_train as RT

needs_ref = pytest.mark.skipif(not ref_import.available(), reason="reference tree not present")


def _own_cli():
    spec = importlib.util.spec_from_file_location("svcb_train_retrieval_cli", os.path.join(ROOT, "svc_train_retrieval.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def _features(base, feature, speaker, sizes, d, seed):
    """base/feature/speaker/{nested paths}.npy with the given row counts."""
    rng = np.random.default_rng(seed)
    out = []
    for i, n in enumerate(sizes):
        p = base / feature / speaker / ("sub" if i % 2 else "") / f"f{i:02d}.npy"
        p.parent.mkdir(parents=True, exist_ok=True)
        m = rng.standard_normal((n, d)).astype(np.float32)
        np.save(p, m)
        out.append(m)
    return np.concatenate(out)


def _rows_sorted(m):
    m = np.asarray(m, np.float32)
    return m[np.lexsort(m.T[::-1])]


class _Recorder:
    """Stands in for the device steps of retrieval_train.train_index: records what would be compressed and trained."""

    def __init__(self, monkeypatch):
        self.compress, self.train, self.written = [], [], []
        monkeypatch.setattr(RT, "compress_features", self._compress)
        monkeypatch.setattr(RT, "train_ivf_flat", self._train)
        monkeypatch.setattr(RT, "write_ivf_flat", self._write)

    def _compress(self, x, n_clusters, device="cuda"):
        self.compress.append((x.shape, n_clusters))
        return np.array(x[:n_clusters], copy=True)

    def _train(self, x, device="cuda"):
        self.train.append(np.array(x, copy=True))
        return None

    def _write(self, path, ix, rewrite=False):
        self.written.append(str(path))


@needs_ref
@pytest.mark.parametrize("n", [39, 40, 1000, 200_000, 10 ** 7])
def test_nlist_matches_reference(monkeypatch, n):
    stm, rec = KO.import_train_retrieval(monkeypatch)
    stm.FaissIVFFlatTrainableFeatureIndexBuilder(8192, distance=RO.METRIC_L2).build(num_vectors=n, vector_dim=256)
    assert rec["factory"] == [(256, f"IVF{RT.default_nlist(n)},Flat", RO.METRIC_L2)]


@needs_ref
@pytest.mark.parametrize("after_delta,prefix", [(0, ""), (-1, "p_"), (1, "")])
def test_create_index_matches_reference(monkeypatch, tmp_path, after_delta, prefix):
    """The compression condition (strictly more rows than compress_features_after), the n_clusters it passes, the
    index path, and the multiset of rows handed to train and add (the reference adds in batches of 8,192)."""
    stm, rec = KO.import_train_retrieval(monkeypatch)
    base = tmp_path / "data_svc"
    x = _features(base, "hubert", "spk", [4000, 3000, 2500], 64, seed=1)
    n = len(x)
    after = n + after_delta
    (base / "indexes").mkdir()
    stm.create_index(feature_name="hubert", prefix=prefix, speaker="spk", base_path=base, indexes_path=base / "indexes",
                     compress_features_after=after, n_clusters=300, n_parallel=3)
    own = _Recorder(monkeypatch)
    cli = _own_cli()
    (tmp_path / "own").mkdir()
    cli.create_index("hubert", prefix, "spk", base, tmp_path / "own", after, 300)
    compressed = n > after
    assert bool(rec["mbk"]) == compressed == bool(own.compress)
    if compressed:
        assert rec["mbk"] == [dict(n_clusters=300, verbose=True, batch_size=768, compute_labels=False, init="k-means++")]
        assert own.compress == [((n, 64), 300)]
    assert rec["write"] == [str(base / "indexes" / "spk" / f"{prefix}hubert.index")]
    assert own.written == [str(tmp_path / "own" / "spk" / f"{prefix}hubert.index")]
    train_ref = rec["train"][0]
    add_ref = np.concatenate(rec["add"])
    assert len(rec["add"]) == -(-len(train_ref) // 8192)
    assert np.array_equal(_rows_sorted(train_ref), _rows_sorted(add_ref))
    if compressed:   # the stubs keep the first n_clusters rows, which depend on the file order
        assert own.train[0].shape == train_ref.shape == (300, 64)
    else:
        assert np.array_equal(_rows_sorted(own.train[0]), _rows_sorted(train_ref))
        assert np.array_equal(_rows_sorted(own.train[0]), _rows_sorted(x))


@needs_ref
def test_existing_index_is_an_error(monkeypatch, tmp_path):
    stm, _ = KO.import_train_retrieval(monkeypatch)
    base = tmp_path / "data_svc"
    _features(base, "whisper", "spk", [200], 64, seed=2)
    (base / "indexes" / "spk").mkdir(parents=True)
    (base / "indexes" / "spk" / "whisper.index").write_bytes(b"x")
    with pytest.raises(FileExistsError):
        stm.create_index(feature_name="whisper", prefix="", speaker="spk", base_path=base, indexes_path=base / "indexes",
                         compress_features_after=10 ** 6, n_clusters=10, n_parallel=1)
    with pytest.raises(FileExistsError):
        _own_cli().create_index("whisper", "", "spk", base, base / "indexes", 10 ** 6, 10)


@pytest.mark.parametrize("sizes,kind", [
    ([3, 0, 5, 1, 2, 0, 7, 4, 1], b"full"),
    ([3, 0, 0, 1, 0, 0, 0, 4, 0], b"sprs"),
    ([2, 0, 1, 0, 0, 5, 0, 1], b"sprs"),   # 4 of 8 non-empty: not more than nlist / 2
    ([2, 0, 1, 0, 3, 5, 0, 1], b"full"),
])
def test_writer_matches_oracle_and_round_trips(tmp_path, sizes, kind):
    cen, lists = RO.clustered_index(4, 128, len(sizes), sizes=sizes)
    ix = RO.from_parts(cen, lists, nprobe=1)
    ours, ref = tmp_path / "a.index", tmp_path / "b.index"
    RT.write_ivf_flat(ours, ix)
    RO.write_ivf_flat(ref, cen, lists, nprobe=1, sparse=kind == b"sprs")
    b = ours.read_bytes()
    assert b == ref.read_bytes() and kind in b
    back = R.read_ivf_flat(ours)
    assert (back.d, back.nlist, back.nprobe, back.metric) == (ix.d, ix.nlist, ix.nprobe, ix.metric)
    for f in ("centroids", "list_offsets", "vectors", "ids"):
        assert np.array_equal(getattr(back, f), getattr(ix, f)), f
    with pytest.raises(FileExistsError):
        RT.write_ivf_flat(ours, ix)
    RT.write_ivf_flat(ours, ix, rewrite=True)
    assert ours.read_bytes() == b


def test_input_errors(tmp_path, monkeypatch):
    own = _Recorder(monkeypatch)
    (tmp_path / "empty").mkdir()
    with pytest.raises(ValueError, match="no \\*.npy"):
        RT.train_index(tmp_path / "empty", tmp_path / "x.index")
    d = tmp_path / "mixed"
    d.mkdir()
    np.save(d / "a.npy", np.zeros((50, 64), np.float32))
    np.save(d / "b.npy", np.zeros((50, 128), np.float32))
    with pytest.raises(ValueError, match="width 128 differs"):
        RT.train_index(d, tmp_path / "x.index")
    d = tmp_path / "nan"
    d.mkdir()
    a = np.zeros((50, 64), np.float32)
    a[3, 5] = np.inf
    np.save(d / "a.npy", a)
    with pytest.raises(ValueError, match="non-finite"):
        RT.train_index(d, tmp_path / "x.index")
    for width in (32, 96, 4096):
        d = tmp_path / f"w{width}"
        d.mkdir()
        np.save(d / "a.npy", np.ones((50, width), np.float32))
        with pytest.raises(ValueError, match="multiple of 64"):
            RT.train_index(d, tmp_path / "x.index")
    d = tmp_path / "small"
    d.mkdir()
    np.save(d / "a.npy", np.ones((38, 64), np.float32))
    with pytest.raises(ValueError, match="at least 39"):
        RT.train_index(d, tmp_path / "x.index")
    np.save(d / "a.npy", np.ones((39, 64), np.float32))
    RT.train_index(d, tmp_path / "x.index")
    assert own.train[-1].shape == (39, 64)
    np.save(d / "a.npy", np.ones((60, 64), np.float32))
    with pytest.raises(ValueError, match="n_clusters must be <="):
        RT.train_index(d, tmp_path / "y.index", compress_after=59, n_clusters=61)
    RT.train_index(d, tmp_path / "y.index", compress_after=59, n_clusters=60)
    assert own.compress[-1] == ((60, 64), 60)
    (tmp_path / "exists.index").write_bytes(b"")
    with pytest.raises(FileExistsError):
        RT.train_index(d, tmp_path / "exists.index")


def test_feature_files_are_read_in_sorted_order(tmp_path):
    x = _features(tmp_path, "hubert", "s", [5, 7, 3, 4], 64, seed=3)
    got = RT.get_feature_matrix(tmp_path / "hubert" / "s")
    files = sorted((tmp_path / "hubert" / "s").rglob("*.npy"))
    assert np.array_equal(got, np.concatenate([np.load(p) for p in files]))
    assert _rows_sorted(got).tobytes() == _rows_sorted(x).tobytes()


def test_split_plan_matches_oracle():
    h = np.array([0, 40, 3, 0, 1, 90, 0, 7], np.float32)
    a, b = h.copy(), h.copy()
    pa = RT.split_plan(a, 200, np.random.default_rng(5))
    pb = KO.split_plan(b, 200, np.random.default_rng(5))
    assert pa == pb and [ci for ci, _ in pa] == [0, 3, 6]
    assert np.array_equal(a, b) and a.sum() == h.sum() and (a > 0).all()
    assert all(h[cj] > 1 for _, cj in pa if cj not in (0, 3, 6))


def test_oracle_kmeans_step_is_faiss_update():
    rng = np.random.default_rng(0)
    x = rng.standard_normal((500, 64)).astype(np.float32)
    c = x[:12].copy()
    c[7] = c[3]   # a duplicate centroid: ties to the lower one, centroid 7 is left empty and untouched
    a, dist, new, counts = KO.kmeans_step(x, c)
    assert counts[7] == 0 and np.array_equal(new[7], c[7]) and counts.sum() == 500
    d64 = ((x[:, None, :].astype(np.float64) - c[None].astype(np.float64)) ** 2).sum(-1)
    assert np.allclose(dist, d64[np.arange(500), a], rtol=1e-4, atol=1e-4)
    for j in range(12):
        if counts[j]:
            s = np.float32(0) * x[0]
            for i in np.flatnonzero(a == j):
                s = s + x[i]
            assert np.array_equal(new[j], s * (np.float32(1) / np.float32(counts[j])))


def test_oracle_compression_vs_minibatch_kmeans():
    """On a clustered fixture the oracle's Lloyd compression reaches an inertia no worse than 1.01x that of
    MiniBatchKMeans configured as transform.py:44-51 configures it."""
    cluster = pytest.importorskip("sklearn.cluster")
    rng = np.random.default_rng(11)
    cen = rng.standard_normal((150, 256)).astype(np.float32)
    x = (cen[rng.integers(0, 150, 30_000)] + 0.3 * rng.standard_normal((30_000, 256))).astype(np.float32)

    def inertia(c):
        _, dist = KO.assign(x, c)
        return float(dist.astype(np.float64).sum())

    ours, _ = KO.kmeans(x, 600, niter=10, max_points_per_centroid=None)
    mbk = cluster.MiniBatchKMeans(n_clusters=600, verbose=False, batch_size=256 * (multiprocessing.cpu_count() - 1 or 1),
                                  compute_labels=False, init="k-means++", random_state=0).fit(x).cluster_centers_
    ratio = inertia(ours) / inertia(mbk.astype(np.float32))
    print(f"Lloyd / MiniBatchKMeans inertia: {ratio:.4f}")
    assert ratio <= 1.01
