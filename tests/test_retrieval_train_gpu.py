"""Building retrieval indexes on the device (csrc/kmeans_api.cu, retrieval_train.py) against float64 arg-mins, the numpy
oracle (oracle/kmeans_oracle.py) and the device search (svcb_ivf_retrieve)."""
import os
import subprocess
import sys
from argparse import Namespace

import numpy as np
import pytest
import torch

from oracle import kmeans_oracle as KO
from oracle import retrieval_oracle as RO
from tests.util import ROOT
from whisper_vits_svc_b200 import retrieval as R
from whisper_vits_svc_b200 import retrieval_train as RT

pytestmark = pytest.mark.gpu


def _points(n, d, k, seed):
    rng = np.random.default_rng(seed)
    cen = rng.standard_normal((k, d)).astype(np.float32)
    x = (cen[rng.integers(0, k, n)] + 0.4 * rng.standard_normal((n, d))).astype(np.float32)
    return x, cen


def _host_image(cen):
    """(centroids, wimg, cnorm) on the device, the image and norms as pack_ivf builds them."""
    wimg, cnorm = R.pack_centroids(cen)
    return torch.from_numpy(cen).cuda(), wimg.cuda(), cnorm.cuda()


def _ambiguous(x, cen, best64):
    """The coarse criterion of test_retrieval_gpu._ambiguous: the two nearest centroids within 1e-5 (|x|^2 + |c|^2)."""
    xt, ct = torch.from_numpy(x).cuda().double(), torch.from_numpy(cen).cuda().double()
    d = (xt[:, None, :] - ct[None]).pow(2).sum(-1) if len(cen) < 64 else \
        (xt.pow(2).sum(1, keepdim=True) + ct.pow(2).sum(1)[None] - 2 * xt @ ct.T)
    if len(cen) == 1:
        return torch.zeros(len(x), dtype=torch.bool).numpy()
    two = torch.topk(d, 2, dim=1, largest=False).values
    scale = xt.pow(2).sum(1) + ct.pow(2).sum(1)[torch.from_numpy(best64).cuda()]
    return ((two[:, 1] - two[:, 0]) < 1e-5 * scale).cpu().numpy()


def _argmin64(x, cen):
    xt, ct = torch.from_numpy(x).cuda().double(), torch.from_numpy(cen).cuda().double()
    d = (xt[:, None, :] - ct[None]).pow(2).sum(-1) if len(cen) < 64 else \
        (xt.pow(2).sum(1, keepdim=True) + ct.pow(2).sum(1)[None] - 2 * xt @ ct.T)
    v, i = d.min(1)
    return i.cpu().numpy(), v.cpu().numpy()


@pytest.mark.parametrize("d", [256, 1280])
@pytest.mark.parametrize("k", [1, 7, 256, 5128, 10_000])
def test_assign_vs_float64(d, k):
    n = 3000
    x, cen = _points(n, d, k, seed=d + k)
    xd = torch.from_numpy(x).cuda()
    a, dist = RT.assign(xd, *_host_image(cen))
    a, dist = a.cpu().numpy(), dist.cpu().numpy()
    a64, d64 = _argmin64(x, cen)
    amb = _ambiguous(x, cen, a64)
    bad = a != a64
    print(f"d={d} k={k}: {bad.sum()} rows differ from float64, ambiguous {amb.sum()}")
    assert amb[bad].all() and amb.sum() / n < 0.01
    scale = (x.astype(np.float64) ** 2).sum(1) + (cen.astype(np.float64) ** 2).sum(1)[a64]
    assert np.all(np.abs(dist[~bad] - d64[~bad]) <= 2e-5 * scale[~bad])
    # chunk sizes, row positions and the device-built image do not change a row's result
    for chunk in (128, 384):
        a2, dist2 = (t.cpu().numpy() for t in RT.assign(xd, *_host_image(cen), chunk=chunk))
        assert np.array_equal(a2, a) and np.array_equal(dist2, dist)
    perm = np.random.default_rng(k).permutation(n)
    a3, dist3 = (t.cpu().numpy() for t in RT.assign(xd[torch.from_numpy(perm).cuda()], *_host_image(cen)))
    assert np.array_equal(a3, a[perm]) and np.array_equal(dist3, dist[perm])
    wimg, cnorm = RT.pack_device(torch.from_numpy(cen).cuda())
    _, hw, hc = _host_image(cen)
    assert torch.equal(wimg, hw)
    ulp = (cnorm.view(torch.int32).long() - hc.view(torch.int32).long()).abs()[:k]
    assert int(ulp.max()) <= 1


@pytest.mark.parametrize("d,k", [(256, 7), (1280, 5128)])
def test_assign_is_the_search_coarse_choice(d, k):
    """An index whose list l holds one vector with id l: its k = 1 search returns the list it probed."""
    x, cen = _points(4097, d, k, seed=3 * k)
    ix = RO.from_parts(cen, [(cen[l:l + 1], np.array([l])) for l in range(k)])
    dev = R.DeviceIVFIndex(ix, 0.5, 1, "cuda")
    xd = torch.from_numpy(x).cuda()
    _, ids = dev.search(xd, 1)
    a, _ = RT.assign(xd, *_host_image(cen), chunk=1024)
    assert torch.equal(ids[:, 0].int(), a)


def test_one_step_bitwise_vs_oracle():
    x, _ = _points(20_000, 256, 64, seed=5)
    c = x[np.random.default_rng(6).permutation(len(x))[:256]].copy()
    c[200] = c[100]   # an empty cluster
    a, dist, cd, counts = RT.kmeans_step(torch.from_numpy(x).cuda(), torch.from_numpy(c).cuda())
    a, cd, counts = a.cpu().numpy(), cd.cpu().numpy(), counts.cpu().numpy()
    ao, disto, co, counto = KO.kmeans_step(x, c)
    bad = a != ao
    touched = np.zeros(256, bool)
    touched[a[bad]] = touched[ao[bad]] = True
    print(f"one step: {bad.sum()} rows differ, clusters compared {(~touched).sum()}")
    assert bad.sum() < 0.001 * len(x) and (~touched).sum() > 240
    assert counts[200] == 0 and np.array_equal(cd[200], c[200])
    assert np.array_equal(counts[~touched], counto[~touched])
    assert np.array_equal(cd[~touched], co[~touched])
    assert np.allclose(dist.cpu().numpy()[~bad], disto[~bad], rtol=1e-4, atol=1e-3)
    # the update alone is bitwise reproducible and its order is the stable sort
    _, offs, order = RT.update(torch.from_numpy(x).cuda(), torch.from_numpy(a).cuda(), 256)
    assert np.array_equal(order.cpu().numpy(), np.argsort(a, kind="stable"))
    assert np.array_equal(offs.cpu().numpy(), np.concatenate([[0], np.cumsum(np.bincount(a, minlength=256))]))


def _split_fixture(n=10_000, k=42, nc=40, d=256, alpha=0.25):
    """nc well separated clusters and k = nc + 2 centroids.  k-means starts from one row of each cluster plus two rows
    made equal to the first two, so centroids 40 and 41 are empty after the first assignment and get split.  The two
    clusters they split are built of two sub-clusters offset by +-alpha (s * centre), s = (+1, -1, +1, ...): the
    direction split_clusters perturbs along, so the rows of a split cluster fall on either side by a clear margin, and
    so does every other assignment of every iteration."""
    init = np.random.default_rng(RT.SEED).permutation(n)[:k]
    s = np.where(np.arange(d) % 2 == 0, 1.0, -1.0).astype(np.float32)
    for seed in range(21, 80):
        rng = np.random.default_rng(seed)
        cen = 2.0 * rng.standard_normal((nc, d)).astype(np.float32)
        label = np.empty(n, np.int64)
        rest = np.setdiff1d(np.arange(n), init[:nc])
        label[init[:nc]] = np.arange(nc)
        label[rest] = rng.permutation(np.repeat(np.arange(nc), len(rest) // nc + 1)[:len(rest)])
        noise = 0.5 * rng.standard_normal((n, d)).astype(np.float32)
        side = np.where(rng.random(n) < 0.5, 1.0, -1.0).astype(np.float32)[:, None]

        def build(bimodal):
            x = cen[label] + noise
            for c in bimodal:
                rows = label == c
                x[rows] += side[rows] * alpha * (s * cen[c])
            x = x.astype(np.float32)
            x[init[nc:]] = x[init[:k - nc]]
            return x

        def pairs_of(x):   # the first iteration, drawing from the stream kmeans draws from
            rng2 = np.random.default_rng(RT.SEED)
            rng2.permutation(n)
            _, _, _, counts = KO.kmeans_step(x, x[init])
            return KO.split_plan(counts.astype(np.float32), n, rng2)

        pairs = pairs_of(build([]))
        cjs = [cj for _, cj in pairs]
        if [ci for ci, _ in pairs] != [nc, nc + 1] or len(set(cjs)) != 2 or max(cjs) >= nc:
            continue
        x = build(cjs)
        if pairs_of(x) == pairs:
            return x
    raise AssertionError("no seed gave two splits of distinct original clusters")


def test_training_matches_oracle_and_splits():
    x = _split_fixture()
    c, st = RT.kmeans(x, 42, niter=10)
    co, sto = KO.kmeans(x, 42, niter=10)
    print("objective", st["obj"], "\noracle   ", sto["obj"], "\nsplits", st["nsplit"], sto["nsplit"])
    assert st["nsplit"][0] >= 2 and st["nsplit"] == sto["nsplit"]
    assert np.allclose(st["obj"], sto["obj"], rtol=1e-5, atol=0)
    c2, st2 = RT.kmeans(x, 42, niter=10)
    assert np.array_equal(c, c2) and st == st2


def test_index_finds_every_training_vector(tmp_path):
    x, _ = _points(6000, 256, 150, seed=8)
    ix = RT.train_ivf_flat(x)
    assert ix.nlist == RT.default_nlist(6000) and ix.ntotal == 6000 and ix.nprobe == 1
    assert np.array_equal(np.sort(ix.ids), np.arange(6000))
    lists = np.repeat(np.arange(ix.nlist), np.diff(ix.list_offsets))
    for lst in range(ix.nlist):   # ascending ids inside each list
        assert np.all(np.diff(ix.ids[ix.list_offsets[lst]:ix.list_offsets[lst + 1]]) > 0)
    assert np.array_equal(ix.vectors, x[ix.ids])
    a, _ = RT.assign(torch.from_numpy(x).cuda(), *_host_image(ix.centroids))
    assert np.array_equal(a.cpu().numpy()[ix.ids], lists)
    p1, p2 = tmp_path / "a.index", tmp_path / "b.index"
    RT.write_ivf_flat(p1, ix)
    RT.write_ivf_flat(p2, RT.train_ivf_flat(x))
    assert p1.read_bytes() == p2.read_bytes()
    dev = R.load_retrieve_index(p1, 0.5, 1, "cuda", expected_dim=256)
    dist, ids = dev.search(torch.from_numpy(x).cuda(), 1)
    assert torch.equal(ids[:, 0].cpu(), torch.arange(6000)) and bool((dist == 0).all())


def test_cli_two_speakers(tmp_path, hp, monkeypatch):
    rng = np.random.default_rng(4)
    base = tmp_path / "data_svc"
    rows = {"alice": [1200, 900, 700], "bob": [500, 400]}   # alice: 2,800 rows, compressed to 400; bob: 900 rows
    for spk, sizes in rows.items():
        (base / "waves-16k" / spk).mkdir(parents=True)
        for feat, d in (("hubert", hp.vits.vec_dim), ("whisper", hp.vits.ppg_dim)):
            cen = rng.standard_normal((30, d)).astype(np.float32)
            for i, n in enumerate(sizes):
                p = base / feat / spk / f"{i}.{'vec' if feat == 'hubert' else 'ppg'}.npy"
                p.parent.mkdir(parents=True, exist_ok=True)
                np.save(p, (cen[rng.integers(0, 30, n)] + 0.3 * rng.standard_normal((n, d))).astype(np.float32))
    cmd = [sys.executable, os.path.join(ROOT, "svc_train_retrieval.py"), "--compress-features-after", "2000",
           "--n-clusters", "400", "--prefix", "t_"]
    r = subprocess.run(cmd, cwd=tmp_path, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert "create hubert index for speaker alice" in r.stderr and "done!" in r.stderr
    monkeypatch.chdir(tmp_path)
    for spk, ntotal in (("alice", 400), ("bob", 900)):
        args = Namespace(enable_retrieval=True, spk=f"x/{spk}.npy", retrieval_index_prefix="t_", hubert_index_path=None,
                         whisper_index_path=None, retrieval_ratio=0.5, n_retrieval_vectors=3)
        ret = R.create_retrival(args, hp)
        for feat, index, d in (("hubert", ret._hubert_index, hp.vits.vec_dim), ("whisper", ret._whisper_index, hp.vits.ppg_dim)):
            ix = R.read_ivf_flat(base / "indexes" / spk / f"t_{feat}.index")
            assert (ix.ntotal, ix.d, ix.nlist) == (ntotal, d, RT.default_nlist(ntotal))
            q = torch.from_numpy(ix.vectors[:16]).cuda()
            assert index.retriv(q).shape == (16, d)
    r = subprocess.run(cmd + ["--speakers", "bob"], cwd=tmp_path, capture_output=True, text=True, timeout=900)
    assert r.returncode != 0 and "FileExistsError" in r.stderr
