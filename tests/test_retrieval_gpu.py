"""Feature retrieval on the device (csrc/retrieval_api.cu) against the numpy oracle (oracle/retrieval_oracle.py) and the
goldens of the unmodified reference."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import retrieval_oracle as RO
from oracle import svc_oracle as O
from tests.util import ROOT
from whisper_vits_svc_b200 import retrieval as R

pytestmark = pytest.mark.gpu


def _index(d, nlist, nprobe, seed):
    # a few vectors per list at nlist = 5128 keep the fixture small; the other sizes hold 0 .. 13 per list,
    # so some lists are shorter than k and some are empty
    sizes = np.random.default_rng(seed).integers(0, 5 if nlist > 1000 else 14, nlist)
    if nlist == 1:
        sizes[:] = 40
    cen, lists = RO.clustered_index(seed, d, nlist, sizes)
    return RO.from_parts(cen, lists, nprobe)


def _queries(ix, M, seed):
    rng = np.random.default_rng(seed)
    return (ix.centroids[rng.integers(0, ix.nlist, M)] + 0.4 * rng.standard_normal((M, ix.d))).astype(np.float32)


def _ambiguous(ix, x, nprobe, k):
    """Rows whose selection is decided by less than the stated float64 margin: the coarse boundary within
    1e-5 (|x|^2 + |c|^2), or two of the k + 1 nearest scanned vectors within 1e-5 dist_k."""
    x64, c64 = x.astype(np.float64), ix.centroids.astype(np.float64)
    out = np.zeros(len(x), bool)
    np_eff = min(nprobe, ix.nlist)
    for m in range(len(x)):
        dc = ((x64[m] - c64) ** 2).sum(1)
        o = np.argsort(dc, kind="stable")
        if ix.nlist > np_eff:
            gap = dc[o[np_eff]] - dc[o[np_eff - 1]]
            if gap < 1e-5 * ((x64[m] ** 2).sum() + (c64[o[np_eff - 1]] ** 2).sum()):
                out[m] = True
                continue
        cand = np.concatenate([np.arange(ix.list_offsets[l], ix.list_offsets[l + 1]) for l in o[:np_eff]])
        if cand.size < 2:
            continue
        dv = np.sort(((x64[m] - ix.vectors[cand].astype(np.float64)) ** 2).sum(1))[:k + 1]
        dk = dv[min(k, dv.size) - 1]
        if (np.diff(dv) < 1e-5 * max(dk, 1e-30)).any():
            out[m] = True
    return out


CASES = []
for _d in (256, 1280):
    for _i, _nl in enumerate((1, 7, 256, 5128)):
        for _j, _np in enumerate((1, 3)):
            _c = 2 * _i + _j
            CASES.append((_d, _nl, _np, (1, 3, 8)[_c % 3], (1, 37, 4097)[(_c + _d // 256) % 3]))


@pytest.mark.parametrize("d,nlist,nprobe,k,M", CASES)
def test_search_and_blend_vs_oracle(d, nlist, nprobe, k, M):
    ix = _index(d, nlist, nprobe, seed=d + nlist + nprobe)
    x = _queries(ix, M, seed=M + k)
    dev = R.DeviceIVFIndex(ix, 0.5, k, "cuda")
    dist, ids = dev.search(torch.from_numpy(x).cuda(), k)
    dist, ids = dist.cpu().numpy(), ids.cpu().numpy()
    dist_o, ids_o, _, vecs_o = RO.search(ix, x, k)
    bad = (ids != ids_o).any(1)
    amb = _ambiguous(ix, x[bad], nprobe, k) if bad.any() else np.zeros(0, bool)
    print(f"d={d} nlist={nlist} nprobe={nprobe} k={k} M={M}: ids differ on {bad.sum()} rows, "
          f"all within the margin: {amb.all() if amb.size else True}; ambiguous fraction {amb.sum() / M:.4f}")
    assert amb.all() and amb.sum() / M < 0.01
    ok = ~bad
    fin = np.isfinite(dist_o)
    assert np.array_equal(np.isfinite(dist[ok]), fin[ok])
    assert np.all(np.abs(dist[ok][fin[ok]] - dist_o[ok][fin[ok]]) <= 1e-5 * np.maximum(dist_o[ok][fin[ok]], 1e-6))
    out = dev.retriv(torch.from_numpy(x).cuda()).cpu().numpy()
    out_o = RO.blend_defined(x, dist_o, vecs_o, 0.5)
    tol = 1e-5 * max(1.0, float(np.abs(x).max()))
    err = float(np.abs(out[ok] - out_o[ok]).max()) if ok.any() else 0.0
    print(f"  blend max-abs {err:.2e} (tol {tol:.1e})")
    assert err <= tol


@pytest.mark.parametrize("name", list(RO.RETRIEVAL_CASES))
def test_goldens(name):
    """Short and empty lists, exact duplicates and queries at a centroid are in the golden queries."""
    ix, g = RO.load_golden(name)
    q, k, ratio = g["queries"], int(g["k"]), float(g["ratio"])
    dev = R.DeviceIVFIndex(ix, ratio, k, "cuda")
    dist, ids = (t.cpu().numpy() for t in dev.search(torch.from_numpy(q).cuda(), k))
    assert np.array_equal(ids, g["search_ids"])
    out = dev.retriv(torch.from_numpy(q)).numpy()   # CPU in, CPU out
    ref = g["retriv"]
    fin = np.isfinite(ref).all(1)
    tol = 1e-5 * max(1.0, float(np.abs(q).max()))
    assert np.abs(out[fin] - ref[fin]).max() <= tol
    # rows the reference leaves NaN follow the defined rules
    _, _, _, vecs = RO.search(ix, q, k)
    dfn = RO.blend_defined(q, g["search_dist"], vecs, ratio)
    assert np.isfinite(out).all() and np.abs(out[~fin] - dfn[~fin]).max() <= tol
    nothing = ~np.isfinite(g["search_dist"]).any(1)
    assert nothing.any() and np.array_equal(out[nothing], q[nothing])   # nothing found: passes through
    assert np.isinf(dist[~np.isfinite(g["search_dist"])]).all() and (ids[~np.isfinite(g["search_dist"])] == -1).all()


def test_degenerate_rows():
    cen, lists = RO.clustered_index(9, 256, 12, sizes=[5, 0, 1, 2, 9, 4, 6, 3, 0, 8, 7, 5])
    ix = RO.from_parts(cen, lists, nprobe=1)
    v = ix.vectors
    x = np.stack([v[0], v[3], cen[1], cen[4], np.zeros(256, np.float32), cen[2], cen[3] + 1e-3, v[10]]).astype(np.float32)
    x[7] = x[6]   # a duplicate row
    dev = R.DeviceIVFIndex(ix, 0.5, 3, "cuda")
    out = dev.retriv(torch.from_numpy(x).cuda()).cpu().numpy()
    dist_o, _, _, vecs_o = RO.search(ix, x, 3)
    out_o = RO.blend_defined(x, dist_o, vecs_o, 0.5)
    assert np.isfinite(out).all()
    assert np.abs(out - out_o).max() <= 1e-5 * max(1.0, float(np.abs(x).max()))
    # an exact duplicate takes the matching vector's value at full weight
    assert np.array_equal(out[0], (np.float32(0.5) * x[0] + np.float32(0.5) * v[0]).astype(np.float32))
    assert np.array_equal(out[2], x[2])   # empty list probed: unchanged


def test_deterministic_and_row_independent():
    ix = _index(1280, 256, 3, seed=77)
    x = _queries(ix, 4097, seed=5)
    x[100] = 0
    dev = R.DeviceIVFIndex(ix, 0.5, 8, "cuda")
    xd = torch.from_numpy(x).cuda()
    a = dev.retriv(xd)
    b = dev.retriv(xd)
    assert torch.equal(a, b)
    da, ia = dev.search(xd, 8)
    assert torch.equal(da, dev.search(xd, 8)[0]) and torch.equal(ia, dev.search(xd, 8)[1])
    assert torch.equal(dev.retriv(xd[100:137]), a[100:137])
    assert torch.equal(dev.retriv(xd[4096:]), a[4096:])
    perm = torch.randperm(4097, generator=torch.Generator().manual_seed(3)).cuda()
    assert torch.equal(dev.retriv(xd[perm]), a[perm])


def test_bad_arguments():
    ix = _index(256, 7, 1, seed=1)
    dev = R.DeviceIVFIndex(ix, 0.5, 3, "cuda")
    with pytest.raises(Exception, match="k <= 32"):
        dev.search(torch.zeros(4, 256, device="cuda"), 33)
    ix.nprobe = 9
    with pytest.raises(R.IndexFormatError):
        R.DeviceIVFIndex(ix, 0.5, 3, "cuda")


# ------------------------------------------------------------------------------------------------ whole path
class _OracleRetrieval:
    def __init__(self, hub, whi, ratio, k):
        self.hub, self.whi, self.ratio, self.k = hub, whi, ratio, k

    def _r(self, ix, x):
        xn = x.numpy()
        dist, _, _, vecs = RO.search(ix, xn, self.k)
        return torch.from_numpy(RO.blend_defined(xn, dist, vecs, self.ratio))

    def retriv_whisper(self, x):
        return self._r(self.whi, x)

    def retriv_hubert(self, x):
        return self._r(self.hub, x)


def _features(hp, n, seed):
    g = torch.Generator().manual_seed(seed)
    ppg = torch.randn(n, hp.vits.ppg_dim, generator=g)
    vec = torch.randn(n, hp.vits.vec_dim, generator=g)
    pit = torch.randint(100, 500, (n,), generator=g).float()
    spk = torch.randn(hp.vits.spk_dim, generator=g) * 0.05
    return ppg, vec, pit, spk


def _feature_index(X, nlist, seed):
    rng = np.random.default_rng(seed)
    cen = X[rng.choice(len(X), nlist, replace=False)] + 0.1 * rng.standard_normal((nlist, X.shape[1])).astype(np.float32)
    lists = []
    for l in range(nlist):
        v = (cen[l] + 0.5 * rng.standard_normal((6, X.shape[1]))).astype(np.float32)
        lists.append((v, np.arange(l * 6, l * 6 + 6)))
    return RO.from_parts(cen, lists)


@pytest.fixture(scope="module")
def model(hp, sd):
    from whisper_vits_svc_b200 import models
    m = models.SynthesizerInfer(hp.data.filter_length // 2 + 1, hp.data.segment_size // hp.data.hop_length, hp)
    m.load_state_dict(sd)
    return m.eval().to("cuda")


def test_svc_infer_with_retrieval(model, hp, sd):
    from whisper_vits_svc_b200 import hostio
    n = 300   # 3 s
    ppg, vec, pit, spk = _features(hp, n, 21)
    hub = _feature_index(vec.numpy(), 11, 1)
    whi = _feature_index(ppg.numpy(), 9, 2)
    g = torch.Generator().manual_seed(22)
    rand_ini = torch.rand(1, 11, generator=g)
    noise = torch.randn(1, n * 320, 11, generator=g)
    eps = torch.randn(1, hp.vits.inter_channels, n, generator=g)
    kw = dict(write_pit_wav=None, rand_ini=rand_ini, noise=noise, eps_fn=lambda i, b, t: eps)
    dev = R.IndexRetrieval(R.DeviceIVFIndex(hub, 0.5, 3, "cuda"), R.DeviceIVFIndex(whi, 0.5, 3, "cuda"))
    out = hostio.svc_infer(model, spk, pit, ppg, vec, hp, "cuda", retrieval=dev, **kw)
    o = _OracleRetrieval(hub, whi, 0.5, 3)
    ppg_o, vec_o = o.retriv_whisper(ppg), o.retriv_hubert(vec)
    assert not torch.equal(ppg_o, ppg)
    src = O.pitch2source(sd, hp, pit[None], rand_ini, noise)
    ref = O.synthesizer_infer(sd, hp, ppg_o[None], vec_o[None], pit[None], spk[None], torch.tensor([n]), src, eps)
    ref = ref[0, 0].numpy()[:-1]
    err = float(np.abs(out - ref).max())
    print(f"svc_infer with retrieval, 3 s: max-abs {err:.3e}")
    assert err <= 1e-3
    # ratio 0: the features pass through bit for bit, and so does the waveform
    dev0 = R.IndexRetrieval(R.DeviceIVFIndex(hub, 0.0, 3, "cuda"), R.DeviceIVFIndex(whi, 0.0, 3, "cuda"))
    a = hostio.svc_infer(model, spk, pit, ppg, vec, hp, "cuda", retrieval=dev0, **kw)
    b = hostio.svc_infer(model, spk, pit, ppg, vec, hp, "cuda", **kw)
    assert np.array_equal(a, b)


def test_cli_enable_retrieval(hp, sd, tmp_path):
    n = 60
    ppg, vec, pit, spk = _features(hp, 2 * n, 31)
    torch.save({"model_g": sd}, tmp_path / "model.pth")
    np.save(tmp_path / "sunny.npy", spk.numpy())
    np.save(tmp_path / "x.ppg.npy", ppg[::2].numpy())
    np.save(tmp_path / "x.vec.npy", vec[::2].numpy())
    (tmp_path / "x.csv").write_text("".join(f"{i},{int(p)}\n" for i, p in enumerate(pit.tolist())))
    d = tmp_path / "data_svc" / "indexes" / "su"   # get_speaker_name_from_path("sunny.npy") == "su"
    d.mkdir(parents=True)
    for name, X, seed in (("hubert", vec.numpy(), 1), ("whisper", ppg.numpy(), 2)):
        ix = _feature_index(X, 5, seed)
        RO.write_ivf_flat(d / f"{name}.index", ix.centroids,
                          [(ix.vectors[ix.list_offsets[l]:ix.list_offsets[l + 1]], ix.ids[ix.list_offsets[l]:ix.list_offsets[l + 1]])
                           for l in range(ix.nlist)])
    cmd = [sys.executable, os.path.join(ROOT, "svc_inference.py"), "--config", os.path.join(ROOT, "configs", "base.yaml"),
           "--model", "model.pth", "--wave", "none.wav", "--spk", "sunny.npy", "--ppg", "x.ppg.npy", "--vec", "x.vec.npy",
           "--pit", "x.csv", "--enable-retrieval"]
    r = subprocess.run(cmd, cwd=tmp_path, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert "load index retrival model" in r.stderr
    from scipy.io import wavfile
    sr, w = wavfile.read(tmp_path / "svc_out.wav")
    assert sr == hp.data.sampling_rate and w.dtype == np.float32 and w.shape == (2 * n * 320 - 1,) and np.isfinite(w).all()
