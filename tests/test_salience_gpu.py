"""Salience-based F0 on the device (svcb_salience_f0_ragged, svcb_salience_dp_ragged, salience_f0.py,
preprocess_f0_salience.py, pitch_inference.py --f0).

Stage by stage against the fp64 oracle on the fixture (tests/golden/salience_synth.npz): the binned spectrogram Y and
the salience Z within 1e-9 relative (1e-12 of the item's maximum as the floor), away from STFT bins whose oracle
frequency lies within 1e-6 Hz of a bin edge or of 45 / 1760 Hz or rests on a rounding-noise phase, with a floor on the
share left to compare; the device's DP fed the oracle's Z gives the oracle's path wherever the decisions that fix it have a relative margin above 1e-9, and a path whose score is within 1e-9 of the
optimum elsewhere; on integer-valued Z with exact ties the paths are identical (the first index of the maximum).  The
share of frames on the float32 oracle's bin measures the distance to the reference's precision.  Each item's F0 is
bitwise the same alone, in ragged batches and in any order; short items are refused before any launch; silence gives
45 Hz and no NaN.  The command lines end to end equal compute_f0_salience called directly."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy.io import wavfile

from oracle import salience_oracle as O
from tests.util import ROOT
from whisper_vits_svc_b200 import _lib, hostio, salience_f0

pytestmark = pytest.mark.gpu

GROUP = 128   # items per pass (csrc/salience_f0_api.cu SF_GROUP)
SAME_BIN_GATE = 0.975  # share of fixture frames on the float32 oracle's bin: 0.9786 measured (DESIGN.md §8)
MIN_Y_COMPARED = 0.96         # share of each item's Y elements left after the exclusions (0.9615 at the least, tone_1000)
MIN_Z_FRAMES_COMPARED = 0.9   # share of each item's frames compared on Z (0.922 at the least, under_chord)
pcm = lambda x: np.clip(np.rint(x * 32767), -32768, 32767).astype(np.int16)


def _raw(clips, taps=False):
    ex = salience_f0.Extractor("cuda")
    try:
        out = ex.raw(clips, taps)
        if taps:
            return [tuple(t.cpu().numpy() for t in o) for o in out]
        return [f.cpu().numpy() for f in out]
    finally:
        ex.close()


def _fixture():
    g = O.load_golden()
    return {k: d for k, d in g.items() if d["x"].shape[0] >= O.MIN_SAMPLES}


def _near_edge(inst_f):
    """[K, F] True where the oracle's instantaneous frequency lies within 1e-6 Hz of a bin edge or of 45 / 1760 Hz."""
    edges = np.sort(np.concatenate([[O.F_MIN, O.F_MAX], O.F_MIN * 2.0 ** ((np.arange(O.B) + 0.5) / 120)]))
    pos = np.searchsorted(edges, inst_f)
    lo = np.abs(inst_f - edges[np.clip(pos - 1, 0, edges.shape[0] - 1)])
    hi = np.abs(inst_f - edges[np.clip(pos, 0, edges.shape[0] - 1)])
    return np.minimum(lo, hi) <= 1e-6


def _nearest_bin(f):
    """The log-frequency bin nearest to each frequency, clipped into 0 .. 635 (45 and 1760 Hz included)."""
    b = np.floor(120 * np.log2(np.maximum(f, 1.0) / O.F_MIN) + 0.5)
    return np.clip(b, 0, O.B - 1).astype(np.int64)


def _close(got, want, mask):
    floor = 1e-12 * np.abs(want).max()
    err = np.abs(got - want)[mask]
    ok = err <= 1e-9 * np.abs(want)[mask] + floor
    return bool(ok.all()), float((err / (np.abs(want)[mask] + floor + 1e-300)).max(initial=0.0))


def _ill_conditioned(X, P):
    """[K, F] True where a bin's instantaneous frequency rests on a rounding-noise phase (its coefficient in the frame
    or in the one before is below 1e-9 of the item's largest) while its power counts (above 1e-13 of the largest).
    An exactly bin-centred tone leaves only rounding noise outside its main lobe in the frames it fills, so where it
    stops inside the next window that frame's leakage gets a random frequency in any implementation."""
    A = np.abs(X)
    noisy = A < 1e-9 * A.max()
    bad = noisy.copy()
    bad[:, 1:] |= noisy[:, :-1]
    bad[:, 0] = bad[:, 1] if X.shape[1] > 1 else bad[:, 0]   # frame 0 takes frame 1's frequencies
    return bad & (P > 1e-13 * P.max())


def test_stage_taps():
    g = _fixture()
    names = sorted(g)
    out = _raw([g[k]["x"] for k in names], taps=True)
    worst_y = worst_z = 0.0
    z_frames = all_frames = 0
    for k, (f0, Y, Z, path) in zip(names, out):
        info = {}
        with np.errstate(all="ignore"):
            O.salience_f0(g[k]["x"], np.float64, info)
        F = info["Y"].shape[1]
        assert Y.shape == Z.shape == (O.B, F) and f0.shape == path.shape == (F,), k
        X = O.stft(g[k]["x"])
        near = _near_edge(info["inst_f"])          # [1025, F]
        ill = _ill_conditioned(X, np.abs(X) ** 2)
        # a near-edge STFT bin may land on either side of its edge: exclude both log-frequency bins in that frame;
        # an ill-conditioned one anywhere within 25 Hz of its centre
        ymask = np.ones_like(Y, bool)
        kk, tt = np.nonzero(near)
        for b in _nearest_bin(info["inst_f"][kk, tt]) + np.array([[-1], [0], [1]]):
            ok = (b >= 0) & (b < O.B)
            ymask[b[ok], tt[ok]] = False
        for kq, t in zip(*np.nonzero(ill)):
            lo, hi = _nearest_bin(np.array([7.8125 * kq - 26.0, 7.8125 * kq + 26.0]))
            ymask[lo:hi + 1, t] = False
        ok, wy = _close(Y, info["Y"], ymask)
        assert ok, (k, wy)
        bad_col = near.any(axis=0) | ill.any(axis=0)
        zmask = np.broadcast_to(~bad_col, Z.shape)
        # the exclusions come from the oracle alone; they must leave nearly everything compared
        assert ymask.mean() >= MIN_Y_COMPARED and (~bad_col).mean() >= MIN_Z_FRAMES_COMPARED, \
            (k, ymask.mean(), (~bad_col).mean())
        z_frames += int((~bad_col).sum())
        all_frames += F
        ok, wz = _close(Z, info["Z"], zmask)
        assert ok, (k, wz)
        assert not np.isnan(Z).any() and not np.isnan(f0).any()
        np.testing.assert_allclose(f0, O.bin_hz()[path], rtol=1e-15, atol=0)   # the bin table within an ulp of numpy's
        worst_y, worst_z = max(worst_y, wy), max(worst_z, wz)
        print(f"{k}: Y {wy:.2e}, Z {wz:.2e}, frames compared for Z {int((~bad_col).sum())} of {F}")
    print(f"worst relative difference: Y {worst_y:.2e}, Z {worst_z:.2e}; Z compared on {z_frames} of {all_frames} frames")
    assert z_frames >= 0.95 * all_frames


def _chain_ok(path, eta, margin, Z):
    """The device path equals the oracle's on every frame fixed by decisions with margin > 1e-9 (from the end back to
    the first small one); from there on, the device path's score is within 1e-9 of the optimum."""
    F = eta.shape[0]
    n = F - 1
    while n >= 0 and margin[n] > 1e-9:
        if path[n] != eta[n]:
            return False
        n -= 1
    if n < 0:
        return True
    best, mine = O.path_score(Z, eta), O.path_score(Z, path)
    return abs(mine - best) <= 1e-9 * abs(best)


def test_dp_on_oracle_salience():
    g = _fixture()
    names = sorted(g)
    zs, infos = [], []
    for k in names:
        info = {}
        with np.errstate(all="ignore"):
            O.salience_f0(g[k]["x"], np.float64, info)
        zs.append(torch.from_numpy(info["Z"]))
        infos.append(info)
    paths = salience_f0.dp_paths(zs)
    for k, p, info in zip(names, paths, infos):
        assert p.shape == info["eta"].shape
        assert _chain_ok(p, info["eta"], info["margin"], info["Z"]), k


def test_dp_exact_ties():
    """Integer-valued Z from {0, 1, 2}: columns with equal tracks, a constant stretch and a silent one.  Sums of the
    same logs in the same order are equal on both sides, so every tie is exact and the first index must win."""
    vals = np.array([0.0, 1.0, 2.0]) + O.EPS32
    assert np.array_equal(np.log(vals), torch.log(torch.from_numpy(vals).cuda()).cpu().numpy())
    rng = np.random.default_rng(9)
    zs = []
    for F in (1, 2, 9, 40, 77):
        Z = np.zeros((O.B, F))
        Z[rng.integers(0, O.B, 6)] = 1.0       # constant tracks tie along their length
        Z[[100, 106, 300, 500], :] = 2.0       # equal tracks inside and beyond the 5-bin band
        Z[:, F // 3:F // 2] = 0.0              # a silent stretch: every bin ties
        Z[rng.integers(0, O.B, F), np.arange(F)] = rng.integers(0, 3, F)
        zs.append(Z)
    zs.append(np.full((O.B, 5), 1.0))
    paths = salience_f0.dp_paths([torch.from_numpy(z) for z in zs])
    for Z, p in zip(zs, paths):
        assert np.array_equal(p, O.dp(Z)), Z.shape
    # offsets that start past 0: the items are read at the given offsets, the paths written from path[0]
    skip = 3
    flat = torch.from_numpy(np.concatenate([np.full(O.B * skip, np.nan)] + [z.reshape(-1) for z in zs])).cuda()
    fo = _lib.offsets([skip] + [z.shape[1] for z in zs])
    offs = (ctypes.c_int64 * (len(zs) + 1))(*list(fo)[1:])   # skip, skip + F_0, ...
    path = torch.full((fo[-1] - skip,), -1, dtype=torch.int32, device="cuda")
    ws = torch.empty(_lib.load().svcb_salience_dp_workspace_bytes(fo[-1] - skip), dtype=torch.uint8, device="cuda")
    _lib.call("salience_dp_ragged", flat.data_ptr(), offs, len(zs), path.data_ptr(), ws.data_ptr(), ws.numel())
    assert np.array_equal(path.cpu().numpy(), np.concatenate(paths))


def test_against_reference_precision():
    g = _fixture()
    names = sorted(g)
    out = _raw([g[k]["x"] for k in names], taps=True)
    same = total = 0
    for k, (_, _, _, path) in zip(names, out):
        same += int((path == g[k]["eta32"]).sum())
        total += path.shape[0]
        print(f"{k}: {np.mean(path == g[k]['eta32']):.3f} of frames on the float32 oracle's bin, "
              f"{np.mean(path == g[k]['eta64']):.3f} on the fp64 oracle's")
    share = same / total
    print(f"share of fixture frames on the float32 oracle's bin: {share:.4f} ({same} / {total})")
    assert share >= SAME_BIN_GATE


def _clip(n, rng):
    tr = np.full(n, rng.uniform(80, 900))
    return (O.tone(tr, rng) + 0.001 * rng.standard_normal(n)).astype(np.float32)


def test_batch_invariance_and_order():
    rng = np.random.default_rng(7)
    g = _fixture()
    clips = [g[k]["x"] for k in sorted(g)]
    for n in (320, 321, 639, 640, 2047, 2048, 2049, 4807, 33333):
        clips.append(_clip(n, rng))
    lone = [_raw([c])[0] for c in clips]
    for c, f in zip(clips, lone):
        assert f.shape == (salience_f0.frames_of(c.shape[0]),)
    for _ in range(2):
        order = rng.permutation(len(clips))
        outs = _raw([clips[i] for i in order])
        for o, i in zip(outs, order):
            assert np.array_equal(o, lone[i]), (i, clips[i].shape)


def test_more_than_one_pass():
    rng = np.random.default_rng(3)
    clips = [_clip(int(rng.integers(320, 4000)), rng) for _ in range(GROUP + 7)]
    outs = _raw(clips)
    for i in (0, 5, GROUP - 1, GROUP, len(clips) - 1):
        assert np.array_equal(outs[i], _raw([clips[i]])[0]), i


def test_short_items_rejected_and_silence():
    lib = _lib.load()
    x = torch.zeros(4000, dtype=torch.float32, device="cuda")
    f0 = torch.full((64,), 7.0, dtype=torch.float64, device="cuda")
    ws = torch.empty(lib.svcb_salience_f0_workspace_bytes(4000, 2), dtype=torch.uint8, device="cuda")
    call = lambda offs, nbytes=ws.numel(): _lib.call(
        "salience_f0_ragged", x.data_ptr(), (ctypes.c_int64 * len(offs))(*offs), len(offs) - 1, f0.data_ptr(), None,
        None, None, ws.data_ptr(), nbytes)
    for offs in ([0, 319, 3500], [0, 2000, 1900], [-1, 1800, 3600], [0, 0, 2000]):
        with pytest.raises(_lib.SvcbError, match="svcb_salience_f0_ragged"):
            call(offs)
    with pytest.raises(_lib.SvcbError, match="one 320-sample hop"):
        call([0, 2000, 2319])
    with pytest.raises(_lib.SvcbError, match="need at least one item"):
        call([0])
    with pytest.raises(_lib.SvcbError, match="workspace"):
        call([0, 2000, 4000], 1024)
    with pytest.raises(_lib.SvcbError, match="svcb_salience_f0_ragged"):
        salience_f0.f0_batch([np.zeros(2000), np.zeros(300)])
    torch.cuda.synchronize()
    assert torch.all(f0 == 7.0)   # nothing was launched
    assert salience_f0.f0_batch([]) == []
    # silent items, alone and beside a tone: 45 Hz everywhere, no NaN in any tap
    rng = np.random.default_rng(1)
    out = _raw([np.zeros(5000, np.float32), _clip(9000, rng), np.zeros(320, np.float32)], taps=True)
    for i in (0, 2):
        f, Y, Z, p = out[i]
        assert np.all(f == 45.0) and not p.any() and not Y.any() and not Z.any()
    for t in out[1]:
        assert not np.isnan(t).any()


def test_cli_end_to_end(tmp_path):
    g = O.load_golden()
    files = {"spk_a/glide": (16000, pcm(g["glide"]["x"])), "spk_a/vib": (16000, pcm(g["vibrato"]["x"])),
             "spk_b/chord": (16000, pcm(g["under_chord"]["x"])), "spk_b/silence": (16000, pcm(g["silence"]["x"])),
             "spk_b/low8k": (8000, pcm(g["tone_220"]["x"][::2])), "spk_b/edge": (16000, pcm(g["edge_320"]["x"])),
             "spk_b/tiny": (16000, pcm(g["edge_319"]["x"]))}
    for name, (sr, x) in files.items():
        os.makedirs(tmp_path / "wav" / os.path.dirname(name), exist_ok=True)
        wavfile.write(tmp_path / "wav" / f"{name}.wav", sr, x)
    (tmp_path / "wav" / "spk_b" / "broken.wav").write_bytes(b"RIFF....")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "preprocess_f0_salience.py"), "-w", "wav", "-p", "pit", "-t",
                        "2", "--batch", "3"], cwd=tmp_path, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert r.stdout.splitlines()[:2] == ["wav", "pit"]
    assert "tiny.wav" in r.stderr and "broken.wav" in r.stderr and "2 of 8 files failed" in r.stderr
    assert not (tmp_path / "pit" / "spk_b" / "broken.pit.npy").exists()
    for name in files:
        p = tmp_path / "pit" / f"{name}.pit.npy"
        if name.endswith("tiny"):
            assert not p.exists()
            continue
        want = salience_f0.compute_f0_salience(str(tmp_path / "wav" / f"{name}.wav"))
        got = np.load(p)
        assert got.dtype == np.float64 and np.array_equal(got, want), name
    # pitch_inference.py --f0 salience / mouth write what the library computes, through the same save_csv_pitch
    wav = str(tmp_path / "wav" / "spk_a" / "glide.wav")
    from whisper_vits_svc_b200 import praat_f0
    for choice, fn in (("salience", salience_f0.compute_f0_salience), ("mouth", praat_f0.compute_f0_mouth)):
        r = subprocess.run([sys.executable, os.path.join(ROOT, "pitch_inference.py"), "-w", wav, "-p", f"{choice}.csv",
                            "--f0", choice], cwd=tmp_path, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
        assert r.stdout.splitlines()[:2] == [wav, f"{choice}.csv"]
        hostio.save_csv_pitch(fn(wav), str(tmp_path / f"{choice}_direct.csv"))
        assert (tmp_path / f"{choice}.csv").read_bytes() == (tmp_path / f"{choice}_direct.csv").read_bytes(), choice


_SEEDED = ("import runpy, sys, numpy, torch; torch.manual_seed(11); numpy.random.seed(11); "
           "sys.argv = {argv!r}; runpy.run_path({script!r}, run_name='__main__')")


def test_pitch_inference_default_is_crepe(tmp_path):
    """No --f0: byte for byte the CSV that crepe_infer.pred_pit writes (the path pitch_inference.py took before --f0),
    both run in fresh processes with torch and numpy seeded alike, so CREPE's 0.001 noise and its +-20 cent dither are
    the same draws.  --f0 sing is the same path."""
    from whisper_vits_svc_b200 import synth
    (tmp_path / "crepe" / "assets").mkdir(parents=True)
    torch.save(synth.crepe_checkpoint(3, "full"), tmp_path / "crepe" / "assets" / "full.pth")
    x = O.load_golden()["glide"]["x"]
    wavfile.write(tmp_path / "z.wav", 16000, pcm(x))
    (tmp_path / "direct.py").write_text(
        "import sys\n"
        "from whisper_vits_svc_b200 import crepe_infer as C\n"
        "C.pred_pit(C.load_model('crepe/assets/full.pth', 'cuda'), sys.argv[1], sys.argv[2])\n")
    env = dict(os.environ, PYTHONPATH=ROOT)
    cli = os.path.join(ROOT, "pitch_inference.py")
    runs = {"cli.csv": [cli, "-w", "z.wav", "-p", "cli.csv"], "sing.csv": [cli, "-w", "z.wav", "-p", "sing.csv", "--f0", "sing"],
            "direct.csv": [str(tmp_path / "direct.py"), "z.wav", "direct.csv"]}
    for argv in runs.values():
        r = subprocess.run([sys.executable, "-c", _SEEDED.format(argv=argv, script=argv[0])], cwd=tmp_path, env=env,
                           capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
    want = (tmp_path / "direct.csv").read_bytes()
    assert len(want.splitlines()) == 2 * (x.shape[0] // 320 + 1)
    assert (tmp_path / "cli.csv").read_bytes() == want
    assert (tmp_path / "sing.csv").read_bytes() == want
