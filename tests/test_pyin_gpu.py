"""pYIN F0 on the device (svcb_pyin_f0_ragged, svcb_pyin_dp_ragged, pyin_f0.py, preprocess_f0_pyin.py,
pitch_inference.py --f0 pyin), against the fixture the numpy oracle wrote (tests/golden/pyin_synth.npz).

The CMNDF tap is within 1e-12 of the fixture's; the device's Viterbi on the fixture's observations gives the fixture's
path on every frame, and on built ties and winning off-band predecessors the oracle's banded path (which
test_pyin_cpu.py pins to the reference's dense Viterbi).  End to end, a frame whose observation column or f0 differs
from the fixture must rest on a decision the oracle found within 1e-9 of flipping (oracle.pyin_oracle.gap: |a - b| over
max(1, |a|, |b|)), and every clip without such a frame
matches the fixture's f0 and conf within 1e-12.  Each item is bitwise the same alone and in a ragged batch; the command
lines write what the library computes, on one rank and on two."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy.io import wavfile

from oracle import pyin_oracle as O
from tests.ranks import RANK_PID_LINES, torchrun
from tests.util import ROOT
from whisper_vits_svc_b200 import _lib, hostio, pyin_f0

pytestmark = pytest.mark.gpu

MARGIN = 1e-9
TIMEOUT = 900
pcm = lambda x: np.clip(np.rint(x * 32767), -32768, 32767).astype(np.int16)


def _raw(clips, taps=False):
    ex = pyin_f0.Extractor("cuda")
    try:
        return [tuple(t.cpu().numpy() for t in o) for o in ex.raw(clips, taps)]
    finally:
        ex.close()


@pytest.fixture(scope="module")
def golden():
    g = O.load_golden()
    names = sorted(g)
    return g, names, _raw([g[k]["x"] for k in names], taps=True)


def test_cmndf_tap(golden):
    g, names, out = golden
    worst = 0.0
    for k, (f0, conf, cm, obs, path) in zip(names, out):
        want = g[k]["cmndf"]
        assert cm.shape == want.shape == (O.LAGS, O.n_frames(g[k]["x"].shape[0])), k
        assert obs.shape == (O.S, want.shape[1]) and f0.shape == conf.shape == path.shape == (want.shape[1],), k
        err = float((np.abs(cm - want) / np.maximum(1.0, np.abs(want))).max())
        worst = max(worst, err)
        assert err <= 1e-12, (k, err)
    print(f"CMNDF: worst max-abs over max(1, |x|) {worst:.2e}")


def test_end_to_end_against_fixture(golden):
    g, names, out = golden
    flagged = []
    for k, (f0, conf, cm, obs, path) in zip(names, out):
        d = g[k]
        differs = (obs != d["O"]).any(axis=0) | (f0 != d["f0"])
        for m in np.flatnonzero(differs):
            flagged.append((k, int(m), float(d["margin"][m])))
            assert d["margin"][m] < MARGIN, (k, m, d["margin"][m])
        if not differs.any():
            assert np.array_equal(obs, d["O"]) and np.array_equal(path, d["path"]), k
            np.testing.assert_allclose(f0, d["f0"], rtol=1e-12, atol=0, err_msg=k)
            np.testing.assert_allclose(conf, d["conf"], rtol=1e-12, atol=0, err_msg=k)
        assert not np.isnan(f0).any() and not np.isnan(conf).any(), k
    print(f"frames differing from the fixture (all with margin < {MARGIN}): {flagged}")


def test_dp_on_fixture_observations(golden):
    g, names, _ = golden
    paths = pyin_f0.dp_paths([g[k]["O"] for k in names])
    for k, p in zip(names, paths):
        assert np.array_equal(p, g[k]["path"]), k


def _built_cases():
    """Observations with exact ties (flat and repeated columns), with an off-band predecessor far enough ahead of the
    whole band to win (a spike hundreds of nats above the rest), and with off-band predecessors whose D differ by less
    than log(tiny) + D can hold."""
    rng = np.random.default_rng(5)
    cases = [np.full((O.S, 6), 1.0 / O.S)]
    o = np.zeros((O.S, 9))
    o[[40, 300, 600], :] = 0.25
    o[O.B:, :] = 0.25 / O.B
    cases.append(o)
    o = np.zeros((O.S, 5))
    o[100, 0] = 1.0
    o[400, 1:] = 1.0
    cases.append(o)                       # a jump of 300 bins: off-band, yet its predecessor wins
    o = np.full((O.S, 7), 1e-250)
    o[rng.integers(0, O.S, 7), np.arange(7)] = 1.0
    cases.append(o)
    cases.append(rng.random((O.S, 1)))
    for d in (1e-15, 5e-15, 1e-14):        # off-band predecessors that log(tiny) + D rounds to one value
        o = np.zeros((O.S, 2))
        o[400, 0] = 1.0
        o[100, 0] = 1.0 - d
        o[700, 1] = 1.0
        cases.append(o)
    return cases


def test_dp_built_ties_and_off_band():
    cases = _built_cases()
    paths = pyin_f0.dp_paths(cases)
    for i, (o, p) in enumerate(zip(cases, paths)):
        assert np.array_equal(p, O.viterbi_banded(o)), i
    assert paths[2][1] == 400 and paths[2][0] == 100
    assert list(paths[5]) == [100, 700]    # the first k of the rounded maximum, not the argmax of D


def test_ragged_batch_equals_lone_calls():
    rng = np.random.default_rng(7)
    g = O.load_golden()
    clips = [g[k]["x"] for k in sorted(g)]
    clips += [np.float32(rng.standard_normal(1)), O.tone(np.full(30 * O.FS, 190.0), rng).astype(np.float32),
              np.float32(0.2 * rng.standard_normal(3 * O.FS + 99)), np.zeros(1, np.float32)]
    lone = [_raw([c])[0] for c in clips]
    for c, (f, cf) in zip(clips, lone):
        assert f.shape == cf.shape == (pyin_f0.frames_of(c.shape[0]),)
    order = rng.permutation(len(clips))
    outs = _raw([clips[i] for i in order])
    for (f, cf), i in zip(outs, order):
        assert np.array_equal(f, lone[i][0]) and np.array_equal(cf, lone[i][1]), (i, clips[i].shape)
    # more than one pass of 128 items
    many = [clips[i % len(clips)] for i in range(131)]
    outs = _raw(many)
    for i in (0, 127, 128, 130):
        assert np.array_equal(outs[i][0], lone[i % len(clips)][0]), i


def test_status_codes():
    lib = _lib.load()
    x = torch.zeros(4000, dtype=torch.float32, device="cuda")
    f0 = torch.full((64,), 7.0, dtype=torch.float64, device="cuda")
    conf = torch.empty_like(f0)
    tab = torch.from_numpy(pyin_f0.tables()).cuda()
    need = lib.svcb_pyin_f0_workspace_bytes(4000, 2)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")

    def status(offs, nbytes=need):
        with torch.cuda.device(0):
            return lib.svcb_pyin_f0_ragged(x.data_ptr(), (ctypes.c_int64 * len(offs))(*offs), len(offs) - 1,
                                           tab.data_ptr(), f0.data_ptr(), conf.data_ptr(), None, None, None,
                                           ws.data_ptr(), nbytes, _lib.stream())
    assert status([0, 2000, 4000], 1024) == -6          # SVCB_E_WORKSPACE
    assert status([0, 2000, 4000], need - 1) == -6
    assert status([0, 0, 2000]) == -1                   # SVCB_E_BAD_SHAPE: an empty item
    assert status([0, 2000, 1900]) == -1                # decreasing offsets
    assert status([-1, 1800, 3600]) == -1
    assert status([0]) == -1
    with pytest.raises(_lib.SvcbError, match="svcb_pyin_dp_ragged"):
        pyin_f0.dp_paths([np.zeros((O.S, 3)), np.zeros((O.S, 0))])
    torch.cuda.synchronize()
    assert torch.all(f0 == 7.0)                          # nothing was launched
    assert status([0, 2000, 4000]) == 0
    assert pyin_f0.f0_batch([]) == [] and pyin_f0.dp_paths([]) == []


def test_compute_f0_pyin_and_cli(tmp_path):
    g = O.load_golden()
    files = {"spk_a/glide": (16000, g["glide"]["x"]), "spk_a/vib": (16000, g["vibrato"]["x"]),
             "spk_b/noise": (16000, g["noise"]["x"]), "spk_b/low8k": (8000, g["tone_220"]["x"][::2]),
             "spk_b/one": (16000, g["edge_1"]["x"])}
    for name, (sr, x) in files.items():
        os.makedirs(tmp_path / "wav" / os.path.dirname(name), exist_ok=True)
        wavfile.write(tmp_path / "wav" / f"{name}.wav", sr, pcm(x))
    wavfile.write(tmp_path / "wav" / "spk_b" / "empty.wav", 16000, np.zeros(0, np.int16))
    (tmp_path / "wav" / "spk_b" / "broken.wav").write_bytes(b"RIFF....")
    from whisper_vits_svc_b200 import hubert_infer
    p = str(tmp_path / "wav" / "spk_a" / "glide.wav")
    want = pyin_f0.compute_f0_pyin(p)
    assert np.array_equal(want, pyin_f0.f0_batch([hubert_infer.load_audio(p, 16000)])[0])
    r = subprocess.run([sys.executable, os.path.join(ROOT, "preprocess_f0_pyin.py"), "-w", "wav", "-p", "pit", "-t",
                        "2", "--batch", "2"], cwd=tmp_path, capture_output=True, text=True, timeout=TIMEOUT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert r.stdout.splitlines()[:2] == ["wav", "pit"]
    assert "empty.wav" in r.stderr and "broken.wav" in r.stderr and "2 of 7 files failed" in r.stderr
    for name in files:
        got = np.load(tmp_path / "pit" / f"{name}.pit.npy")
        want = pyin_f0.compute_f0_pyin(str(tmp_path / "wav" / f"{name}.wav"))
        assert got.dtype == np.float64 and np.array_equal(got, want), name
    assert not (tmp_path / "pit" / "spk_b" / "empty.pit.npy").exists()
    r = subprocess.run([sys.executable, os.path.join(ROOT, "pitch_inference.py"), "-w", p, "-p", "pyin.csv", "--f0",
                        "pyin"], cwd=tmp_path, capture_output=True, text=True, timeout=TIMEOUT)
    assert r.returncode == 0, r.stderr[-3000:]
    hostio.save_csv_pitch(pyin_f0.compute_f0_pyin(p), str(tmp_path / "direct.csv"))
    assert (tmp_path / "pyin.csv").read_bytes() == (tmp_path / "direct.csv").read_bytes()


WRAPPER = ("import runpy, sys\n"
           "sys.argv = sys.argv[1:]\n"
           "runpy.run_path(sys.argv[0], run_name='__main__')\n")


def test_two_ranks_equal_one_process(tmp_path):
    rng = np.random.default_rng(3)
    for root in ("two", "one"):
        for i, sec in enumerate((0.4, 1.3, 2.2, 0.7, 3.1)):
            x = O.tone(np.full(int(sec * O.FS), 120.0 + 40 * i), np.random.default_rng(i))
            d = tmp_path / root / "wav" / f"spk{i % 2}"
            d.mkdir(parents=True, exist_ok=True)
            wavfile.write(d / f"f{i}.wav", 16000, pcm(x))
    del rng
    (tmp_path / "two" / "wrapper.py").write_text(RANK_PID_LINES + WRAPPER)
    env = dict(os.environ, CUDA_VISIBLE_DEVICES=os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0],
               OMP_NUM_THREADS="1", PYTHONPATH=ROOT)
    code, out, err = torchrun(["wrapper.py", os.path.join(ROOT, "preprocess_f0_pyin.py"), "-w", "wav", "-p", "pit"],
                              2, tmp_path / "two", env, TIMEOUT, tmp_path / "two")
    assert code == 0, err[-3000:]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "preprocess_f0_pyin.py"), "-w", "wav", "-p", "pit"],
                       cwd=tmp_path / "one", capture_output=True, text=True, timeout=TIMEOUT)
    assert r.returncode == 0, r.stderr[-3000:]
    files = lambda root: sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs)
    two, one = files(tmp_path / "two" / "pit"), files(tmp_path / "one" / "pit")
    assert two == one and len(one) == 5
    for f in one:
        assert (tmp_path / "two" / "pit" / f).read_bytes() == (tmp_path / "one" / "pit" / f).read_bytes(), f
