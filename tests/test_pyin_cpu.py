"""pYIN F0 on the host (oracle/pyin_oracle.py, pyin_f0.py's tables, preprocess_f0_pyin.py's and
pitch_inference.py --f0 pyin's host logic).

The oracle equals the live, unmodified reference (pitch/core/pyin.py with numba) on every fixture clip: f0, conf,
observations and path bitwise.  Its banded Viterbi equals the reference's dense one on seeded observations, built ties
and off-band predecessors that win.  A built frame shows the lag correction taken from the first minimum overall and
the handling of the minima at 16 and 319.  Tones and glides are within 1 % of their true F0; silence, frame 0 and quiet
passages are unvoiced.  The device's host table equals the reference's values, and the fixture is reproduced."""
import importlib.machinery
import importlib.util
import os
import subprocess
import sys
import types

import numpy as np
import pytest
from scipy.io import wavfile

from oracle import pyin_oracle as O
from oracle import ref_import
from tests.util import ROOT
from whisper_vits_svc_b200 import hostio, pyin_f0

CLI = os.path.join(ROOT, "preprocess_f0_pyin.py")
KW = dict(Fs=16000, N=2048, H=160, F_min=50.0, F_max=1000.0)
pcm = lambda x: np.clip(np.rint(x * 32767), -32768, 32767).astype(np.int16)


def _module(name):
    m = types.ModuleType(name)
    m.__spec__ = importlib.machinery.ModuleSpec(name, loader=None)
    return m


@pytest.fixture(scope="module")
def synth():
    return O.synth_items()


@pytest.fixture(scope="module")
def P():
    """pitch.core.pyin of the reference tree; librosa and crepe (imported by pitch/__init__) stubbed empty."""
    if not ref_import.available():
        pytest.skip("reference tree absent")
    pytest.importorskip("numba")
    stubs = {"librosa": _module("librosa"), "crepe": _module("crepe"), "resampy": _module("resampy")}
    saved = {k: sys.modules.get(k) for k in stubs}
    sys.modules.update(stubs)
    sys.path.insert(0, ref_import.REF_ROOT)
    try:
        import pitch.core.pyin as P
        yield P
    finally:
        sys.path.remove(ref_import.REF_ROOT)
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
        for k in [k for k in sys.modules if k == "pitch" or k.startswith("pitch.")]:
            del sys.modules[k]


def _ref_obs(P, x):
    xp = np.concatenate((np.zeros(O.N // 2), x, np.zeros(O.N // 2)))
    return P.yin_multi_thr(xp, O.FS, O.N, O.HOP, O.F_MIN, O.F_MAX, O.thresholds(), O.beta_distr(), O.ABS_MIN_PROB,
                           O.f_axis(), O.VOICING_PROB)


def test_oracle_matches_reference(P, synth):
    A = P.compute_transition_matrix(O.B, O.triang_distr())
    assert np.array_equal(A, O.transition_matrix())
    for name, (x, _) in synth.items():
        info = {}
        f0, conf = O.pyin(x, info)
        with np.errstate(all="ignore"):
            f0_ref, t_ref, conf_ref = P.pyin(x, **KW)
            O_ref, rms, _, _ = _ref_obs(P, x)
            path_ref = P.viterbi_log_likelihood(A, np.ones(O.S) / O.S, O_ref)
        assert np.array_equal(f0, f0_ref), name
        assert np.array_equal(conf, conf_ref), name
        assert np.array_equal(info["O"], O_ref), name
        assert np.array_equal(info["path"], path_ref), name
        assert f0.shape == (O.n_frames(x.shape[0]),) and np.array_equal(t_ref, np.arange(f0.shape[0]) * O.HOP / O.FS)


def _seeded_and_built():
    rng = np.random.default_rng(11)
    cases = []
    for F in (1, 2, 17, 60):
        o = rng.random((O.S, F)) ** 8
        o[rng.random((O.S, F)) < 0.9] = 0.0                 # zeros: log(tiny) entries tie everywhere
        cases.append(o)
    cases.append(np.full((O.S, 6), 1.0 / O.S))             # every state ties
    o = np.zeros((O.S, 9))
    o[[40, 300, 600], :] = 0.25                             # equal tracks in and out of each other's band
    o[O.B:, :] = 0.25 / O.B
    cases.append(o)
    o = np.zeros((O.S, 5))
    o[100, 0] = 1.0
    o[400, 1:] = 1.0                                        # the band of 400 lies 708 nats below state 100
    cases.append(o)
    o = np.zeros((O.S, 4))
    o[[7, 900], 0] = 1.0
    o[[500, 1030], 1:] = 1.0                                # off-band winners that tie with each other
    cases.append(o)
    cases += _absorbed()
    return cases


def _absorbed():
    """Off-band predecessors whose D differ in the last bits: log(tiny) + D rounds them to one value, so the dense
    argmax takes the earlier one (100), not the argmax of D (400)."""
    cases = []
    for d in (1e-15, 5e-15, 1e-14):
        o = np.zeros((O.S, 2))
        o[400, 0] = 1.0
        o[100, 0] = 1.0 - d
        o[700, 1] = 1.0
        cases.append(o)
    return cases


def test_banded_viterbi_equals_dense(P):
    A = P.compute_transition_matrix(O.B, O.triang_distr())
    tabs = O.band(A)
    off_band_wins = 0
    for i, o in enumerate(_seeded_and_built()):
        want = P.viterbi_log_likelihood(A, np.ones(O.S) / O.S, o)
        got = O.viterbi_banded(o, tabs)
        assert np.array_equal(got, want), i
        off_band_wins += int(np.sum(A[got[:-1], got[1:]] == 0))
    assert off_band_wins >= 2
    assert list(O.viterbi_banded(_absorbed()[0], tabs)) == [100, 700]


def test_first_minimum_correction_quirk(P):
    """Two minima, the first (at 40) above every threshold below 0.6: a threshold that only the second (at 100)
    passes takes lag 100 plus the *first* minimum's parabolic offset."""
    c = np.linspace(1.0, 0.9, O.LAGS)
    c[39:42] = [0.7, 0.6, 0.68]
    c[99:102] = [0.3, 0.2, 0.22]
    thr, beta, fa = O.thresholds(), O.beta_distr(), O.f_axis()
    O_ref, lag_ref, val_ref = P.probabilistic_thresholding(c.copy(), thr, O.P_MIN, O.P_MAX, O.ABS_MIN_PROB, fa,
                                                           O.FS, beta)
    Om, lags, vals, _, _ = O.threshold_frame(c, thr, beta, fa)
    assert np.array_equal(Om, O_ref) and np.array_equal(lags, lag_ref) and np.array_equal(vals, val_ref, equal_nan=True)
    x40, _ = O.parabolic(0.7, 0.6, 0.68)
    x100, _ = O.parabolic(0.3, 0.2, 0.22)
    i = int(np.flatnonzero(thr > 0.2)[0])                   # 0.21: only the second minimum is under it
    assert lags[i] == 100 + x40 != 100 + x100
    # a minimum at 16 is interpolated against the inf below it into NaN: never under a threshold, and the first NaN
    # is the frame's argmin; p_corr[0] is then the 0 put in front
    c2 = c.copy()
    c2[16:18] = [0.1, 0.5]
    O_ref, lag_ref, val_ref = P.probabilistic_thresholding(c2.copy(), thr, O.P_MIN, O.P_MAX, O.ABS_MIN_PROB, fa,
                                                           O.FS, beta)
    Om, lags, vals, _, _ = O.threshold_frame(c2, thr, beta, fa)
    assert np.array_equal(Om, O_ref) and np.array_equal(lags, lag_ref) and np.array_equal(vals, val_ref, equal_nan=True)
    assert lags[0] == 16 and np.isnan(vals[0]) and lags[i] == 100


def test_noise_edge_minima_match_reference(P, synth):
    """Noise frames with a minimum at 319 and one whose lag equals its count less one: delete_numba drops the first
    minimum from the interpolation."""
    fr = O.frames(synth["noise"][0])
    C, _ = O.cmndf(fr)
    thr, beta, fa = O.thresholds(), O.beta_distr(), O.f_axis()
    hits = 0
    for m in range(fr.shape[0]):
        c = C[m].copy()
        c[:O.P_MIN] = np.inf
        c[O.P_MAX:] = np.inf
        mins = np.flatnonzero((c[1:-1] < c[:-2]) & (c[1:-1] < c[2:])) + 1
        hits += int(mins.size > 0 and mins[-1] == O.P_MAX - 1 and (mins == mins.size - 1).any())
        with np.errstate(all="ignore"):
            ref = P.probabilistic_thresholding(C[m].copy(), thr, O.P_MIN, O.P_MAX, O.ABS_MIN_PROB, fa, O.FS, beta)
            got = O.threshold_frame(C[m], thr, beta, fa)
        for a, b in zip(ref, got[:3]):
            assert np.array_equal(a, b, equal_nan=True), m
    assert hits >= 1


VOICED = [f"tone_{int(f)}" for f in O.TONES] + ["glide", "second_harmonic"]


@pytest.mark.parametrize("name", VOICED)
def test_ground_truth(synth, name):
    x, tr = synth[name]
    f0, _ = O.pyin(x)
    truth, ok = O.frame_truth(tr)
    ok[0] = False
    assert ok.sum() >= 10
    assert np.all(f0[ok] > 0), name
    rel = np.abs(f0[ok] / truth[ok] - 1)
    assert rel.max() < 0.01, (name, rel.max())
    assert f0[0] == 0


def test_unvoiced(synth):
    for name in ("silence", "quiet", "edge_1", "edge_159"):
        f0, conf = O.pyin(synth[name][0])
        assert not f0.any(), name
        assert not np.isnan(conf).any()
    rms = np.sqrt(np.mean(synth["quiet"][0].astype(np.float64) ** 2))
    assert rms < 0.01


def test_frame_counts():
    for n in (1, 159, 160, 161, 2048, 2049):
        assert O.frames(np.zeros(n, np.float32)).shape == (n // 160 + 1, O.N)
        assert pyin_f0.frames_of(n) == n // 160 + 1
    with pytest.raises(ValueError):
        O.frames(np.zeros(0, np.float32))
    assert (O.B, O.S, O.P_MIN, O.P_MAX, O.LAGS) == (518, 1036, 16, 320, 321) == \
        (pyin_f0.BINS, pyin_f0.STATES, 16, 320, pyin_f0.LAGS)


def test_device_table(P):
    tab = pyin_f0.tables()
    idx, val = O.band(P.compute_transition_matrix(O.B, O.triang_distr()))
    assert np.array_equal(tab[pyin_f0.TAB_THR:pyin_f0.TAB_BETA], O.thresholds())
    assert np.array_equal(tab[pyin_f0.TAB_BETA:pyin_f0.TAB_FAXIS], O.beta_distr())
    assert np.array_equal(tab[pyin_f0.TAB_FAXIS:pyin_f0.TAB_BIDX], O.f_axis())
    assert np.array_equal(tab[pyin_f0.TAB_BIDX:pyin_f0.TAB_BLOG].reshape(O.S, O.BAND), idx)
    assert np.array_equal(tab[pyin_f0.TAB_BLOG:].reshape(O.S, O.BAND), val)
    A = P.compute_transition_matrix(O.B, O.triang_distr())
    tiny = np.finfo(0.).tiny
    assert np.array_equal(val[idx >= 0], np.log(A.T[np.arange(O.S)[:, None], np.maximum(idx, 0)] + tiny)[idx >= 0])
    assert ((idx >= 0).sum(axis=1) <= O.BAND).all()
    hdr = open(os.path.join(ROOT, "include", "svcb.h")).read()
    for key, v in (("THR", 0), ("BETA", 99), ("FAXIS", 198), ("BIDX", 716), ("BLOG", 13148), ("DOUBLES", 25580)):
        assert f"#define SVCB_PYIN_TAB_{key} {v}\n" in hdr
        assert getattr(pyin_f0, f"TAB_{key}") == v


def test_fixture_reproduced(synth):
    g = O.load_golden()
    assert sorted(g) == sorted(synth)
    assert os.path.getsize(O.GOLDEN) < 1 << 20
    for k, d in g.items():
        assert np.array_equal(d["x"], synth[k][0]), k
        info = {}
        f0, conf = O.pyin(d["x"], info)
        assert np.array_equal(d["cmndf"], info["cmndf"].T), k
        assert np.array_equal(d["O"], info["O"]) and np.array_equal(d["path"], info["path"]), k
        assert np.array_equal(d["f0"], f0) and np.array_equal(d["conf"], conf), k
        assert np.array_equal(d["margin"], info["margin"]), k


def _cli():
    spec = importlib.util.spec_from_file_location("preprocess_f0_pyin_cli", CLI)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


class _Fake:
    calls = []

    def __init__(self, device):
        assert device == "cuda"
        self.closed = False
        _Fake.calls.append(self)

    def f0_batch(self, clips):   # the device call, stubbed by the oracle
        return [O.pyin(c)[0] for c in clips]

    def close(self):
        self.closed = True


def test_cli_host_logic(tmp_path, monkeypatch, capsys, synth):
    monkeypatch.chdir(tmp_path)
    for s in ("spk_b", "spk_a"):
        (tmp_path / "wav" / s).mkdir(parents=True)
    wavfile.write(tmp_path / "wav" / "spk_a" / "b.wav", 16000, pcm(synth["vibrato"][0]))
    wavfile.write(tmp_path / "wav" / "spk_a" / "a.wav", 16000, pcm(synth["tone_220"][0]))
    wavfile.write(tmp_path / "wav" / "spk_b" / "one.wav", 16000, pcm(synth["edge_1"][0]))
    wavfile.write(tmp_path / "wav" / "spk_b" / "empty.wav", 16000, np.zeros(0, np.int16))
    (tmp_path / "wav" / "spk_b" / "broken.wav").write_bytes(b"RIFF....")
    (tmp_path / "wav" / "top.wav").write_bytes(b"")   # not in a speaker directory: not taken
    m = _cli()
    assert m.pit_jobs("wav", "pit") == [("wav/spk_a/a.wav", "pit/spk_a/a.pit"), ("wav/spk_a/b.wav", "pit/spk_a/b.pit"),
                                        ("wav/spk_b/broken.wav", "pit/spk_b/broken.pit"),
                                        ("wav/spk_b/empty.wav", "pit/spk_b/empty.pit"),
                                        ("wav/spk_b/one.wav", "pit/spk_b/one.pit")]
    _Fake.calls = []
    monkeypatch.setattr(pyin_f0, "Extractor", _Fake)
    capsys.readouterr()
    assert m.main(["-w", "wav", "-p", "pit", "-t", "2", "--batch", "2"]) == 0
    out, err = capsys.readouterr()
    assert out.splitlines()[:2] == ["wav", "pit"]
    assert len(_Fake.calls) == 1 and _Fake.calls[0].closed
    assert "empty.wav" in err and "no samples" in err and "broken.wav" in err and "2 of 5 files failed" in err
    assert sorted(os.listdir(tmp_path / "pit" / "spk_a")) == ["a.pit.npy", "b.pit.npy"]
    assert sorted(os.listdir(tmp_path / "pit" / "spk_b")) == ["one.pit.npy"]
    from whisper_vits_svc_b200 import hubert_infer
    for s, f in (("spk_a", "a"), ("spk_a", "b"), ("spk_b", "one")):
        x = hubert_infer.load_audio(f"wav/{s}/{f}.wav", 16000)
        got = np.load(tmp_path / "pit" / s / f"{f}.pit.npy")
        assert got.dtype == np.float64 and got.shape == (x.shape[0] // 160 + 1,)
        assert np.array_equal(got, O.pyin(x)[0])


def test_pitch_inference_csv(tmp_path, synth):
    """pitch_inference.py --f0 pyin writes save_csv_pitch of compute_f0_pyin (here the oracle, behind a stub)."""
    x = synth["glide"][0]
    wavfile.write(tmp_path / "g.wav", 16000, pcm(x))
    (tmp_path / "run.py").write_text(
        "import runpy, sys, torch\n"
        "torch.cuda.is_available = lambda: True\n"
        "from oracle import pyin_oracle as O\n"
        "from whisper_vits_svc_b200 import hubert_infer, pyin_f0\n"
        "pyin_f0.compute_f0_pyin = lambda p, d: O.pyin(hubert_infer.load_audio(p, 16000))[0]\n"
        f"sys.argv = [{os.path.join(ROOT, 'pitch_inference.py')!r}, '-w', 'g.wav', '-p', 'g.csv', '--f0', 'pyin']\n"
        "runpy.run_path(sys.argv[0], run_name='__main__')\n")
    r = subprocess.run([sys.executable, "run.py"], cwd=tmp_path, capture_output=True, text=True, timeout=300,
                       env=dict(os.environ, PYTHONPATH=ROOT))
    assert r.returncode == 0, r.stderr[-3000:]
    assert r.stdout.splitlines()[:2] == ["g.wav", "g.csv"]
    from whisper_vits_svc_b200 import hubert_infer
    hostio.save_csv_pitch(O.pyin(hubert_infer.load_audio(str(tmp_path / "g.wav"), 16000))[0], str(tmp_path / "d.csv"))
    assert (tmp_path / "g.csv").read_bytes() == (tmp_path / "d.csv").read_bytes()
    assert len((tmp_path / "g.csv").read_text().splitlines()) == x.shape[0] // 160 + 1
