"""Praat autocorrelation F0 on the host (oracle/praat_f0_oracle.py, praat_f0.frames_of, preprocess_f0_mouth.py's host
logic).

The oracle is checked against the true F0 of synthetic tones, its direct autocorrelation against the FFT form, its
path finder against brute force, and it reproduces its fixture; it is pinned to parselmouth where parselmouth imports.
The CLI's walk, names, dtype, lengths, printed lines and skips run against a stubbed device call, and against the
reference script run with a parselmouth stub built from the oracle."""
import concurrent.futures
import contextlib
import importlib.util
import io
import itertools
import math
import os
import runpy
import sys
import types

import numpy as np
import pytest
from scipy.io import wavfile

from oracle import praat_f0_oracle as O, ref_import
from tests.util import ROOT
from whisper_vits_svc_b200 import praat_f0

CLI = os.path.join(ROOT, "preprocess_f0_mouth.py")
pcm = lambda x: np.clip(np.rint(x * 32767), -32768, 32767).astype(np.int16)


def _cli():
    spec = importlib.util.spec_from_file_location("preprocess_f0_mouth_cli", CLI)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


@pytest.fixture(scope="module")
def synth():
    items = O.synth_items()
    return {k: (x, tr, O.praat_f0_unpadded(x)) for k, (x, tr) in items.items()}


VOICED = [f"tone_{int(f)}" for f in O.TONES] + ["glide", "vibrato", "onsets"]


@pytest.mark.parametrize("name", VOICED)
def test_ground_truth_tones(synth, name):
    """Within 1 % of the true F0 on voiced frames whose window lies 30 ms or more inside a voiced run."""
    x, tr, f0 = synth[name]
    truth, ok = O.frame_truth(tr)
    v = ok & (truth > 0)
    assert v.sum() >= 25
    rel = np.abs(f0[v] - truth[v]) / truth[v]
    assert rel.max() < 0.01, (name, rel.max())


def test_no_octave_errors_on_strong_second_harmonic(synth):
    for f in O.TONES:
        x, tr, f0 = synth[f"tone_{int(f)}"]
        assert O.STRONG2[1] > O.STRONG2[0]
        assert (f0 > 0).all(), f
        ratio = f0 / f
        assert np.all(np.abs(ratio - 1.0) < 0.01), (f, ratio.min(), ratio.max())


def test_silence_and_noise(synth):
    assert not synth["silence"][2].any()
    assert synth["silence"][2].shape == (O.n_frames(synth["silence"][0].shape[0]),)
    f0 = synth["noise"][2]
    assert (f0 == 0).mean() >= 0.95
    assert not O.praat_f0(np.zeros(5000)).any()


def test_frame_count_rule():
    """floor((n dx - 0.1) / 0.01) + 1 at every length within 2 samples of each 160-sample boundary from 1600 to 4800."""
    rng = np.random.default_rng(2)
    assert O.MIN_SAMPLES == praat_f0.MIN_SAMPLES == 1600 and O.PAD == praat_f0.PAD == 6
    assert O.n_frames(1760) == 1 and O.n_frames(1761) == 2   # (0.11 - 0.1) / 0.01 = 0.99999...
    for edge in range(1600, 4801, 160):
        for n in range(edge - 2, edge + 3):
            want = math.floor((n * (1.0 / 16000) - 0.1) / 0.01) + 1 if n >= 1600 else 0
            assert O.n_frames(n) == praat_f0.frames_of(n) == want, n
            if n < 1600:
                with pytest.raises(ValueError):
                    O.praat_f0(rng.standard_normal(n))
                continue
            assert abs(want - (n // 160 - 9)) <= 1
            x = O.tone(np.full(n, 200.0), rng) + 1e-3 * rng.standard_normal(n)
            f = O.praat_f0(x)
            assert f.dtype == np.float64 and f.shape == (want + 12,), n
            lefts = O.frame_lefts(n)
            assert lefts[0] - O.HALF + 1 >= 0 and lefts[-1] + O.HALF <= n - 1


def test_padding(synth):
    x, _, f0 = synth["glide"]
    f = O.praat_f0(x)
    assert f.shape == (f0.shape[0] + 12,)
    assert not f[:6].any() and not f[-6:].any() and np.array_equal(f[6:-6], f0)


def test_direct_autocorrelation_equals_fft(synth):
    """The direct sum (the device's form) and Praat's zero-padded FFT agree to 1e-12 at every lag the candidates read."""
    for name in ("tone_40", "tone_950", "vibrato", "noise", "onsets", "short_1600"):
        x = synth[name][0]
        rd, lpd, gpd = O.frame_data(x)
        rf, lpf, gpf = O.frame_data(x, fft=True)
        assert rd.shape == rf.shape and rd.shape[1] == O.NLAG
        assert np.abs(rd - rf).max() <= 1e-12, (name, np.abs(rd - rf).max())
        assert np.array_equal(lpd, lpf) and gpd == gpf
    assert O.NFFT >= 1.5 * O.W and O.NFFT >= O.W + O.NLAG


def test_viterbi_equals_brute_force():
    rng = np.random.default_rng(4)
    for trial in range(60):
        F = int(rng.integers(1, 6))
        freqs, strengths = [], []
        for _ in range(F):
            k = int(rng.integers(0, 4))
            freqs.append([0.0] + list(rng.uniform(30, 1000, k)))
            strengths.append(list(rng.uniform(0, 2.5, k + 1)))
        path, margin = O.viterbi(freqs, strengths)
        best, arg = -math.inf, None
        for p in itertools.product(*[range(len(f)) for f in freqs]):
            s = O.path_score(freqs, strengths, p)
            if s > best:
                best, arg = s, p
        assert tuple(path) == arg, (trial, path, arg)
        assert abs(O.path_score(freqs, strengths, path) - best) <= 1e-12
    # ties go to the lowest candidate index
    path, margin = O.viterbi([[0.0, 200.0], [0.0, 200.0]], [[1.0, 1.0], [1.0, 1.0]])
    assert path == [0, 0] and margin == 0.0


def test_fixture_reproduced(synth):
    g = O.load_golden()
    assert sorted(g) == sorted(synth)
    assert os.path.getsize(O.GOLDEN) < 1 << 20
    for k, (x, f0) in g.items():
        assert np.array_equal(x, synth[k][0]), k
        got = synth[k][2]
        assert np.array_equal(got > 0, f0 > 0), k
        np.testing.assert_allclose(got, f0, rtol=1e-12, atol=0, err_msg=k)
        info = {}
        O.praat_f0_unpadded(x, info)
        assert info["path_margin"] >= 1e-9 and info["candidate_margin"] >= 1e-12, k


def _tree(tmp_path, items, bad=True):
    for s in ("spk_b", "spk_a"):
        (tmp_path / "wav" / s).mkdir(parents=True)
    wavfile.write(tmp_path / "wav" / "spk_a" / "b.wav", 16000, pcm(items["vibrato"][0]))
    wavfile.write(tmp_path / "wav" / "spk_a" / "a.wav", 16000, pcm(items["onsets"][0][:16161]))
    wavfile.write(tmp_path / "wav" / "spk_b" / "edge.wav", 16000, pcm(items["short_1760"][0]))
    if bad:
        wavfile.write(tmp_path / "wav" / "spk_b" / "tiny.wav", 16000, pcm(items["short_1600"][0][:1599]))
        (tmp_path / "wav" / "spk_b" / "broken.wav").write_bytes(b"RIFF....")
    (tmp_path / "wav" / "spk_b" / "notes.txt").write_text("not audio")


def test_cli_host_logic(tmp_path, monkeypatch, capsys):
    monkeypatch.chdir(tmp_path)
    items = O.synth_items()
    _tree(tmp_path, items)
    (tmp_path / "wav" / "top.wav").write_bytes(b"")   # not in a speaker directory: not taken
    (tmp_path / "pit" / "spk_a").mkdir(parents=True)
    (tmp_path / "pit" / "spk_a" / "a.pit.npy").write_bytes(b"old")   # overwritten
    m = _cli()
    assert m.pit_jobs("wav", "pit") == [("wav/spk_a/a.wav", "pit/spk_a/a.pit"), ("wav/spk_a/b.wav", "pit/spk_a/b.pit"),
                                        ("wav/spk_b/broken.wav", "pit/spk_b/broken.pit"),
                                        ("wav/spk_b/edge.wav", "pit/spk_b/edge.pit"),
                                        ("wav/spk_b/tiny.wav", "pit/spk_b/tiny.pit")]
    calls = []

    class Fake:
        def __init__(self, device):
            assert device == "cuda"
            self.closed = False
            calls.append(self)

        def f0_batch(self, clips):   # the device call, stubbed by the oracle
            return [O.praat_f0(c) for c in clips]

        def close(self):
            self.closed = True

    monkeypatch.setattr(praat_f0, "Extractor", Fake)
    capsys.readouterr()
    assert m.main(["-w", "wav", "-p", "pit", "-t", "2", "--batch", "2"]) == 0
    out, err = capsys.readouterr()
    assert out.splitlines()[:2] == ["wav", "pit"]
    assert len(calls) == 1 and calls[0].closed
    assert "tiny.wav" in err and "1599 samples" in err and "broken.wav" in err and "2 of 5 files failed" in err
    assert sorted(os.listdir(tmp_path / "pit" / "spk_a")) == ["a.pit.npy", "b.pit.npy"]
    assert sorted(os.listdir(tmp_path / "pit" / "spk_b")) == ["edge.pit.npy"]
    from whisper_vits_svc_b200 import hubert_infer
    for s, f in (("spk_a", "a"), ("spk_a", "b"), ("spk_b", "edge")):
        x = hubert_infer.load_audio(f"wav/{s}/{f}.wav", 16000)
        got = np.load(tmp_path / "pit" / s / f"{f}.pit.npy")
        assert got.dtype == np.float64 and got.shape == (O.n_frames(x.shape[0]) + 12,)
        assert np.array_equal(got, O.praat_f0(x))
    assert np.load(tmp_path / "pit" / "spk_b" / "edge.pit.npy").shape == (13,)


class _Sound:
    """parselmouth.Sound, as far as the reference uses it, computed by the oracle."""

    def __init__(self, x, sr):
        assert sr == 16000
        self.x = np.asarray(x, np.float64)

    def to_pitch_ac(self, time_step, voicing_threshold, pitch_floor, pitch_ceiling):
        assert (time_step, voicing_threshold, pitch_floor, pitch_ceiling) == (0.01, 0.5, 30, 1000)
        return types.SimpleNamespace(selected_array={"frequency": O.praat_f0_unpadded(self.x)})


@pytest.mark.skipif(not ref_import.available(), reason="reference tree absent")
def test_cli_matches_reference(tmp_path, monkeypatch):
    """The reference script, with parselmouth stubbed by the oracle and librosa.load by the project's loader, and the
    CLI with its device call stubbed by the oracle print the same first lines and write byte-equal files."""
    from whisper_vits_svc_b200 import hubert_infer
    items = O.synth_items()
    _tree(tmp_path, items, bad=False)
    monkeypatch.chdir(tmp_path)
    monkeypatch.setitem(sys.modules, "parselmouth", types.SimpleNamespace(Sound=_Sound))
    monkeypatch.setitem(sys.modules, "librosa", types.SimpleNamespace(
        load=lambda path, sr: (hubert_infer.load_audio(path, sr), sr)))
    monkeypatch.setattr(concurrent.futures, "ProcessPoolExecutor", concurrent.futures.ThreadPoolExecutor)
    out = io.StringIO()
    monkeypatch.setattr(sys, "argv", ["preprocess_f0_mouth.py", "-w", "wav", "-p", "pit_ref", "-t", "2"])
    with contextlib.redirect_stdout(out), contextlib.redirect_stderr(io.StringIO()):
        runpy.run_path(os.path.join(ref_import.REF_ROOT, "prepare", "preprocess_f0_mouth.py"), run_name="__main__")

    class Fake:
        def __init__(self, device):
            pass

        def f0_batch(self, clips):
            return [O.praat_f0(c) for c in clips]

        def close(self):
            pass

    monkeypatch.setattr(praat_f0, "Extractor", Fake)
    mine = io.StringIO()
    with contextlib.redirect_stdout(mine), contextlib.redirect_stderr(io.StringIO()):
        assert _cli().main(["-w", "wav", "-p", "pit_new", "-t", "2"]) == 0
    assert out.getvalue().splitlines()[:2] == ["wav", "pit_ref"] and mine.getvalue().splitlines()[:2] == ["wav", "pit_new"]

    def files(root):
        return {os.path.relpath(os.path.join(d, f), root): open(os.path.join(d, f), "rb").read()
                for d, _, fs in os.walk(root) for f in fs}

    ref, new = files(tmp_path / "pit_ref"), files(tmp_path / "pit_new")
    assert sorted(ref) == ["spk_a/a.pit.npy", "spk_a/b.pit.npy", "spk_b/edge.pit.npy"]
    assert new == ref


def test_pin_to_parselmouth():
    """The oracle equals parselmouth's to_pitch_ac at the reference's arguments, wherever parselmouth imports."""
    pm = pytest.importorskip("parselmouth")
    rng = np.random.default_rng(5)
    items = list(O.synth_items(seed=11).values())
    for _ in range(4):
        n = int(rng.integers(4000, 40000))
        tr = np.interp(np.arange(n), [0, n // 2, n - 1], rng.uniform(60, 900, 3))
        items.append(((O.tone(tr, rng) + 0.01 * rng.standard_normal(n)).astype(np.float32), tr))
    for x, _ in items:
        ref = pm.Sound(x.astype(np.float64), 16000).to_pitch_ac(
            time_step=160 / 16000, voicing_threshold=0.5, pitch_floor=30, pitch_ceiling=1000).selected_array["frequency"]
        got = O.praat_f0_unpadded(x)
        assert got.shape == ref.shape
        assert np.array_equal(got > 0, ref > 0)
        v = ref > 0
        if v.any():
            assert np.abs(got[v] - ref[v]).max() / ref[v].min() < 1e-3
