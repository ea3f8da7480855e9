"""WORLD DIO + StoneMask F0 on the host (oracle/f0_oracle.py, world_f0.round1, preprocess_f0.py's host logic).

The oracle is checked against the true F0 of synthetic tones, reproduces its fixture, and is pinned to pyworld where
pyworld imports.  The CLI's walk, names, dtype, lengths, printed lines and skips run against a stubbed device call."""
import importlib.util
import math
import os

import numpy as np
import pytest
from scipy.io import wavfile

from oracle import f0_oracle as O
from tests.util import ROOT
from whisper_vits_svc_b200 import world_f0

CLI = os.path.join(ROOT, "preprocess_f0.py")


def _cli():
    spec = importlib.util.spec_from_file_location("preprocess_f0_cli", CLI)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


@pytest.fixture(scope="module")
def synth():
    items = O.synth_items()
    return {k: (x, tr, O.world_f0(x)) for k, (x, tr) in items.items()}


@pytest.mark.parametrize("name", ["glide_up", "glide_down", "vibrato", "voiced_unvoiced", "steady_100"])
def test_ground_truth_tones(synth, name):
    """Within 1 % of the true F0 on voiced frames at least 30 ms from an onset or an end."""
    x, tr, f0 = synth[name]
    truth, ok = O.frame_truth(tr)
    v = ok & (truth > 0)
    assert v.sum() >= 90
    rel = np.abs(f0[v] - truth[v]) / truth[v]
    assert rel.max() < 0.01, (name, rel.max())


def test_ground_truth_silence_and_noise(synth):
    assert not synth["silence"][2].any()
    f0 = synth["noise"][2]
    assert (f0 == 0).mean() >= 0.95
    x, tr, f0 = synth["voiced_unvoiced"]
    truth, _ = O.frame_truth(tr)
    far = np.array([np.all(tr[max(0, i * 160 - 800):i * 160 + 800] == 0) for i in range(f0.shape[0])])
    assert far.sum() > 50 and (f0[far] == 0).mean() >= 0.95   # 50 ms or more from any voicing


def test_frames_and_bands():
    assert O.n_bands() == 8 and O.half_lengths() == [80, 56, 40, 28, 20, 14, 10, 7]
    for n in (0, 1, 159, 160, 161, 479, 480, 16000, 16001, 123457):
        assert O.n_frames(n) == n // 160 + 1 == world_f0.frames_of(n)
    assert O.MIN_SAMPLES == world_f0.MIN_SAMPLES == 480
    assert not O.world_f0(np.ones(479, np.float32)).any()   # at most 3 frames: zero


def test_fixture_reproduced(synth):
    g = O.load_golden()
    assert sorted(g) == sorted(synth)
    for k, (x, f0) in g.items():
        assert np.array_equal(x, synth[k][0]), k
        got = synth[k][2]
        assert np.array_equal(got > 0, f0 > 0), k
        np.testing.assert_allclose(got, f0, rtol=1e-9, atol=0, err_msg=k)


def test_round1_is_python_round():
    vals = [0.05, 0.15, 0.25, 0.35, 100.25, 100.75, 123.45, 220.05, 599.95, 71.35, 0.0, 899.99999]
    rng = np.random.default_rng(0)
    for k in rng.integers(0, 9000, 200):
        vals.append(k / 10 + 0.05)                 # near .x5: the nearest double is above or below the tie
    vals += [np.nextafter(v, np.inf) for v in vals] + [np.nextafter(v, -np.inf) for v in vals]
    vals += list(rng.uniform(0, 900, 500))
    got = world_f0.round1(np.array(vals))
    want = np.array([round(float(v), 1) for v in vals])
    assert got.dtype == np.float64 and np.array_equal(got, want)
    assert np.array_equal(O.round1(np.array(vals)), want)
    assert round(100.25, 1) == 100.2 and world_f0.round1([100.25])[0] == 100.2   # a binary tie goes to even
    assert round(0.15, 1) == 0.1 and np.round(0.15, 1) == 0.2 and world_f0.round1([0.15])[0] == 0.1


def test_cli_host_logic(tmp_path, monkeypatch, capsys):
    monkeypatch.chdir(tmp_path)
    items = O.synth_items()
    for s in ("spk_b", "spk_a"):
        (tmp_path / "wav" / s).mkdir(parents=True)
    pcm = lambda x: np.clip(np.rint(x * 32767), -32768, 32767).astype(np.int16)
    wavfile.write(tmp_path / "wav" / "spk_a" / "b.wav", 16000, pcm(items["vibrato"][0]))
    wavfile.write(tmp_path / "wav" / "spk_a" / "a.wav", 16000, pcm(items["glide_down"][0][:16161]))
    wavfile.write(tmp_path / "wav" / "spk_b" / "tiny.wav", 16000, pcm(items["short"][0][:479]))
    wavfile.write(tmp_path / "wav" / "spk_b" / "edge.wav", 16000, pcm(items["short"][0][:480]))
    (tmp_path / "wav" / "spk_b" / "broken.wav").write_bytes(b"RIFF....")
    (tmp_path / "wav" / "spk_b" / "notes.txt").write_text("not audio")
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
            return [O.round1(O.world_f0(c)) for c in clips]

        def close(self):
            self.closed = True

    monkeypatch.setattr(world_f0, "Extractor", Fake)
    capsys.readouterr()
    assert m.main(["-w", "wav", "-p", "pit", "-t", "2", "--batch", "2"]) == 0
    out, err = capsys.readouterr()
    assert out.splitlines()[:2] == ["wav", "pit"]
    assert len(calls) == 1 and calls[0].closed
    assert "tiny.wav" in err and "479 samples" in err and "broken.wav" in err and "2 of 5 files failed" in err
    assert sorted(os.listdir(tmp_path / "pit" / "spk_a")) == ["a.pit.npy", "b.pit.npy"]
    assert sorted(os.listdir(tmp_path / "pit" / "spk_b")) == ["edge.pit.npy"]
    from whisper_vits_svc_b200 import hubert_infer
    for s, f in (("spk_a", "a"), ("spk_a", "b"), ("spk_b", "edge")):
        x = hubert_infer.load_audio(f"wav/{s}/{f}.wav", 16000)
        got = np.load(tmp_path / "pit" / s / f"{f}.pit.npy")
        assert got.dtype == np.float64 and got.shape == (x.shape[0] // 160 + 1,)
        assert np.array_equal(got, O.round1(O.world_f0(x.astype(np.float64))))
    assert np.load(tmp_path / "pit" / "spk_b" / "edge.pit.npy").shape == (4,)


def test_pin_to_pyworld():
    """The oracle equals pyworld.dio + stonemask rounded to 0.1, wherever pyworld imports."""
    pw = pytest.importorskip("pyworld")
    rng = np.random.default_rng(5)
    items = list(O.synth_items(seed=11).values())
    for _ in range(4):
        n = int(rng.integers(4000, 40000))
        tr = np.interp(np.arange(n), [0, n // 2, n - 1], rng.uniform(90, 700, 3))
        items.append(((O.tone(tr, rng) + 0.01 * rng.standard_normal(n)).astype(np.float32), tr))
    total = diff = 0
    for x, _ in items:
        xd = x.astype(np.double)
        f0, t = pw.dio(xd, fs=16000, f0_ceil=900, frame_period=1000 * 160 / 16000)
        ref = np.array([round(v, 1) for v in pw.stonemask(xd, f0, t, fs=16000)])
        got = O.round1(O.world_f0(xd))
        assert got.shape == ref.shape
        assert np.array_equal(got > 0, ref > 0)
        total += ref.shape[0]
        diff += int(np.count_nonzero(got != ref))
        assert np.abs(got - ref).max() <= 0.1 + 1e-9
    assert diff <= math.ceil(0.001 * total), (diff, total)   # rounding ties only
