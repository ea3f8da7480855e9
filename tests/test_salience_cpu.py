"""Salience-based F0 on the host (oracle/salience_oracle.py, salience_f0's host tail, preprocess_f0_salience.py's host
logic).

The float32 oracle equals the live, unmodified reference (pitch/core/salience.py with its numba DP, and
pitch/inference.py:compute_f0_salience) behind a librosa stub whose stft is the oracle's.  The oracle's STFT is pinned to
torch.stft, its smoothing, correlation and threshold to scipy and the reference's formula, and its correlation to the
one-bin offset of the reference's origin.  The fp64 oracle is within 20 cents of the true F0 of tones and a glide and
gives 45 Hz on silence, and reproduces its fixture.  The CLI's walk, skips and exit code run against a stubbed
device call."""
import importlib.machinery
import importlib.util
import os
import sys
import types

import numpy as np
import pytest
import torch
from scipy import ndimage
from scipy.io import wavfile

from oracle import ref_import, salience_oracle as O
from tests.util import ROOT
from whisper_vits_svc_b200 import salience_f0

CLI = os.path.join(ROOT, "preprocess_f0_salience.py")
pcm = lambda x: np.clip(np.rint(x * 32767), -32768, 32767).astype(np.int16)


def _module(name, **attrs):
    m = types.ModuleType(name)
    m.__spec__ = importlib.machinery.ModuleSpec(name, loader=None)
    m.__dict__.update(attrs)
    return m


@pytest.fixture(scope="module")
def synth():
    return O.synth_items()


@pytest.fixture(scope="module")
def reference():
    """pitch.core.salience and pitch.inference of the reference tree, librosa's stft and load stubbed by the oracle's
    STFT and the project's loader; resampy (imported by the reference's crepe package) stubbed empty."""
    if not ref_import.available():
        pytest.skip("reference tree absent")
    pytest.importorskip("numba")
    from whisper_vits_svc_b200 import hubert_infer

    def stft(x, n_fft, hop_length, win_length, pad_mode):
        assert (n_fft, hop_length, win_length, pad_mode) == (2048, 320, 2048, "constant") and x.dtype == np.float32
        return O.stft(x, np.float32)

    stubs = {"librosa": _module("librosa", stft=stft, load=lambda p, sr: (hubert_infer.load_audio(p, sr), sr)),
             "resampy": _module("resampy")}
    saved = {k: sys.modules.get(k) for k in stubs}
    sys.modules.update(stubs)
    sys.path.insert(0, ref_import.REF_ROOT)
    try:
        import pitch.core.salience as S
        import pitch.inference as I
        yield S, I
    finally:
        sys.path.remove(ref_import.REF_ROOT)
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
        for k in [k for k in sys.modules if k == "pitch" or k.startswith("pitch.") or k == "crepe"
                  or k.startswith("crepe.")]:
            del sys.modules[k]


def test_oracle_matches_reference(reference, synth):
    S, _ = reference
    for name, (x, _) in synth.items():
        if x.shape[0] < O.MIN_SAMPLES:
            continue
        with np.errstate(all="ignore"):
            f0_ref, _, _ = S.salience(x, Fs=16000, H=320, N=2048, F_min=45.0, F_max=1760.0)
            Z_ref, _ = S.compute_salience_rep(x, 16000, 2048, 320, 45.0, 1760.0, 10.0, 10, 11, 0.9, 0.0)
        info = {}
        f0 = O.salience_f0(x, np.float32, info)
        assert np.array_equal(f0, f0_ref), name
        assert np.abs(info["Z"] - Z_ref).max() <= 1e-12 * max(np.abs(Z_ref).max(), 1e-300), name


def test_compute_f0_salience_matches_reference(reference, synth, tmp_path):
    _, I = reference
    for name in ("glide", "silence", "edge_320"):
        p = str(tmp_path / f"{name}.wav")
        wavfile.write(p, 16000, pcm(synth[name][0]))
        from whisper_vits_svc_b200 import hubert_infer
        x = hubert_infer.load_audio(p, 16000)
        with np.errstate(all="ignore"):
            want = I.compute_f0_salience(p, "cpu")
        got = O.compute_f0_salience(x, np.float32)
        assert got.shape == want.shape == (2 * (x.shape[0] // 320 + 1),), name
        assert np.array_equal(got, want), name
        assert np.array_equal(salience_f0.finish(O.salience_f0(x, np.float32)), want), name


def test_stft_pinned_to_torch(synth):
    for name in ("glide", "noise", "edge_321"):
        x = synth[name][0]
        X = O.stft(x)
        T = torch.stft(torch.from_numpy(x.astype(np.float64)), 2048, 320, 2048,
                       window=torch.hann_window(2048, periodic=True, dtype=torch.float64), center=True,
                       pad_mode="constant", return_complex=True).numpy()
        assert X.shape == T.shape == (1025, x.shape[0] // 320 + 1)
        assert np.abs(X - T).max() <= 1e-12 * np.abs(T).max(), name
        assert O.stft(x, np.float32).dtype == np.complex64


def test_smoothing_correlation_and_threshold_pinned_to_scipy():
    rng = np.random.default_rng(1)
    Y = rng.random((O.B, 7)) * (rng.random((O.B, 7)) < 0.3)
    sm = ndimage.convolve1d(Y, np.hanning(11), axis=0, mode="constant")
    assert np.abs(O.smooth(Y) - sm).max() <= 1e-15 * np.abs(sm).max()
    w = O.harmonic_taps()
    assert w.shape == (641,) and list(O.HARM_OFFSETS) == [0, 120, 190, 240, 279, 310, 337, 360, 380, 399]
    Z = ndimage.correlate1d(Y, w, axis=0, mode="constant", cval=0, origin=-len(w) // 2 + 5)
    assert np.array_equal(O.correlate(Y), Z)
    # the off-by-one: a partial in bin k gives its largest salience at bin k - 1, and bin i reads Y[i + j - 4]
    for k in (1, 200, 635):
        d = np.zeros((O.B, 1))
        d[k] = 1.0
        z = O.correlate(d)[:, 0]
        assert int(np.argmax(z)) == k - 1 and z[k - 1] == w[5]
        j = k + 4 - np.arange(O.B)        # z[i] = w[j] Y[i + j - 4] is non-zero only at i + j - 4 = k
        np.testing.assert_array_equal(z, np.where((j >= 0) & (j < w.shape[0]), w[np.clip(j, 0, w.shape[0] - 1)], 0.0))
    # the threshold: the reference's 20 log10(v / max + eps32) < 0, over the whole array
    eps = np.finfo(np.float32).eps
    V = rng.random((O.B, 9))
    V[3, 4] = V.max() * (1 - eps / 2)      # within eps32 of the maximum: cleared with it
    V[5, 1] = V.max() * (1 - 2 * eps)      # kept
    want = V * ((20 * np.log10(V / np.max(V) + eps)) < 0)
    got = O.threshold(V)
    assert np.array_equal(got, want)
    assert got[3, 4] == 0 and got[5, 1] > 0 and (got == 0).sum() == 2
    with np.errstate(all="ignore"):
        z = O.threshold(np.zeros((O.B, 3)))
    assert not np.isnan(z).any() and not z.any()


VOICED = [f"tone_{int(f)}" for f in O.TONES] + ["glide"]


@pytest.mark.parametrize("name", VOICED)
def test_ground_truth(synth, name):
    """Frames whose centre lies 40 ms or more inside a tone or the glide are within 20 cents of its true F0."""
    x, tr = synth[name]
    f0 = O.salience_f0(x)
    truth, ok = O.frame_truth(tr)
    assert ok.sum() >= 15
    cents = np.abs(1200 * np.log2(f0[ok] / truth[ok]))
    assert cents.max() < 20, (name, cents.max())


def test_silence_gives_45_hz(synth):
    x = synth["silence"][0]
    info = {}
    with np.errstate(all="ignore"):
        f0 = O.salience_f0(x, np.float64, info)
    assert f0.shape == (x.shape[0] // 320 + 1,) and np.all(f0 == 45.0) and not info["Z"].any()
    assert np.all(O.compute_f0_salience(np.zeros(3000))[1:-1] == 45.0)


def test_edges_and_frames(synth):
    with pytest.raises(ValueError):
        O.salience_f0(synth["edge_319"][0])
    for n in (320, 321, 639, 640, 641):
        assert O.salience_f0(np.zeros(n, np.float32)).shape == (n // 320 + 1,) == (salience_f0.frames_of(n),)
    assert O.MIN_SAMPLES == salience_f0.MIN_SAMPLES == 320 and O.B == salience_f0.BINS == 636
    np.testing.assert_array_equal(O.bin_hz()[[0, 120, 635]], [45.0, 90.0, 45.0 * 2 ** (635 / 120)])


def test_dp_first_index_on_ties():
    Z = np.zeros((O.B, 4))
    Z[[10, 300], :] = 2.0                  # two equal tracks: the first index wins at the end and on the way
    assert list(O.dp(Z)) == [10] * 4
    Z[300, 3] = 3.0                        # a larger last value moves the end, and the path follows it back
    assert list(O.dp(Z)) == [300] * 4


def test_fixture_reproduced(synth):
    g = O.load_golden()
    assert sorted(g) == sorted(synth)
    assert os.path.getsize(O.GOLDEN) < 1 << 20
    for k, d in g.items():
        assert np.array_equal(d["x"], synth[k][0]), k
        if d["x"].shape[0] < O.MIN_SAMPLES:
            assert "eta64" not in d
            continue
        with np.errstate(all="ignore"):
            for field, dt in (("eta64", np.float64), ("eta32", np.float32)):
                info = {}
                O.salience_f0(d["x"], dt, info)
                assert np.array_equal(info["eta"], d[field]), (k, field)


def _cli():
    spec = importlib.util.spec_from_file_location("preprocess_f0_salience_cli", CLI)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_cli_host_logic(tmp_path, monkeypatch, capsys, synth):
    monkeypatch.chdir(tmp_path)
    for s in ("spk_b", "spk_a"):
        (tmp_path / "wav" / s).mkdir(parents=True)
    wavfile.write(tmp_path / "wav" / "spk_a" / "b.wav", 16000, pcm(synth["vibrato"][0]))
    wavfile.write(tmp_path / "wav" / "spk_a" / "a.wav", 16000, pcm(synth["tone_220"][0]))
    wavfile.write(tmp_path / "wav" / "spk_b" / "edge.wav", 16000, pcm(synth["edge_320"][0]))
    wavfile.write(tmp_path / "wav" / "spk_b" / "tiny.wav", 16000, pcm(synth["edge_319"][0]))
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
            return [O.compute_f0_salience(c) for c in clips]

        def close(self):
            self.closed = True

    monkeypatch.setattr(salience_f0, "Extractor", Fake)
    capsys.readouterr()
    assert m.main(["-w", "wav", "-p", "pit", "-t", "2", "--batch", "2"]) == 0
    out, err = capsys.readouterr()
    assert out.splitlines()[:2] == ["wav", "pit"]
    assert len(calls) == 1 and calls[0].closed
    assert "tiny.wav" in err and "319 samples" in err and "broken.wav" in err and "2 of 5 files failed" in err
    assert sorted(os.listdir(tmp_path / "pit" / "spk_a")) == ["a.pit.npy", "b.pit.npy"]
    assert sorted(os.listdir(tmp_path / "pit" / "spk_b")) == ["edge.pit.npy"]
    from whisper_vits_svc_b200 import hubert_infer
    for s, f in (("spk_a", "a"), ("spk_a", "b"), ("spk_b", "edge")):
        x = hubert_infer.load_audio(f"wav/{s}/{f}.wav", 16000)
        got = np.load(tmp_path / "pit" / s / f"{f}.pit.npy")
        assert got.dtype == np.float64 and got.shape == (2 * (x.shape[0] // 320 + 1),)
        assert np.array_equal(got, O.compute_f0_salience(x))
    assert np.load(tmp_path / "pit" / "spk_b" / "edge.pit.npy").shape == (4,)
