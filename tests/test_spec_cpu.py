"""Linear spectrograms of the training data without a device: the oracle against the live reference and the fixture,
the wav loader's accept / reject rules, the config check, and the CLI's flags, walk and output paths."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import ref_import, spec_oracle as SO
from tests.util import ROOT
from whisper_vits_svc_b200 import hparams, spectrogram

CLI = os.path.join(ROOT, "preprocess_spec.py")


@pytest.fixture(scope="module")
def hp():
    return hparams.load_hparams(os.path.join(ROOT, "configs", "base.yaml"))


def _write(path, sr, data):
    from scipy.io import wavfile
    wavfile.write(path, sr, data)
    return str(path)


def _pcm(rng, n, ch=1):
    shape = (n,) if ch == 1 else (n, ch)
    return (rng.standard_normal(shape) * 6000).clip(-32768, 32767).astype(np.int16)


@pytest.mark.skipif(not ref_import.available(), reason="reference tree absent")
def test_oracle_bitwise_equals_live_reference():
    ref = SO.reference_spectrogram()
    clips = {k: x for k, (x, _) in SO.load_golden().items()}
    clips["loud"] = (1.5 * SO.synth_clips()["sweep"][:320 * 7 + 5]).astype(np.float32)   # leaves [-1, 1]
    for name, x in clips.items():
        y = torch.from_numpy(x)[None]
        want = ref(y, 1024, 32000, 320, 1024, center=False)
        got = SO.spectrogram(y)
        assert want.dtype == torch.float32 and torch.equal(got, want), name


def test_golden_reproduces_from_oracle():
    g, clips = SO.load_golden(), SO.synth_clips()
    assert sorted(g) == sorted(clips)
    lens = {x.shape[0] for x, _ in g.values()}
    assert 353 in lens and any(n % 320 == 0 for n in lens) and any(n % 320 == 17 for n in lens)
    for name, (x, s) in g.items():
        assert np.array_equal(x, clips[name]), name
        got = SO.spectrogram(torch.from_numpy(x)[None])[0].numpy()
        assert got.shape == s.shape == (513, x.shape[0] // 320)
        err = np.abs(got - s).max()
        assert err <= 2e-6 * max(1.0, float(np.abs(s).max())), (name, err)


def test_load_wav_accepts_and_rejects(tmp_path, hp):
    rng = np.random.default_rng(0)
    for n in (353, 32000 + 17):
        path = _write(tmp_path / f"ok{n}.wav", 32000, _pcm(rng, n))
        x = spectrogram.load_wav(path, hp)
        want, sr = SO.load_wav(path)
        assert sr == 32000 and x.dtype == np.float32 and x.shape == (n,)
        assert np.array_equal(x, want.numpy())
    with pytest.raises(ValueError, match="16000 is not 32000"):
        spectrogram.load_wav(_write(tmp_path / "sr16k.wav", 16000, _pcm(rng, 16000)), hp)
    with pytest.raises(ValueError, match="2 channels"):
        spectrogram.load_wav(_write(tmp_path / "stereo.wav", 32000, _pcm(rng, 32000, 2)), hp)
    with pytest.raises(ValueError, match="352 samples"):
        spectrogram.load_wav(_write(tmp_path / "short.wav", 32000, _pcm(rng, 352)), hp)
    f32 = _write(tmp_path / "float.wav", 32000, (0.25 * rng.standard_normal(1000)).astype(np.float32))
    assert np.array_equal(spectrogram.load_wav(f32, hp), SO.load_wav(f32)[0].numpy())


@pytest.mark.parametrize("n", [353, 639, 640, 641, 320 * 1000 + 17])
def test_frame_rule(n):
    assert spectrogram.frames(n) == n // 320 == SO.spectrogram(torch.zeros(1, n)).shape[-1]


def test_config_check(hp):
    spectrogram.check_hparams(hp)
    for key, v in (("filter_length", 2048), ("hop_length", 256), ("win_length", 800)):
        with pytest.raises(ValueError, match="unsupported spectrogram config"):
            spectrogram.check_hparams(hparams.override(hp, **{f"data__{key}": v}))
        with pytest.raises(ValueError):
            spectrogram.spec_batch([np.zeros(1000, np.float32)], hparams.override(hp, **{f"data__{key}": v}))


def test_cli_flags():
    r = subprocess.run([sys.executable, CLI, "-h"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0
    for flag in ("-w WAV, --wav WAV", "-s SPE, --spe SPE", "-t THREAD_COUNT, --thread_count THREAD_COUNT", "--batch BATCH"):
        assert flag in r.stdout, flag


def test_cli_walk_and_output_paths(tmp_path, monkeypatch):
    import importlib.util
    monkeypatch.chdir(tmp_path)
    for s in ("alice", "bob"):
        (tmp_path / "wav" / s).mkdir(parents=True)
        for f in ("a.wav", "b.wav", "notes.txt"):
            (tmp_path / "wav" / s / f).write_bytes(b"")
    (tmp_path / "wav" / "top.wav").write_bytes(b"")            # not in a speaker directory: not taken
    spec = importlib.util.spec_from_file_location("preprocess_spec_cli", CLI)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    want = [(f"wav/{s}/{f}.wav", f"spe/{s}/{f}.pt") for s in ("alice", "bob") for f in ("a", "b")]
    assert m.spec_jobs("wav", "spe") == want
    assert (tmp_path / "spe" / "alice").is_dir() and (tmp_path / "spe" / "bob").is_dir()
    torch.save(torch.zeros(513, 1), tmp_path / "spe" / "alice" / "a.pt")
    assert m.spec_jobs("wav", "spe") == want                    # existing outputs are overwritten, not skipped


def test_cli_rejects_config_before_any_file(tmp_path):
    (tmp_path / "configs").mkdir()
    text = open(os.path.join(ROOT, "configs", "base.yaml")).read().replace("hop_length: 320", "hop_length: 256")
    (tmp_path / "configs" / "base.yaml").write_text(text)
    (tmp_path / "wav" / "spk").mkdir(parents=True)
    _write(tmp_path / "wav" / "spk" / "a.wav", 32000, _pcm(np.random.default_rng(1), 4000))
    r = subprocess.run([sys.executable, CLI, "-w", "wav", "-s", "spe"], cwd=tmp_path, capture_output=True, text=True,
                       timeout=120)
    assert r.returncode != 0 and "unsupported spectrogram config" in r.stderr
    assert r.stdout.splitlines()[:2] == ["wav", "spe"]
    assert not (tmp_path / "spe").exists()
