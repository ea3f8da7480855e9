"""LSTM speaker encoder on the device (csrc/speaker_api.cu) against the float64 / fp32 oracle
(oracle/speaker_oracle.py) and the goldens of the unmodified reference."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import speaker_oracle as SO
from tests.util import ROOT
from whisper_vits_svc_b200 import _lib, synth
from whisper_vits_svc_b200 import speaker_infer as S

pytestmark = pytest.mark.gpu

CONFIG = """{
    "model_name": "lstm",
    "audio": {
        // the speaker_pretrain/config.json values the device path reads
        "num_mels": 80, "fft_size": 1024, "sample_rate": 16000, "win_length": 1024, "hop_length": 256,
        "frame_length_ms": null, "frame_shift_ms": null, "preemphasis": 0.98, "min_level_db": -100,
        "ref_level_db": 20, "power": 1.5, "griffin_lim_iters": 60, "signal_norm": true, "symmetric_norm": true,
        "max_norm": 4.0, "clip_norm": true, "mel_fmin": 0.0, "mel_fmax": 8000.0, "do_trim_silence": true, "trim_db": 60
    },
    "model": {"input_dim": 80, "proj_dim": 256, "lstm_dim": 768, "num_lstm_layers": 3, "use_lstm_with_projection": true}
}
"""
CASES = tuple(SO.SPEAKER_CASES)


@pytest.fixture(scope="module")
def goldens():
    return {n: SO.load_golden(n) for n in CASES}


@pytest.fixture(scope="module")
def encoders(goldens, tmp_path_factory):
    cfg = tmp_path_factory.mktemp("spk") / "config.json"
    cfg.write_text(CONFIG)
    audio = S.audio_params(S.read_json(str(cfg)))
    assert audio == dict(preemphasis=0.98, ref_level_db=20.0, min_level_db=-100.0, max_norm=4.0, trim_db=60.0)
    out = {}
    for g in goldens.values():
        seed = int(g["seed"])
        if seed not in out:
            out[seed] = S.SpeakerEncoderB200(synth.speaker_checkpoint(seed)["model"], audio, "cuda")
    return out


def _wav(g):
    return S.prepare_wav(g["wav"].astype(np.float32) / np.float32(32768))


@pytest.mark.parametrize("name", CASES)
def test_mel_fixture_against_float64_oracle(goldens, encoders, name):
    g = goldens[name]
    enc = encoders[int(g["seed"])]
    wav = _wav(g)
    mel = enc.melspectrogram(wav).cpu().numpy()
    ref = SO.melspectrogram(wav).T
    assert mel.shape == ref.shape == g["mel"].shape
    assert np.abs(mel - ref).max() <= 2e-3
    assert np.abs(mel - g["mel"]).max() <= 2e-3


def test_mel_random_lengths_ragged(encoders):
    enc = next(iter(encoders.values()))
    rng = np.random.default_rng(3)
    lens = [513, 1000, 4097, 16000, 63744, 100003]
    wavs = [(0.3 * rng.standard_normal(n) * np.sin(np.arange(n) / 700.0)).astype(np.float32) for n in lens]
    mel, fo = enc.mel_batch(wavs)
    mel = mel.cpu().numpy()
    for b, w in enumerate(wavs):
        ref = SO.melspectrogram(w).T
        assert fo[b + 1] - fo[b] == ref.shape[0] == 1 + len(w) // 256
        assert np.abs(mel[fo[b]:fo[b + 1]] - ref).max() <= 2e-3, b


@pytest.mark.parametrize("name", CASES)
def test_lstm_from_oracle_mel_is_bf16x3_grade(goldens, encoders, name):
    """The reference's mel straight into the LSTM: 2e-5 against the fp32 reference (a bf16 recurrence is ~3e-4)."""
    g = goldens[name]
    enc = encoders[int(g["seed"])]
    mel = torch.from_numpy(g["mel"])
    out, win = enc.embed_mels(mel, [0, mel.shape[0]], windows=True)
    assert np.abs(out[0].cpu().numpy() - g["embedding"]).max() <= 2e-5
    assert np.abs(win[0].cpu().numpy() - g["windows"]).max() <= 2e-5
    e, _ = SO.compute_embedding(synth.speaker_checkpoint(int(g["seed"]))["model"], g["mel"])
    assert np.abs(out[0].cpu().numpy() - e).max() <= 2e-5


@pytest.mark.parametrize("T", [1, 2, 3, 249])
def test_lstm_short_mels(encoders, T):
    """Fewer than 250 frames, down to one: the recurrence runs Lw = T steps (one step: no recurrent product at all)."""
    seed, enc = next(iter(encoders.items()))
    mel = np.random.default_rng(T).uniform(-4, 4, (T, 80)).astype(np.float32)
    out, win = enc.embed_mels(torch.from_numpy(mel), [0, T], windows=True)
    e, w = SO.compute_embedding(synth.speaker_checkpoint(seed)["model"], mel)
    assert np.abs(out[0].cpu().numpy() - e).max() <= 2e-5
    assert np.abs(win[0].cpu().numpy() - w).max() <= 2e-5
    both = enc.embed_mels(torch.from_numpy(np.concatenate([mel, mel[:1]])), [0, T, T + 1]).cpu().numpy()
    assert np.array_equal(both[0], out[0].cpu().numpy())


@pytest.mark.parametrize("name", CASES)
def test_goldens_end_to_end_from_audio(goldens, encoders, name):
    g = goldens[name]
    e = encoders[int(g["seed"])].embed([_wav(g)])[0].cpu().numpy()
    ref = g["embedding"]
    assert np.abs(e - ref).max() <= 2e-4
    assert float(e @ ref / np.linalg.norm(e) / np.linalg.norm(ref)) >= 0.9999


def test_ragged_batch_bitwise_equals_single(encoders):
    enc = next(iter(encoders.values()))
    rng = np.random.default_rng(9)
    lens = [20000, 249 * 256, 40000, 160400, 3000, 249 * 256 + 255, 90000]   # frames 79, 250, 157, 627, 12, 250, 352
    wavs = [(0.2 * rng.standard_normal(n)).astype(np.float32) for n in lens]
    batch = enc.embed(wavs).cpu().numpy()
    again = enc.embed(wavs).cpu().numpy()
    assert np.array_equal(batch, again)
    for b, w in enumerate(wavs):
        assert np.array_equal(enc.embed([w]).cpu().numpy()[0], batch[b]), b
    assert np.isfinite(batch).all()


def test_large_batch_spans_passes(encoders):
    """More items than one device pass (64): each item equals its run alone."""
    enc = next(iter(encoders.values()))
    rng = np.random.default_rng(11)
    wavs = [(0.2 * rng.standard_normal(int(n))).astype(np.float32) for n in rng.integers(600, 30000, 70)]
    batch = enc.embed(wavs).cpu().numpy()
    for b in (0, 63, 64, 69):
        assert np.array_equal(enc.embed([wavs[b]]).cpu().numpy()[0], batch[b]), b


def test_rejects_short_and_silent_audio(encoders):
    enc = next(iter(encoders.values()))
    with pytest.raises(_lib.SvcbError):
        enc.embed([np.zeros(400, np.float32) + 0.1])    # shorter than the reflect padding of one frame
    with pytest.raises(_lib.SvcbError):
        S.prepare_wav(np.zeros(32000, np.float32))      # silent: the reference divides by zero
    with pytest.raises(_lib.SvcbError):
        S.prepare_wav(np.ones(300, np.float32))         # nothing left after the 160-sample margins


def _model_files(tmp_path, seed=72):
    d = tmp_path / "speaker_pretrain"
    d.mkdir(exist_ok=True)
    torch.save(synth.speaker_checkpoint(seed), d / "best_model.pth.tar")
    (d / "config.json").write_text(CONFIG)
    return d


def _write_wav(path, g):
    from scipy.io import wavfile
    wavfile.write(path, 16000, g["wav"])


def test_cli_speaker_infer_matches_api(goldens, tmp_path):
    g = goldens["speaker_10s"]
    d = _model_files(tmp_path, int(g["seed"]))
    _write_wav(tmp_path / "in.wav", g)
    cmd = [sys.executable, os.path.join(ROOT, "speaker_infer.py"), str(d / "best_model.pth.tar"), str(d / "config.json"),
           "-s", "in.wav", "-t", "out.npy"]
    r = subprocess.run(cmd, cwd=tmp_path, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    got = np.load(tmp_path / "out.npy", allow_pickle=False)
    assert got.dtype == np.float32 and got.shape == (256,)
    assert not (tmp_path / "model_small.pth").exists()
    m = S.load_model(str(d / "best_model.pth.tar"), str(d / "config.json"), "cuda")
    assert np.array_equal(got, m.embed([m.load_wav(str(tmp_path / "in.wav"))])[0].cpu().numpy())
    assert np.abs(got - g["embedding"]).max() <= 2e-4


def test_cli_preprocess_speaker_tree(goldens, tmp_path, hp, sd):
    from scipy.io import wavfile
    _model_files(tmp_path)
    rng = np.random.default_rng(5)
    for s in ("spk_a", "spk_b"):
        (tmp_path / "data" / s).mkdir(parents=True)
        for i in range(3):
            wavfile.write(tmp_path / "data" / s / f"u{i}.wav", 16000,
                          SO.synth_voice(int(rng.integers(1000)), float(rng.uniform(1.0, 4.0)), 0.2))
    (tmp_path / "data" / "spk_b" / "notes.txt").write_text("not audio")
    wavfile.write(tmp_path / "data" / "spk_b" / "silent.wav", 16000, np.zeros(8000, np.int16))   # fails: skipped
    # non-silent but too short to frame after the margins: skipped alone, the rest of its batch is written
    wavfile.write(tmp_path / "data" / "spk_a" / "short.wav", 16000, SO.synth_voice(9, 600 / 16000, 0.0))
    cmd = [sys.executable, os.path.join(ROOT, "preprocess_speaker.py"), "data", "out", "-t", "2"]
    r = subprocess.run(cmd, cwd=tmp_path, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert "silent.wav" in r.stderr and "short.wav" in r.stderr
    m = S.load_model(str(tmp_path / "speaker_pretrain" / "best_model.pth.tar"), str(tmp_path / "speaker_pretrain" / "config.json"))
    for s in ("spk_a", "spk_b"):
        names = sorted(os.listdir(tmp_path / "out" / s))
        assert names == [f"u{i}.spk.npy" for i in range(3)]
        for i in range(3):
            e = np.load(tmp_path / "out" / s / f"u{i}.spk.npy")
            ref = m.embed([m.load_wav(str(tmp_path / "data" / s / f"u{i}.wav"))])[0].cpu().numpy()
            assert e.shape == (256,) and np.array_equal(e, ref)
    # the generated embedding drives the conversion CLI
    out = tmp_path / "out" / "spk_a" / "u0.spk.npy"
    n = 40
    g = torch.Generator().manual_seed(3)
    torch.save({"model_g": sd}, tmp_path / "model.pth")
    np.save(tmp_path / "x.ppg.npy", torch.randn(n // 2, hp.vits.ppg_dim, generator=g).numpy())
    np.save(tmp_path / "x.vec.npy", torch.randn(n // 2, hp.vits.vec_dim, generator=g).numpy())
    (tmp_path / "x.csv").write_text("".join(f"{i},{200 + i}\n" for i in range(n)))
    cmd = [sys.executable, os.path.join(ROOT, "svc_inference.py"), "--config", os.path.join(ROOT, "configs", "base.yaml"),
           "--model", "model.pth", "--wave", "none.wav", "--spk", str(out), "--ppg", "x.ppg.npy", "--vec", "x.vec.npy",
           "--pit", "x.csv"]
    r = subprocess.run(cmd, cwd=tmp_path, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    sr, w = wavfile.read(tmp_path / "svc_out.wav")
    assert w.dtype == np.float32 and w.size > 0 and np.isfinite(w).all()
