"""Bare recordings on the device: `pred_pit` writes `compute_f0_sing`'s CSV, the batch CLI's ragged F0 pass writes what
one `pred_pit` per file writes, and both conversion command lines extract a missing F0 and convert."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy.io import wavfile

from oracle import speaker_oracle as SO
from tests.util import ROOT
from whisper_vits_svc_b200 import crepe_infer as C, hostio, hubert_infer, synth

pytestmark = pytest.mark.gpu
CONFIG = os.path.join(ROOT, "configs", "base.yaml")
HOP = 320


@pytest.fixture(scope="module")
def crepe_sd():
    return synth.crepe_checkpoint(11, "full")


@pytest.fixture(scope="module")
def crepe(crepe_sd):
    return C.CrepeB200(crepe_sd, "cuda", "full")


def _voice(path, seed, seconds):
    x = SO.synth_voice(seed, seconds, 0.0)
    wavfile.write(path, 16000, x)
    return x.shape[0]


def _draws(n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, generator=g), (torch.rand(C.frames_of(n, HOP), generator=g) - 0.5) * 40


def _csv_lines_ok(path, n):
    lines = open(path, encoding="utf-8").read().splitlines()
    assert len(lines) == 2 * (1 + n // HOP)
    for i, line in enumerate(lines):
        m = re.fullmatch(r"(\d+)m (\d+)s ([ \d]{3}),(-?\d+)", line)
        assert m and int(m[1]) * 60000 + int(m[2]) * 1000 + int(m[3]) == 10 * i, line
    return len(lines)


def test_pred_pit_writes_compute_f0_sing(tmp_path, crepe):
    n = _voice(tmp_path / "x.wav", 1, 1.7)
    noise, dither = _draws(n, 2)
    C.pred_pit(crepe, str(tmp_path / "x.wav"), str(tmp_path / "got.csv"), noise, dither)
    audio = hubert_infer.load_audio(str(tmp_path / "x.wav"), 16000)
    hostio.save_csv_pitch(C.compute_f0_sing(crepe, audio, noise, dither), str(tmp_path / "want.csv"))
    assert (tmp_path / "got.csv").read_bytes() == (tmp_path / "want.csv").read_bytes()
    _csv_lines_ok(tmp_path / "got.csv", n)


def test_ragged_pass_equals_pred_pit_per_file(tmp_path, crepe):
    import svc_inference_batch as B
    wavs, lengths = [], []
    for k, s in enumerate((3.2, 0.03, 0.4, 6.0, 1.0, 2.5)):
        wavs.append(str(tmp_path / f"w{k}.wav"))
        lengths.append(_voice(wavs[-1], 10 + k, s))
    (tmp_path / "bad.wav").write_bytes(b"not a wav")
    wavs.insert(2, str(tmp_path / "bad.wav"))
    lengths.insert(2, 100)
    draws = [_draws(n, 20 + k) for k, n in enumerate(lengths)]
    csvs = [str(tmp_path / f"ragged{k}.csv") for k in range(len(wavs))]
    lost = B.extract_pitch(crepe, wavs, csvs, [d[0] for d in draws], [d[1] for d in draws], threads=2, batch=3)
    assert lost == [2] and not os.path.exists(csvs[2])
    for k, (wav, (noise, dither)) in enumerate(zip(wavs, draws)):
        if k == 2:
            continue
        C.pred_pit(crepe, wav, str(tmp_path / "alone.csv"), noise, dither)
        assert open(csvs[k], "rb").read() == (tmp_path / "alone.csv").read_bytes(), k
        _csv_lines_ok(csvs[k], lengths[k])


def _models(tmp_path, hp, sd, crepe_sd):
    if crepe_sd is not None:
        (tmp_path / "crepe" / "assets").mkdir(parents=True)
        torch.save(crepe_sd, tmp_path / "crepe" / "assets" / "full.pth")
    torch.save({"model_g": sd}, tmp_path / "g.pth")
    np.save(tmp_path / "x.spk.npy", (np.random.RandomState(3).randn(hp.vits.spk_dim) * 0.05).astype(np.float32))


def _features(stem, hp, ppg_rows, vec_rows, seed):
    rs = np.random.RandomState(seed)
    np.save(f"{stem}.ppg.npy", rs.randn(ppg_rows, hp.vits.ppg_dim).astype(np.float32))
    np.save(f"{stem}.vec.npy", rs.randn(vec_rows, hp.vits.vec_dim).astype(np.float32))


def test_svc_inference_extracts_a_missing_pit(tmp_path, hp, sd, crepe_sd):
    _models(tmp_path, hp, sd, crepe_sd)
    n = _voice(tmp_path / "x.wav", 5, 2.0)
    pit_rows = 2 * (1 + n // HOP)
    _features(tmp_path / "x", hp, pit_rows // 2 + 9, pit_rows // 2 + 4, 6)     # the pitch is the shortest feature
    cmd = [sys.executable, os.path.join(ROOT, "svc_inference.py"), "--config", CONFIG, "--model", "g.pth", "--wave", "x.wav",
           "--spk", "x.spk.npy", "--ppg", "x.ppg.npy", "--vec", "x.vec.npy"]
    r = subprocess.run(cmd, cwd=tmp_path, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert "Auto run : H100 CREPE pitch extractor -w x.wav -p svc_tmp.pit.csv" in r.stdout.splitlines()
    assert _csv_lines_ok(tmp_path / "svc_tmp.pit.csv", n) == pit_rows
    ppg_rows, vec_rows = np.load(tmp_path / "x.ppg.npy").shape[0], np.load(tmp_path / "x.vec.npy").shape[0]
    rate, w = wavfile.read(tmp_path / "svc_out.wav")
    assert rate == hp.data.sampling_rate and w.dtype == np.float32 and np.isfinite(w).all()
    assert w.shape == (min(pit_rows, 2 * ppg_rows, 2 * vec_rows) * HOP - 1,)


def _batch(tmp_path):
    cmd = [sys.executable, os.path.join(ROOT, "svc_inference_batch.py"), "--config", CONFIG, "--model", "g.pth", "--wave",
           "waves", "--spk", "x.spk.npy", "--feat", "feat"]
    return subprocess.run(cmd, cwd=tmp_path, capture_output=True, text=True, timeout=900)


def test_batch_extracts_missing_pitch_and_converts(tmp_path, hp, sd, crepe_sd):
    _models(tmp_path, hp, sd, crepe_sd)
    (tmp_path / "waves").mkdir()
    (tmp_path / "feat").mkdir()
    want = {}
    for k, (name, seconds) in enumerate((("a", 3.1), ("b", 0.7), ("c", 5.4), ("d", 1.9))):
        n = _voice(tmp_path / "waves" / f"{name}.wav", 30 + k, seconds)
        pit_rows = 2 * (1 + n // HOP)
        if name == "d":     # a hand-written constant F0, shorter than the audio
            pit_rows -= 17
            hostio.save_csv_pitch([200] * pit_rows, str(tmp_path / "feat" / "d.pit.csv"))
        ppg_rows, vec_rows = [(pit_rows // 2 + 5, pit_rows // 2 + 3), (pit_rows // 2 - 6, pit_rows // 2 + 2),
                              (pit_rows // 2 + 1, pit_rows // 2 - 4), (pit_rows // 2 + 20, pit_rows // 2 + 30)][k]
        _features(tmp_path / "feat" / name, hp, ppg_rows, vec_rows, 40 + k)
        want[name] = (n, pit_rows, min(pit_rows, 2 * ppg_rows, 2 * vec_rows) * HOP - 1)
    (tmp_path / "waves" / "bad.wav").write_bytes(b"not a wav")
    _features(tmp_path / "feat" / "bad", hp, 50, 50, 49)
    given = (tmp_path / "feat" / "d.pit.csv").read_bytes()
    r = _batch(tmp_path)
    log = r.stdout[-3000:] + r.stderr[-3000:]
    assert r.returncode == 1, log
    assert "bad.wav: FAILED" in r.stdout and "svc_inference_batch: 4/5 files converted" in r.stdout, log
    out = tmp_path / "_svc_out"
    for name, (n, pit_rows, samples) in want.items():
        rate, w = wavfile.read(out / f"{name}.wav")
        assert rate == hp.data.sampling_rate and w.dtype == np.float32 and w.shape == (samples,), name
        assert np.isfinite(w).all(), name
        if name == "d":
            assert not (out / "d.wav.pit.csv").exists()
        else:
            assert _csv_lines_ok(out / f"{name}.wav.pit.csv", n) == pit_rows
    assert not (out / "bad.wav").exists()
    assert (tmp_path / "feat" / "d.pit.csv").read_bytes() == given


def test_batch_without_the_crepe_checkpoint_converts_the_rest(tmp_path, hp, sd):
    _models(tmp_path, hp, sd, None)
    (tmp_path / "waves").mkdir()
    (tmp_path / "feat").mkdir()
    for k, name in enumerate(("a", "d")):
        n = _voice(tmp_path / "waves" / f"{name}.wav", 50 + k, 1.0)
        _features(tmp_path / "feat" / name, hp, n // HOP, n // HOP, 60 + k)
    hostio.save_csv_pitch([180] * (2 * (n // HOP)), str(tmp_path / "feat" / "d.pit.csv"))
    r = _batch(tmp_path)
    assert r.returncode == 1, r.stdout[-3000:] + r.stderr[-3000:]
    assert "F0 extraction FAILED" in r.stdout and "a.wav: FAILED" in r.stdout
    assert "svc_inference_batch: 1/2 files converted" in r.stdout
    assert sorted(os.listdir(tmp_path / "_svc_out")) == ["d.wav"]
