"""svc_preprocessing.py on the device: the ten steps in one process against the ten CLIs' `main`s called one by one,
each step's release of device memory, one run as a command, and the stop at a missing model file."""
import importlib.util
import os
import random
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.test_speaker_gpu import CONFIG as SPEAKER_CONFIG
from tests.util import ROOT
from whisper_vits_svc_b200 import synth

pytestmark = pytest.mark.gpu

SEED = 1234
MIB = 1 << 20
# speaker/file: (seconds, rate); 0.5 s is kept by every step but dropped by the loader check, which takes 1 s and up
CLIPS = {"alto/a00": (0.5, 44100), "alto/a01": (1.7, 48000), "alto/a02": (2.6, 44100), "alto/a03": (3.3, 48000),
         "alto/a04": (4.4, 44100), "alto/a05": (6.0, 48000), "tenor/t00": (1.2, 48000), "tenor/t01": (2.1, 44100),
         "tenor/t02": (2.9, 48000), "tenor/t03": (3.8, 44100), "tenor/t04": (5.1, 48000), "tenor/t05": (5.6, 44100)}
OUTPUTS = {"waves-16k": ".wav", "waves-32k": ".wav", "pitch": ".pit.npy", "whisper": ".ppg.npy", "hubert": ".vec.npy",
           "speaker": ".spk.npy", "specs": ".pt"}


def _cli(name):
    spec = importlib.util.spec_from_file_location(name.replace(".py", "_cli"), os.path.join(ROOT, name))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


@pytest.fixture(scope="module")
def models(tmp_path_factory):
    """The five model files at the reference's relative paths (Whisper at a reduced width), and configs/base.yaml."""
    d = tmp_path_factory.mktemp("models")
    dims = dict(synth.WHISPER_LARGE_V2_DIMS, n_audio_state=256, n_audio_head=4, n_audio_layer=4)
    for rel, obj in (("whisper_pretrain/large-v2.pt", synth.whisper_checkpoint(dims, seed=11)),
                     ("hubert_pretrain/hubert-soft-0d54a1f4.pt", synth.hubert_checkpoint(31)),
                     ("speaker_pretrain/best_model.pth.tar", synth.speaker_checkpoint(5)),
                     ("crepe/assets/full.pth", synth.crepe_checkpoint(11, "full"))):
        (d / rel).parent.mkdir(parents=True, exist_ok=True)
        torch.save(obj, d / rel)
    (d / "speaker_pretrain" / "config.json").write_text(SPEAKER_CONFIG)
    (d / "configs").mkdir()
    shutil.copy(os.path.join(ROOT, "configs", "base.yaml"), d / "configs")
    return d


def _tree(root, models):
    from scipy.io import wavfile
    shutil.copytree(models, root, dirs_exist_ok=True)
    for i, (rel, (sec, rate)) in enumerate(CLIPS.items()):
        n = int(sec * rate)
        t = np.arange(n) / rate
        g = np.random.default_rng(i)
        x = 0.3 * np.sin(2 * np.pi * (140.0 + 25 * i) * t) * (1 + 0.4 * np.sin(2 * np.pi * 3 * t)) + 0.02 * g.standard_normal(n)
        p = root / "dataset_raw" / f"{rel}.wav"
        p.parent.mkdir(parents=True, exist_ok=True)
        wavfile.write(p, rate, (x * 32767).astype(np.int16))
    (root / "dataset_raw" / "alto" / "broken.wav").write_bytes(b"not a wav file")
    wavfile.write(root / "dataset_raw" / "tenor" / "silent.wav", 48000, np.zeros(48000, np.int16))
    return root


def _seed():
    torch.manual_seed(SEED)
    random.seed(SEED)
    np.random.seed(SEED)


def _outputs(root):
    return {os.path.relpath(os.path.join(d, f), root): open(os.path.join(d, f), "rb").read()
            for top in ("data_svc", "files") for d, _, fs in os.walk(root / top) for f in fs}


def _memory():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return torch.cuda.memory_allocated(), torch.cuda.mem_get_info()[0]


def _check_outputs(root):
    """Every good clip has each step's output with the shape and dtype its CLI writes; the two bad ones have none."""
    from scipy.io import wavfile
    from whisper_vits_svc_b200 import hubert_infer, whisper_infer
    for rel, (sec, rate) in CLIPS.items():
        n = int(sec * rate)
        n16, n32 = -(-n * 160 // (rate // 100)), -(-n * 320 // (rate // 100))
        for sr, m in ((16000, n16), (32000, n32)):
            r, x = wavfile.read(root / "data_svc" / f"waves-{sr // 1000}k" / f"{rel}.wav")
            assert r == sr and x.dtype == np.int16 and x.shape == (m,), rel
        shapes = {"pitch": (1 + n16 // 160,), "whisper": (whisper_infer.ppg_rows(n16), 256),
                  "hubert": (hubert_infer.HubertSoftB200.frames(n16), 256),
                  "speaker": (256,)}
        for d, shape in shapes.items():
            a = np.load(root / "data_svc" / d / f"{rel}{OUTPUTS[d]}")
            assert a.dtype == np.float32 and a.shape == shape, (d, rel)
        spec = torch.load(root / "data_svc" / "specs" / f"{rel}.pt")
        assert spec.dtype == torch.float32 and spec.shape == (513, n32 // 320), rel
    for d, ext in OUTPUTS.items():
        assert sorted(os.listdir(root / "data_svc" / d)) == ["alto", "tenor"], d
        for bad in ("alto/broken", "tenor/silent"):
            assert not (root / "data_svc" / d / f"{bad}{ext}").exists(), (d, bad)
    for s in ("alto", "tenor"):
        a = np.load(root / "data_svc" / "singer" / f"{s}.spk.npy")
        assert a.dtype == np.float32 and a.shape == (256,)
    valid = (root / "files" / "valid.txt").read_text().splitlines()
    train = (root / "files" / "train.txt").read_text().splitlines()
    assert len(valid) == 10 and len(valid) + len(train) == len(CLIPS)
    return valid + train


def test_pipeline_in_process_equals_the_steps_one_by_one(tmp_path, models, capfd):
    P = _cli("svc_preprocessing.py")
    one = _tree(tmp_path / "one", models)
    steps = _tree(tmp_path / "steps", models)
    cwd = os.getcwd()
    try:
        os.chdir(one)
        _seed()
        assert P.main(["-t", "2"]) == 0
        out, err = capfd.readouterr()
        assert [ln[len("Command: python "):] for ln in out.splitlines() if ln.startswith("Command: ")] == P.STEPS
        assert "broken.wav" in err and "silent" in err and "Traceback" not in err

        os.chdir(steps)
        _seed()
        for step in P.STEPS:
            before = _memory()
            run, argv = P.step_main(step)
            assert run(argv) == 0, step
            after = _memory()
            print(f"{step.split()[0]}: allocated {before[0]} -> {after[0]} B, free {before[1] / MIB:.0f} -> "
                  f"{after[1] / MIB:.0f} MiB")
            assert after[0] == before[0], step
            assert abs(after[1] - before[1]) <= 64 * MIB, step
    finally:
        os.chdir(cwd)
    got, want = _outputs(one), _outputs(steps)
    assert sorted(got) == sorted(want)
    for k in want:
        assert got[k] == want[k], k
    _check_outputs(one)


def test_pipeline_command(tmp_path, models):
    """One run as a command: exit 0, the ten Command lines in order, every output.  Its CREPE noise and the list
    shuffle are unseeded, so pitch and lists are compared with a seeded in-process run by shape and entries only."""
    P = _cli("svc_preprocessing.py")
    cmd = _tree(tmp_path / "cmd", models)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "svc_preprocessing.py"), "-t", "2"], cwd=cmd,
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert [ln for ln in r.stdout.splitlines() if ln.startswith("Command: ")] == [f"Command: python {s}" for s in P.STEPS]
    assert r.stdout.startswith("CPU Count is : ")
    assert "broken.wav" in r.stderr and "silent" in r.stderr
    entries = _check_outputs(cmd)

    one = _tree(tmp_path / "one", models)
    cwd = os.getcwd()
    try:
        os.chdir(one)
        _seed()
        assert P.main([]) == 0
    finally:
        os.chdir(cwd)
    assert sorted(entries) == sorted(_check_outputs(one))
    got, want = _outputs(cmd), _outputs(one)
    assert sorted(got) == sorted(want)
    for k in want:
        if k.startswith(os.path.join("data_svc", "pitch")):
            a, b = np.load(cmd / k), np.load(one / k)
            assert a.dtype == b.dtype and a.shape == b.shape, k
        elif not k.startswith("files"):
            assert got[k] == want[k], k


def test_missing_crepe_model_stops_after_resampling(tmp_path, models):
    root = _tree(tmp_path / "nocrepe", models)
    os.remove(root / "crepe" / "assets" / "full.pth")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "svc_preprocessing.py")], cwd=root,
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 1, r.stdout[-3000:] + r.stderr[-3000:]
    commands = [ln for ln in r.stdout.splitlines() if ln.startswith("Command: ")]
    assert commands == [f"Command: python {s}" for s in _cli("svc_preprocessing.py").STEPS[:3]]
    assert "Traceback" in r.stderr and "full.pth" in r.stderr
    for sr in ("16k", "32k"):
        assert len(list((root / "data_svc" / f"waves-{sr}").rglob("*.wav"))) == len(CLIPS)
    for d in ("whisper", "hubert", "speaker", "singer", "specs"):
        assert not (root / "data_svc" / d).exists(), d
    assert not (root / "files").exists()
