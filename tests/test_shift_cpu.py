"""The pitch-shift sweep CLI (svc_inference_shift.py) on the host: the per-shift pitch, and every way the CLI stops
before a model loads."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.util import ROOT
from whisper_vits_svc_b200 import hostio

CLI = os.path.join(ROOT, "svc_inference_shift.py")


@pytest.mark.parametrize("shift", range(-12, 13))
def test_shift_pitch_is_the_reference_expression(tmp_path, shift):
    p = str(tmp_path / "x.pit.csv")
    hostio.save_csv_pitch([0, 0, 97, 110, 123, 0, 440, 441, 1100, 0, 2047, 65, 0], p)
    # svc_inference_shift.py:63-65 of the reference
    want = torch.FloatTensor(np.array(hostio.load_csv_pitch(p)) * (2 ** (shift / 12)))
    got = hostio.shift_pitch(hostio.load_csv_pitch(p), shift)
    assert got.dtype == torch.float32 and torch.equal(got, want)
    assert torch.equal(got == 0, want == 0) and int((got == 0).sum()) == 5
    assert torch.equal(hostio.prepare_features(*_features(tmp_path), p, shift)[2], want)


def _features(tmp_path):
    np.save(tmp_path / "x.ppg.npy", np.zeros((7, 2), np.float32))
    np.save(tmp_path / "x.vec.npy", np.zeros((7, 3), np.float32))
    return str(tmp_path / "x.ppg.npy"), str(tmp_path / "x.vec.npy")


def _run(tmp_path, *extra, pit=True):
    cmd = [sys.executable, CLI, "--config", os.path.join(ROOT, "configs", "base.yaml"), "--model", "missing.pth",
           "--wave", "missing.wav", "--spk", "missing.spk.npy", *extra]
    if pit:
        cmd += ["--pit", "missing.pit.csv"]
    # no device visible, whatever the host has: each of these calls must stop before any device work
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    return subprocess.run(cmd, cwd=tmp_path, env=env, capture_output=True, text=True, timeout=300)


def test_cli_flags():
    r = subprocess.run([sys.executable, CLI, "-h"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    for flag in ("--config CONFIG", "--model MODEL", "--wave WAVE", "--spk SPK", "--ppg PPG", "--vec VEC", "--pit PIT",
                 "--shift_l SHIFT_L", "--shift_r SHIFT_R"):
        assert flag in r.stdout, flag


@pytest.mark.parametrize("l,r", [(1, 0), (-13, 0), (0, 13), (13, 13), (-13, -13), (12, -12)])
def test_bad_shifts_stop_before_anything_loads(tmp_path, l, r):
    res = _run(tmp_path, "--shift_l", str(l), "--shift_r", str(r))
    assert res.returncode != 0 and "AssertionError" in res.stderr, res.stderr
    assert "no CPU path" not in res.stderr and "pitch shift" not in res.stdout
    assert not (tmp_path / "_svc_out").exists()


def test_missing_pit_stops_with_the_svc_inference_message(tmp_path):
    res = _run(tmp_path, "--shift_l", "-2", "--shift_r", "1", pit=False)
    assert res.returncode != 0
    assert "--pit is required: the CREPE pitch extractor is out of scope of this build" in res.stderr, res.stderr
    assert "Auto run" not in res.stdout


def test_no_device_stops_with_no_cpu_path(tmp_path):
    res = _run(tmp_path, "--shift_l", "-12", "--shift_r", "12")
    assert res.returncode != 0
    assert "this build has no CPU path: a CUDA (sm_90a) device is required" in res.stderr, res.stderr
    assert "Auto run" not in res.stdout and "pitch shift" not in res.stdout
    assert os.listdir(tmp_path / "_svc_out") == []
