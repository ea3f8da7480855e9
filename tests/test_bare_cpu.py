"""Bare recordings without a device: `svc_inference.py` without --pit stops before any model loads or file is written,
and the batch CLI's pitch-file lookup and F0 schedule."""
import os
import subprocess
import sys

from tests.util import ROOT


def test_svc_inference_without_pit_or_device_stops_first(tmp_path):
    cmd = [sys.executable, os.path.join(ROOT, "svc_inference.py"), "--config", os.path.join(ROOT, "configs", "base.yaml"),
           "--model", "missing.pth", "--wave", "missing.wav", "--spk", "missing.spk.npy"]
    r = subprocess.run(cmd, cwd=tmp_path, env=dict(os.environ, CUDA_VISIBLE_DEVICES=""), capture_output=True, text=True,
                       timeout=300)
    assert r.returncode != 0
    assert "this build has no CPU path: a CUDA (sm_90a) device is required" in r.stderr, r.stderr
    assert "Auto run" not in r.stdout
    assert os.listdir(tmp_path) == []          # no svc_tmp.pit.csv, nor any other file


def _touch(path):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w", encoding="utf-8") as f:
        f.write("0m 0s   0,200\n")


def test_batch_pitch_lookup_is_feat_then_svc_out(tmp_path, monkeypatch):
    import svc_inference_batch as B
    monkeypatch.chdir(tmp_path)
    feat = str(tmp_path / "feat")
    out = os.path.join(B.out_path, "x.wav.pit.csv")
    assert B.feature_path(feat, "x.wav", ".pit.csv") == out      # nothing yet: where the F0 pass writes
    _touch(out)
    assert B.feature_path(feat, "x.wav", ".pit.csv") == out
    _touch(os.path.join(feat, "x.pit.csv"))
    assert B.feature_path(feat, "x.wav", ".pit.csv") == os.path.join(feat, "x.pit.csv")
    for ext in (".ppg.npy", ".vec.npy"):                         # the same rule for the other two features
        assert B.feature_path(feat, "x.wav", ext) == os.path.join(B.out_path, "x.wav" + ext)


def test_batch_never_schedules_a_given_pitch_file(tmp_path, monkeypatch):
    import svc_inference_batch as B
    monkeypatch.chdir(tmp_path)
    feat = str(tmp_path / "feat")
    waves = ["a.wav", "b.wav", "c.wav", "d.wav"]
    _touch(os.path.join(feat, "b.pit.csv"))
    _touch(os.path.join(feat, "d.wav.pit.csv"))    # not `<stem>.pit.csv`: d has no pitch file
    _touch(os.path.join(B.out_path, "c.wav.pit.csv"))   # left by an earlier run: extracted again, like the PPG and units
    assert B.missing_pitch(waves, [3, 1, 0, 2], feat) == [3, 0, 2]
    assert B.missing_pitch(waves, [1], feat) == []
    assert B.missing_pitch(waves, [], feat) == []
