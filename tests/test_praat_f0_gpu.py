"""Praat autocorrelation F0 on the device (svcb_praat_f0_ragged, praat_f0.py, preprocess_f0_mouth.py).

The device equals the oracle on the fixture (tests/golden/praat_f0_synth.npz): voiced / unvoiced agrees in every frame
and voiced F0 to 1e-9 relative.  Every item's F0 is bitwise the same alone, in ragged batches of mixed lengths (the
one-frame minimum, lengths off the 160-sample grid, more than one pass of 128 items) and in any order.  Short items
and bad offsets are refused before any launch.  The CLI end to end writes the files the oracle predicts."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy.io import wavfile

from oracle import praat_f0_oracle as O
from tests.util import ROOT
from whisper_vits_svc_b200 import _lib, praat_f0

pytestmark = pytest.mark.gpu

GROUP = 128   # items per pass (csrc/praat_f0_api.cu PR_GROUP)


def _raw(clips):
    ex = praat_f0.Extractor("cuda")
    try:
        return [f.cpu().numpy() for f in ex.raw(clips)]
    finally:
        ex.close()


def _clip(n, rng):
    tr = np.full(n, rng.uniform(60, 900))
    return (O.tone(tr, rng) + 0.001 * rng.standard_normal(n)).astype(np.float32)


def test_fixture():
    g = O.load_golden()
    names = sorted(g)
    got = _raw([g[k][0] for k in names])
    worst = 0.0
    for k, f in zip(names, got):
        want = g[k][1]
        assert f.dtype == np.float64 and f.shape == want.shape, k
        assert np.array_equal(f > 0, want > 0), k
        v = want > 0
        if v.any():
            rel = np.abs(f[v] - want[v]) / want[v]
            worst = max(worst, float(rel.max()))
            assert rel.max() <= 1e-9, (k, rel.max())
        assert not f[~v].any(), k
    print(f"worst relative difference on voiced frames: {worst:.2e}")
    padded = praat_f0.f0_batch([g["glide"][0]])[0]
    assert padded.shape == (g["glide"][1].shape[0] + 12,) and not padded[:6].any() and not padded[-6:].any()


def test_batch_invariance_and_order():
    rng = np.random.default_rng(7)
    g = O.load_golden()
    clips = [g[k][0] for k in sorted(g)]
    for n in (1600, 1601, 1760, 1761, 1919, 3333, 4807, 33333):   # the one-frame minimum and lengths off the grid
        clips.append(_clip(n, rng))
    lone = [_raw([c])[0] for c in clips]
    for c, f in zip(clips, lone):
        assert f.shape == (praat_f0.frames_of(c.shape[0]),)
    for _ in range(2):
        order = rng.permutation(len(clips))
        outs = _raw([clips[i] for i in order])
        for o, i in zip(outs, order):
            assert np.array_equal(o, lone[i]), (i, clips[i].shape)


def test_more_than_one_pass():
    rng = np.random.default_rng(3)
    clips = [_clip(int(rng.integers(1600, 5000)), rng) for _ in range(GROUP + 7)]
    outs = _raw(clips)
    for i in (0, 5, GROUP - 1, GROUP, len(clips) - 1):
        assert np.array_equal(outs[i], _raw([clips[i]])[0]), i
    for i in (2, GROUP + 3):
        want = O.praat_f0_unpadded(clips[i])
        assert np.array_equal(outs[i] > 0, want > 0), i


def test_short_items_and_bad_offsets_rejected():
    lib = _lib.load()
    x = torch.zeros(4000, dtype=torch.float64, device="cuda")
    out = torch.full((64,), 7.0, dtype=torch.float64, device="cuda")
    ws = torch.empty(lib.svcb_praat_f0_workspace_bytes(4000, 2), dtype=torch.uint8, device="cuda")
    cases = ([0, 1599, 3500], [0, 2000, 1900], [-1, 1800, 3600], [0, 0, 2000])
    for offs in cases:
        o = (ctypes.c_int64 * 3)(*offs)
        with pytest.raises(_lib.SvcbError, match="svcb_praat_f0_ragged"):
            _lib.call("praat_f0_ragged", x.data_ptr(), o, 2, out.data_ptr(), ws.data_ptr(), ws.numel())
    with pytest.raises(_lib.SvcbError, match="0.1 s analysis window"):
        _lib.call("praat_f0_ragged", x.data_ptr(), (ctypes.c_int64 * 3)(0, 1599, 3500), 2, out.data_ptr(), ws.data_ptr(),
                  ws.numel())
    with pytest.raises(_lib.SvcbError, match="need at least one item"):
        _lib.call("praat_f0_ragged", x.data_ptr(), (ctypes.c_int64 * 1)(0), 0, out.data_ptr(), ws.data_ptr(), ws.numel())
    with pytest.raises(_lib.SvcbError, match="workspace"):
        _lib.call("praat_f0_ragged", x.data_ptr(), (ctypes.c_int64 * 3)(0, 2000, 4000), 2, out.data_ptr(), ws.data_ptr(),
                  1024)
    with pytest.raises(_lib.SvcbError, match="svcb_praat_f0_ragged"):
        praat_f0.f0_batch([np.zeros(2000), np.zeros(1500)])
    torch.cuda.synchronize()
    assert torch.all(out == 7.0)   # nothing was launched
    assert praat_f0.f0_batch([]) == []


def test_cli_end_to_end(tmp_path):
    g = O.load_golden()
    pcm = lambda x: np.clip(np.rint(x * 32767), -32768, 32767).astype(np.int16)
    files = {"spk_a/glide": (16000, pcm(g["glide"][0])), "spk_a/vib": (16000, pcm(g["vibrato"][0])),
             "spk_b/on": (16000, pcm(g["onsets"][0])), "spk_b/silence": (16000, pcm(g["silence"][0])),
             "spk_b/low8k": (8000, pcm(g["tone_220"][0][::2])), "spk_b/edge": (16000, pcm(g["short_1600"][0])),
             "spk_b/tiny": (16000, pcm(g["short_1600"][0][:1599]))}
    for name, (sr, x) in files.items():
        os.makedirs(tmp_path / "wav" / os.path.dirname(name), exist_ok=True)
        wavfile.write(tmp_path / "wav" / f"{name}.wav", sr, x)
    (tmp_path / "wav" / "spk_b" / "broken.wav").write_bytes(b"RIFF....")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "preprocess_f0_mouth.py"), "-w", "wav", "-p", "pit", "-t", "2",
                        "--batch", "3"], cwd=tmp_path, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert r.stdout.splitlines()[:2] == ["wav", "pit"]
    assert "tiny.wav" in r.stderr and "broken.wav" in r.stderr and "2 of 8 files failed" in r.stderr
    from whisper_vits_svc_b200 import hubert_infer
    assert not (tmp_path / "pit" / "spk_b" / "broken.pit.npy").exists()
    for name in files:
        p = tmp_path / "pit" / f"{name}.pit.npy"
        if name.endswith("tiny"):
            assert not p.exists()
            continue
        got = np.load(p)
        x = hubert_infer.load_audio(str(tmp_path / "wav" / f"{name}.wav"), 16000)
        want = O.praat_f0(x)
        assert got.dtype == np.float64 and got.shape == want.shape, name
        assert np.array_equal(got > 0, want > 0), name
        v = want > 0
        assert np.all(np.abs(got[v] - want[v]) <= 1e-9 * want[v]), name
