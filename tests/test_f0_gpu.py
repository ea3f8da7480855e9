"""WORLD DIO + StoneMask F0 on the device (svcb_world_f0_ragged, world_f0.py, preprocess_f0.py).

The device equals the oracle on the fixture (tests/golden/f0_synth.npz): after the 0.1 rounding voiced / unvoiced
agrees in every frame and values differ by at most 0.1 Hz in at most 0.1 % of frames; before rounding voiced frames
agree to 1e-9 relative.  Every item's F0 is bitwise the same alone, in ragged batches of mixed lengths (1-3 frames,
lengths off the 160-sample grid, more than one pass of 128 items) and in any order.  The CLI end to end writes the
files the oracle predicts."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy.io import wavfile

from oracle import f0_oracle as O
from tests.util import ROOT
from whisper_vits_svc_b200 import _lib, world_f0

pytestmark = pytest.mark.gpu

GROUP = 128   # items per pass (csrc/f0_api.cu F0_GROUP)


def _raw(clips):
    ex = world_f0.Extractor("cuda")
    try:
        return [f.cpu().numpy() for f in ex.raw(clips)]
    finally:
        ex.close()


def test_fixture_after_rounding():
    g = O.load_golden()
    names = sorted(g)
    got = world_f0.f0_batch([g[k][0] for k in names])
    total = off = 0
    for k, f in zip(names, got):
        want = O.round1(g[k][1])
        assert f.dtype == np.float64 and f.shape == want.shape, k
        assert np.array_equal(f > 0, want > 0), k
        d = np.abs(f - want)
        assert d.max() <= 0.1 + 1e-9, (k, d.max())
        total += f.shape[0]
        off += int(np.count_nonzero(d))
    print(f"frames differing after rounding: {off} of {total} ({off / total:.4%})")
    assert off <= 0.001 * total, (off, total)


def test_fixture_before_rounding():
    """1e-9 relative on voiced frames, except where DIO's value sits on a step of StoneMask's window length
    int(1.5 fs / f0 + 1): a tone of exactly 100 Hz gives DIO exactly 100.0 (crossings 160 samples apart), where one ulp
    more shortens the window by a sample and moves the refined F0 by 5e-6 relative.  There 1e-5 is allowed."""
    g = O.load_golden()
    names = sorted(g)
    got = _raw([g[k][0] for k in names])
    worst, on_step = 0.0, 0
    for k, f in zip(names, got):
        want = g[k][1]
        assert np.array_equal(f > 0, want > 0), k
        v = want > 0
        if v.any():
            d = O.dio(g[k][0])
            with np.errstate(divide="ignore", invalid="ignore"):
                r = 1.5 * O.FS / d + 1.0
                step = (d > 0) & (np.abs(r - np.rint(r)) <= 1e-9 * r)
            on_step += int(np.count_nonzero(step & v))
            rel = np.abs(f[v] - want[v]) / want[v]
            tol = np.where(step[v], 1e-5, 1e-9)
            worst = max(worst, float(rel[~step[v]].max(initial=0.0)))
            assert np.all(rel <= tol), (k, rel.max())
        assert not f[~v].any(), k
    print(f"worst relative difference on voiced frames off the window steps: {worst:.2e}; frames on a step: {on_step}")


def test_batch_invariance_and_order():
    rng = np.random.default_rng(7)
    g = O.load_golden()
    clips = [g[k][0] for k in sorted(g)]
    for n in (1, 2, 159, 160, 161, 321, 479, 480, 481, 4007, 33333):   # 1-3 frames and lengths off the grid
        tr = np.full(n, rng.uniform(90, 600))
        clips.append((O.tone(tr, rng) + 0.001 * rng.standard_normal(n)).astype(np.float32))
    lone = [_raw([c])[0] for c in clips]
    for c, f in zip(clips, lone):
        assert f.shape == (c.shape[0] // 160 + 1,)
        if c.shape[0] < 480:
            assert not f.any()
    for _ in range(2):
        order = rng.permutation(len(clips))
        outs = _raw([clips[i] for i in order])
        for o, i in zip(outs, order):
            assert np.array_equal(o, lone[i]), (i, clips[i].shape)


def test_more_than_one_pass():
    rng = np.random.default_rng(3)
    clips = []
    for k in range(GROUP + 7):
        n = int(rng.integers(1, 6000))
        tr = np.full(n, rng.uniform(80, 800))
        clips.append((O.tone(tr, rng) + 0.001 * rng.standard_normal(n)).astype(np.float32))
    outs = _raw(clips)
    for i in (0, 5, GROUP - 1, GROUP, len(clips) - 1):
        assert np.array_equal(outs[i], _raw([clips[i]])[0]), i
    for i in (2, GROUP + 3):
        want = O.world_f0(clips[i])
        assert np.array_equal(outs[i] > 0, want > 0), i


def test_bad_offsets_rejected():
    lib = _lib.load()
    x = torch.zeros(1000, dtype=torch.float64, device="cuda")
    out = torch.full((16,), 7.0, dtype=torch.float64, device="cuda")
    ws = torch.empty(lib.svcb_world_f0_workspace_bytes(1000, 2), dtype=torch.uint8, device="cuda")
    cases = ([0, 600, 500], [0, 0, 500], [-1, 400, 900])
    for offs in cases:
        o = (ctypes.c_int64 * 3)(*offs)
        with pytest.raises(_lib.SvcbError, match="svcb_world_f0_ragged"):
            _lib.call("world_f0_ragged", x.data_ptr(), o, 2, out.data_ptr(), ws.data_ptr(), ws.numel())
    with pytest.raises(_lib.SvcbError, match="need at least one item"):
        _lib.call("world_f0_ragged", x.data_ptr(), (ctypes.c_int64 * 1)(0), 0, out.data_ptr(), ws.data_ptr(), ws.numel())
    with pytest.raises(_lib.SvcbError, match="workspace"):
        _lib.call("world_f0_ragged", x.data_ptr(), (ctypes.c_int64 * 3)(0, 500, 1000), 2, out.data_ptr(), ws.data_ptr(), 1024)
    torch.cuda.synchronize()
    assert torch.all(out == 7.0)   # nothing was launched
    assert world_f0.f0_batch([]) == []


def test_cli_end_to_end(tmp_path):
    g = O.load_golden()
    pcm = lambda x: np.clip(np.rint(x * 32767), -32768, 32767).astype(np.int16)
    files = {"spk_a/glide": (16000, pcm(g["glide_up"][0])), "spk_a/vib": (16000, pcm(g["vibrato"][0])),
             "spk_b/vu": (16000, pcm(g["voiced_unvoiced"][0])), "spk_b/silence": (16000, pcm(g["silence"][0])),
             "spk_b/low8k": (8000, pcm(g["glide_down"][0][::2])), "spk_b/tiny": (16000, pcm(g["short"][0][:300]))}
    for name, (sr, x) in files.items():
        os.makedirs(tmp_path / "wav" / os.path.dirname(name), exist_ok=True)
        wavfile.write(tmp_path / "wav" / f"{name}.wav", sr, x)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "preprocess_f0.py"), "-w", "wav", "-p", "pit", "-t", "2",
                        "--batch", "3"], cwd=tmp_path, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert r.stdout.splitlines()[:2] == ["wav", "pit"]
    assert "tiny.wav" in r.stderr and "1 of 6 files failed" in r.stderr
    from whisper_vits_svc_b200 import hubert_infer
    for name in files:
        p = tmp_path / "pit" / f"{name}.pit.npy"
        if name.endswith("tiny"):
            assert not p.exists()
            continue
        got = np.load(p)
        x = hubert_infer.load_audio(str(tmp_path / "wav" / f"{name}.wav"), 16000)
        want = O.round1(O.world_f0(x))
        assert got.dtype == np.float64 and got.shape == (x.shape[0] // 160 + 1,), name
        assert np.array_equal(got > 0, want > 0), name
        assert np.abs(got - want).max() <= 0.1 + 1e-9, name
        assert np.count_nonzero(got != want) <= max(1, 0.001 * got.shape[0]), name
