"""Silero VAD on the device (csrc/vad_api.cu) against the live model's fixtures (tests/golden/vad_*.npz), ragged
batches against lone runs, and svc_inference_post.py end to end."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import vad_oracle as VO
from tests.util import ROOT
from whisper_vits_svc_b200 import _lib
from whisper_vits_svc_b200 import vad_infer as V

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def tensors():
    return VO.load_tensors()


@pytest.fixture(scope="module")
def vad(tensors):
    return V.VadB200(tensors, "cuda")


@pytest.fixture(scope="module")
def fixtures():
    out = []
    for name in VO.FIXTURES:
        g = VO.load_golden(name)
        out += [(f"{name}/{c}", g[f"{c}.wav"], g[f"{c}.probs"], g[f"{c}.enc"], g[f"{c}.ts"], float(g[f"{c}.margin"]))
                for c in VO.clips(g)]
    return out


def test_probs_and_encoder_against_live_model(vad, fixtures):
    """All fixture clips as one ragged batch: probabilities within 1e-4 of the live model, the encoder tap within 1e-4
    of max |x|."""
    probs, feats = vad.speech_probs([f[1] for f in fixtures], features=True)
    worst_p = worst_e = 0.0
    for (name, wav, p_ref, e_ref, _, _), p, e in zip(fixtures, probs, feats):
        assert p.shape == p_ref.shape and e.shape == e_ref.shape, name
        dp = float(np.abs(p - p_ref).max())
        de = float(np.abs(e - e_ref).max()) / max(float(np.abs(e_ref).max()), 1e-30)
        print(f"{name}: {p.size} windows, prob max-abs {dp:.2e}, encoder max-abs / max|x| {de:.2e}")
        worst_p, worst_e = max(worst_p, dp), max(worst_e, de)
        assert dp <= 1e-4 and de <= 1e-4, name
    print(f"worst: prob {worst_p:.2e}, encoder {worst_e:.2e}")


def test_timestamps_equal_live_reference(vad, fixtures):
    used = 0
    for name, wav, _, _, ts_ref, margin in fixtures:
        if margin < 1e-3:    # a probability within 1e-3 of a threshold may legitimately land on the other side
            continue
        p = vad.speech_probs([wav])[0]
        ts = V.get_speech_timestamps(p, wav.shape[0], threshold=0.2)
        assert np.array_equal(np.array([[t["start"], t["end"]] for t in ts], np.int64).reshape(-1, 2), ts_ref), name
        used += 1
    assert used >= 2


def _ragged_wavs():
    rng = np.random.default_rng(21)
    test = VO.load_golden("vad_test10s")["test10s.wav"]
    lens = [1, 511, 512, 513, 16000 + 7, 30 * 16000, 60 * 16000]
    wavs = [np.resize(test, n).astype(np.float32) * np.float32(rng.uniform(0.5, 1.5)) for n in lens]
    wavs[1] = (0.3 * rng.standard_normal(511)).astype(np.float32)
    return wavs


def test_ragged_batch_bitwise_equals_single(vad):
    wavs = _ragged_wavs()
    lone = [vad.speech_probs_device([w])[0] for w in wavs]
    for order in (list(range(len(wavs))), [6, 2, 0, 5, 3, 1, 4]):
        p, wo = vad.speech_probs_device([wavs[i] for i in order])
        for pos, i in enumerate(order):
            got = p[wo[pos]:wo[pos + 1]]
            assert got.shape[0] == V.windows(wavs[i].shape[0])
            assert torch.equal(got, lone[i]), (order, i)
    assert all(torch.isfinite(x).all() for x in lone)


def test_empty_items_and_extremes(vad):
    rng = np.random.default_rng(2)
    noise = np.clip(rng.standard_normal(40000) * 2.0, -1, 1).astype(np.float32)   # full scale
    silence = np.zeros(40000, np.float32)
    probs = vad.speech_probs([np.zeros(0, np.float32), noise, np.zeros(0, np.float32), silence])
    assert [p.shape[0] for p in probs] == [0, 79, 0, 79]
    assert np.isfinite(probs[1]).all() and np.isfinite(probs[3]).all()
    assert np.array_equal(probs[1], vad.speech_probs([noise])[0])
    assert vad.speech_probs([np.zeros(0, np.float32)])[0].shape == (0,)


def test_offsets_checked_before_launch(vad):
    lib = _lib.load()
    offs = (V.ctypes.c_int64 * 3)(0, 1000, 500)
    st = lib.svcb_vad_probs(vad._handle, None, offs, 2, None, None, None, 0, V._stream())
    assert st != 0 and b"decrease" in lib.svcb_last_error()


def test_cli_post_end_to_end(tensors, fixtures, tmp_path):
    from scipy.io import wavfile
    from scipy.signal import resample_poly
    (tmp_path / "vad" / "assets").mkdir(parents=True)
    VO.write_jit(str(tmp_path / "vad" / "assets" / "silero_vad.jit"), tensors)
    src = VO.load_golden("vad_test10s")["test10s.wav"]
    ref48 = resample_poly(src, 3, 1)
    stereo = np.stack([ref48, 0.5 * ref48], 1)
    wavfile.write(tmp_path / "ref.wav", 48000, np.clip(stereo * 32768, -32768, 32767).astype(np.int16))
    rng = np.random.default_rng(8)
    svc = (0.1 * rng.standard_normal(2 * src.shape[0] - 3000)).astype(np.float32)
    wavfile.write(tmp_path / "svc.wav", 32000, svc)
    cmd = [sys.executable, os.path.join(ROOT, "svc_inference_post.py"), "--ref", "ref.wav", "--svc", "svc.wav", "--out", "post.wav"]
    r = subprocess.run(cmd, cwd=tmp_path, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert r.stdout.splitlines()[:3] == ["svc in wave : ref.wav", "svc out wave : svc.wav", "svc post wave : post.wav"]
    sr, out = wavfile.read(tmp_path / "post.wav")
    from whisper_vits_svc_b200.whisper_infer import load_audio
    ref16 = load_audio(str(tmp_path / "ref.wav"), 16000)
    assert sr == 32000 and out.dtype == np.float32 and out.shape == (min(2 * ref16.shape[0], svc.shape[0]),)
    model = V.VadB200(tensors, "cuda")
    ts = V.get_speech_timestamps(model.speech_probs([ref16])[0], ref16.shape[0], threshold=0.2)
    assert ts, "the excerpt has speech"
    mask = np.zeros(ref16.shape[0], bool)
    for t in ts:
        mask[t["start"]:t["end"]] = True
    mask = np.repeat(mask, 2)[:out.shape[0]]
    assert np.array_equal(out[mask], svc[:out.shape[0]][mask]) and not out[~mask].any()
    assert 0 < mask.sum() < mask.size

    # no model: a clear message; empty source: no speech, all zeros, without the device
    wavfile.write(tmp_path / "empty.wav", 16000, np.zeros(0, np.int16))
    r = subprocess.run(cmd[:3] + ["empty.wav"] + cmd[4:], cwd=tmp_path, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    assert wavfile.read(tmp_path / "post.wav")[1].shape == (0,)
    r = subprocess.run(cmd, cwd=tmp_path / "vad", capture_output=True, text=True, timeout=600)
    assert r.returncode != 0 and "VAD model not found" in r.stderr
