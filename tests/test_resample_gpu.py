"""Resampling of raw recordings on the device (svcb_resample_ragged, svcb_pcm16_normalise_ragged, resample.py,
preprocess_a.py).

Parity with the oracle computed live with scipy (resample_poly in float64, cast to float32; the reference's float32
normalisation): float32 outputs within 1 ulp and int16 outputs exactly equal, with the mismatch counts printed (fp64
accumulation makes bitwise agreement the expected case).  Ragged batches bitwise equal to lone runs, passes of more
than one launch, a 10-minute clip whose FIR index passes 2^31, silence, the identity rate, argument checks, and the
CLI end to end on a small tree followed by preprocess_spec.py."""
import ctypes
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy.io import wavfile

from oracle import resample_oracle as RO
from tests.util import ROOT
from whisper_vits_svc_b200 import _lib, resample

pytestmark = pytest.mark.gpu

GROUP = 128   # items per launch (csrc/resample_api.cu RS_GROUP)
RATES = [(44100, 16000), (44100, 32000), (48000, 16000), (48000, 32000), (22050, 16000), (22050, 32000),
         (24000, 16000), (8000, 16000), (16000, 32000), (96000, 16000), (44056, 16000)]


def _clip(seed, n):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 44100
    x = 0.5 * np.sin(2 * np.pi * (110.0 + 53 * (seed % 13)) * t) + 0.1 * rng.standard_normal(n)
    return np.clip(x, -1, 1).astype(np.float32)


def _f32(tag, got, want):
    assert got.dtype == np.float32 and got.shape == want.shape, (tag, got.shape, want.shape)
    bad = got != want
    print(f"{tag}: {int(bad.sum())} of {want.size} float32 outputs differ from the oracle")
    assert np.all(np.abs(got[bad].astype(np.float64) - want[bad]) <= np.spacing(np.abs(want[bad]))), tag
    return int(bad.sum())


def _i16(tag, got, want):
    assert got.dtype == np.int16 and got.shape == want.shape, (tag, got.shape, want.shape)
    bad = int((got != want).sum())
    print(f"{tag}: {bad} of {want.size} int16 outputs differ from the oracle")
    assert bad == 0, tag


@pytest.mark.parametrize("sr_in,sr_out", RATES)
def test_ratio_parity(sr_in, sr_out):
    up, down = resample.ratio(sr_in, sr_out)
    half_span = 10 * max(up, down) // up   # inputs under half the filter
    lens = [1, 2, max(3, half_span - 1), 997, 7919, 48017]
    clips = [_clip(i, n) for i, n in enumerate(lens)]
    out = resample.resample_batch(clips, sr_in, sr_out)
    pcm, peak = resample.pcm16_batch(clips, sr_in, sr_out)
    for n, x, y, p, m in zip(lens, clips, out, pcm, peak):
        want = RO.resample(x, sr_in, sr_out)
        assert y.shape[0] == math.ceil(n * sr_out / sr_in)
        _f32(f"{sr_in}->{sr_out} n={n}", y, want)
        assert m == np.abs(want).max()
        _i16(f"{sr_in}->{sr_out} n={n} int16", p, RO.pcm16(want))


def test_ragged_equals_lone_in_two_orders():
    lens = [1, 5, 441, 30011, 44100 * 3 + 7, 2, 160 * 441 + 1]
    clips = [_clip(20 + i, n) for i, n in enumerate(lens)]
    lone = [resample.resample_batch([c], 44100, 16000)[0] for c in clips]
    lone16 = [resample.pcm16_batch([c], 44100, 16000)[0][0] for c in clips]
    for order in (list(range(len(clips))), list(reversed(range(len(clips))))):
        out = resample.resample_batch([clips[i] for i in order], 44100, 16000)
        pcm = resample.pcm16_batch([clips[i] for i in order], 44100, 16000)[0]
        for o, p, i in zip(out, pcm, order):
            assert np.array_equal(o, lone[i]) and np.array_equal(p, lone16[i]), (i, lens[i])


@pytest.mark.parametrize("sr_in", [48000, 8000])
def test_more_than_one_pass(sr_in):
    rng = np.random.default_rng(sr_in)
    lens = [int(n) for n in rng.integers(1, 3000, GROUP + 9)]
    lens[3:40] = [1] * 37   # a run of one-sample items: tiles straddle many items
    clips = [_clip(100 + i, n) for i, n in enumerate(lens)]
    out = resample.resample_batch(clips, sr_in, 16000)
    pcm, peak = resample.pcm16_batch(clips, sr_in, 16000)
    assert len(out) == len(pcm) == len(peak) == len(clips)
    for i in list(range(0, len(clips), 7)) + [GROUP - 1, GROUP, len(clips) - 1]:
        want = RO.resample(clips[i], sr_in, 16000)
        _f32(f"item {i} ({lens[i]} samples)", out[i], want)
        _i16(f"item {i} int16", pcm[i], RO.pcm16(want))
    assert np.array_equal(out[GROUP], resample.resample_batch([clips[GROUP]], sr_in, 16000)[0])   # second pass


def test_ten_minute_clip_passes_2_31():
    n = 600 * 44100
    up, down = resample.ratio(44100, 16000)
    _, rm = resample.design(up, down)
    assert (resample.out_len(n, 44100, 16000) - 1 + rm) * down > 2 ** 31
    x = _clip(7, n)
    y = resample.resample_batch([x], 44100, 16000)[0]
    want = RO.resample(x, 44100, 16000)
    _f32("10 min 44.1->16", y, want)
    _i16("10 min 44.1->16 int16", resample.pcm16_batch([x], 44100, 16000)[0][0], RO.pcm16(want))


def test_silence_and_identity():
    pcm, peak = resample.pcm16_batch([np.zeros(44100, np.float32), _clip(3, 1000)], 44100, 32000)
    assert peak[0] == 0 and not pcm[0].any() and pcm[0].shape == (32000,) and peak[1] > 0
    x = [_clip(4, 16000), _clip(5, 1)]
    y = resample.resample_batch(x, 16000, 16000)
    assert all(np.array_equal(a, b) for a, b in zip(y, x))
    pcm, peak = resample.pcm16_batch(x, 16000, 16000)
    for a, b, m in zip(pcm, x, peak):
        _i16("identity", a, RO.pcm16(b))
        assert m == np.abs(b).max()


def test_arguments_are_checked():
    dev = torch.device("cuda")
    x = torch.zeros(100, device=dev)
    y = torch.empty(100, device=dev)
    taps = torch.ones(5, dtype=torch.float64, device=dev)
    out16 = torch.empty(100, dtype=torch.int16, device=dev)
    peak = torch.empty(4, device=dev)

    def offs(*v):
        return (ctypes.c_int64 * len(v))(*v)

    for args, match in (((offs(0, 10), 0, 1, 2, 5, 0), "at least one item"),
                        ((offs(0, 10), 1, 0, 2, 5, 0), "need up, down"),
                        ((offs(0, 10), 1, 1, 0, 5, 0), "need up, down"),
                        ((offs(0, 10), 1, 1, 2, 0, 0), "n_taps"),
                        ((offs(0, 10, 10), 2, 1, 2, 5, 0), "item 1 has 0 samples"),
                        ((offs(0, 10, 4), 2, 1, 2, 5, 0), "item 1 has -6 samples")):
        o, B, up, down, nt, rm = args
        with pytest.raises(_lib.SvcbError, match=match):
            _lib.call("resample_ragged", x.data_ptr(), o, B, up, down, taps.data_ptr(), nt, rm, y.data_ptr())
    for o, B, match in ((offs(0, 10), 0, "at least one item"), (offs(0, 0), 1, "item 0 has 0"),
                        (offs(-1, 10), 1, "negative")):
        with pytest.raises(_lib.SvcbError, match=match):
            _lib.call("pcm16_normalise_ragged", y.data_ptr(), o, B, out16.data_ptr(), peak.data_ptr())
    with pytest.raises(_lib.SvcbError, match="item 1 has 0"):
        resample.resample_batch([np.ones(5, np.float32), np.zeros(0, np.float32)], 44100, 16000)


def test_cli_end_to_end(tmp_path):
    raw = tmp_path / "raw"
    for s in ("spk_a", "spk_b"):
        (raw / s).mkdir(parents=True)

    def tone(n, seed):
        return _clip(seed, n).astype(np.float64) * 0.9

    good = {"spk_a/a44": (44100, (tone(44100 * 2 + 17, 1) * 32767).astype(np.int16)),
            "spk_a/b48_stereo": (48000, (np.stack([tone(48000 + 5, 2), tone(48000 + 5, 3)], 1) * 32767).astype(np.int16)),
            "spk_a/c22_i32": (22050, (tone(30001, 4) * 2 ** 31).astype(np.int32)),
            "spk_b/d48_u8": (48000, (tone(20011, 5) * 127 + 128).astype(np.uint8)),
            "spk_b/e16": (16000, (tone(16000 * 3, 6) * 32767).astype(np.int16)),
            "spk_b/f96": (96000, (tone(96000 + 3, 7) * 32767).astype(np.int16))}
    for g, (sr, x) in good.items():
        wavfile.write(raw / f"{g}.wav", sr, x)
    wavfile.write(raw / "spk_a" / "silent.wav", 44100, np.zeros(5000, np.int16))
    wavfile.write(raw / "spk_b" / "empty.wav", 44100, np.zeros(0, np.int16))
    (raw / "spk_b" / "unreadable.wav").write_bytes(b"RIFF\x00\x00not a wav")
    (tmp_path / "configs").mkdir()
    (tmp_path / "configs" / "base.yaml").write_text(open(os.path.join(ROOT, "configs", "base.yaml")).read())
    for sr, out in ((16000, "waves-16k"), (32000, "waves-32k")):
        (tmp_path / out / "spk_a").mkdir(parents=True)
        (tmp_path / out / "spk_a" / "a44.wav").write_bytes(b"old")     # overwritten
        r = subprocess.run([sys.executable, os.path.join(ROOT, "preprocess_a.py"), "-w", "raw", "-o", out, "-s",
                            str(sr), "-t", "2", "--batch", "3"], cwd=tmp_path, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
        assert r.stdout.splitlines()[:3] == ["raw", out, str(sr)]
        for bad, why in (("silent.wav", "silent"), ("empty.wav", "no samples"), ("unreadable.wav", "")):
            line = [s for s in r.stderr.splitlines() if bad in s]
            assert line and line[0].startswith("[!] skipped") and why in line[0], (bad, r.stderr)
        assert "3 of 9 files failed" in r.stderr
        for s in ("spk_a", "spk_b"):
            assert sorted(os.listdir(tmp_path / out / s)) == sorted(f"{g.split('/')[1]}.wav" for g in good if g.startswith(s))
        for g, (sr_in, x) in good.items():
            path = tmp_path / out / f"{g}.wav"
            rate, data = wavfile.read(path)
            assert rate == sr and data.dtype == np.int16 and data.shape == (math.ceil(x.shape[0] * sr / sr_in),), g
            want = tmp_path / "want.wav"
            wavfile.write(want, sr, RO.pcm16(RO.load(str(raw / f"{g}.wav"), sr)))
            assert open(path, "rb").read() == open(want, "rb").read(), (sr, g)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "preprocess_spec.py"), "-w", "waves-32k", "-s", "specs"],
                       cwd=tmp_path, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "failed" not in r.stderr, r.stderr[-3000:]
    for g in good:
        spec = torch.load(tmp_path / "specs" / f"{g}.pt")
        assert spec.shape == (513, wavfile.read(tmp_path / "waves-32k" / f"{g}.wav")[1].shape[0] // 320), g
