"""Cutting the two lowest STFT bins on the device (svcb_cdc_ragged, cdc.py, preprocess_cdc.py).

Parity with the committed oracle outputs (tests/golden/cdc_synth.npz): equal lengths, every sample within 1 LSB and at
most 0.2 % of the samples different, with the counts printed (the device computes in fp64, the reference's FFTs in
float32).  Ragged batches in shuffled order bitwise equal to lone calls, batches of more than one pass, and the CLI end to
end on a small tree with files it must skip."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy.io import wavfile

from oracle import cdc_oracle as CO
from tests.test_cdc_cpu import within_gate
from tests.util import ROOT
from whisper_vits_svc_b200 import _lib, cdc

pytestmark = pytest.mark.gpu

GROUP = 128   # items per launch (csrc/cdc_api.cu CDC_GROUP)
SHARE = 0.002


def _clip(seed, n, sr=48000):
    """Float32 samples of an int16 clip: harmonics, a DC offset, hum and noise."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / sr
    x = sum(0.25 / k * np.sin(2 * np.pi * k * (100.0 + 31 * (seed % 11)) * t) for k in (1, 2, 3))
    x = x + 0.03 * (seed % 5 - 2) + 0.1 * np.sin(2 * np.pi * (30 + seed % 21) * t) + 0.02 * rng.standard_normal(n)
    return (np.clip(x, -1, 1) * 32767).astype(np.int16).astype(np.float32) / np.float32(32768)


def _gate(tag, outs, wants):
    bad = sum(within_gate(f"{tag} {i}", o, w) for i, (o, w) in enumerate(zip(outs, wants)))
    total = sum(w.size for w in wants)
    print(f"{tag}: {bad} of {total} samples differ from the oracle by 1 LSB")
    assert bad <= SHARE * total, (tag, bad, total)


def test_golden_parity():
    g = CO.load_golden()
    names = sorted(g)
    clips = [g[k][1].astype(np.float32) / np.float32(32768) for k in names]
    outs = cdc.cdc_batch(clips)
    assert [o.shape for o in outs] == [g[k][2].shape for k in names]
    _gate("golden", outs, [g[k][2] for k in names])
    sq = outs[names.index("square48k_9031")]
    assert (sq == 32767).any() and (sq == -32768).any()


def test_ragged_shuffled_equals_lone():
    lens = [513, 767, 768, 1024, 48000, 3 * 48000 + 129, 514, 256 * 61 + 512, 256 * 61 + 511, 256 * 122 + 700, 9000]
    clips = [_clip(10 + i, n) for i, n in enumerate(lens)]
    lone = [cdc.cdc_batch([c])[0] for c in clips]
    _gate("lone", lone, [CO.cdc(c) for c in clips])
    rng = np.random.default_rng(1)
    for _ in range(2):
        order = rng.permutation(len(clips))
        outs = cdc.cdc_batch([clips[i] for i in order])
        for o, i in zip(outs, order):
            assert np.array_equal(o, lone[i]), (i, lens[i])


def test_more_than_one_pass():
    rng = np.random.default_rng(5)
    lens = [int(n) for n in rng.integers(513, 4000, 2 * GROUP + 9)]
    lens[3:60] = [513 + (i % 3) * 255 for i in range(57)]   # runs of 2-hop items: tiles straddle many items
    clips = [_clip(200 + i, n) for i, n in enumerate(lens)]
    outs = cdc.cdc_batch(clips)
    assert len(outs) == len(clips) and all(o.shape == (cdc.out_len(n),) for o, n in zip(outs, lens))
    _gate("multi-pass", outs, [CO.cdc(c) for c in clips])
    for i in (0, GROUP - 1, GROUP, 2 * GROUP, len(clips) - 1):
        assert np.array_equal(outs[i], cdc.cdc_batch([clips[i]])[0]), i


def test_short_item_rejected():
    with pytest.raises(_lib.SvcbError, match="item 1 has 512 samples"):
        cdc.cdc_batch([np.zeros(1000, np.float32), np.zeros(512, np.float32)])
    assert cdc.cdc_batch([]) == []


def test_cli_end_to_end(tmp_path):
    raw = tmp_path / "raw"
    for s in ("spk_a", "spk_b"):
        (raw / s).mkdir(parents=True)

    def pcm(seed, n, sr):
        return (_clip(seed, n, sr) * 32768).astype(np.int16)

    good = {"spk_a/a48": (48000, pcm(1, 48000 * 2 + 17, 48000)),
            "spk_a/b22_i32": (22050, (_clip(2, 30001, 22050).astype(np.float64) * 2 ** 31).astype(np.int32)),
            "spk_a/c513": (48000, pcm(3, 513, 48000)),
            "spk_b/d16_u8": (16000, (_clip(4, 20011, 16000) * 127 + 128).astype(np.uint8)),
            "spk_b/e44_f32": (44100, _clip(5, 44100 + 255, 44100)),
            "spk_b/f48": (48000, pcm(6, 48000 * 3, 48000))}
    for name, (sr, x) in good.items():
        wavfile.write(raw / f"{name}.wav", sr, x)
    wavfile.write(raw / "spk_a" / "stereo.wav", 48000, np.stack([pcm(7, 5000, 48000)] * 2, 1))
    wavfile.write(raw / "spk_b" / "short.wav", 48000, pcm(8, 400, 48000))
    wavfile.write(raw / "spk_b" / "nan.wav", 48000, np.where(np.arange(2000) == 5, np.nan, 0.1).astype(np.float32))
    (raw / "spk_b" / "unreadable.wav").write_bytes(b"RIFF\x00\x00not a wav")
    (raw / "spk_a" / "notes.txt").write_text("not audio")
    (tmp_path / "out" / "spk_a").mkdir(parents=True)
    (tmp_path / "out" / "spk_a" / "a48.wav").write_bytes(b"old")   # overwritten
    r = subprocess.run([sys.executable, os.path.join(ROOT, "preprocess_cdc.py"), "-i", "raw", "-o", "out", "-t", "2",
                        "--batch", "3"], cwd=tmp_path, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert r.stdout.splitlines()[:2] == ["raw", "out"]
    for bad, why in (("stereo.wav", "2 channels"), ("short.wav", "400 samples"), ("nan.wav", "non-finite"),
                     ("unreadable.wav", "")):
        line = [s for s in r.stderr.splitlines() if bad in s]
        assert line and line[0].startswith("[!] skipped") and why in line[0], (bad, r.stderr)
    assert "4 of 10 files failed" in r.stderr and "notes.txt" not in r.stderr
    for s in ("spk_a", "spk_b"):
        assert sorted(os.listdir(tmp_path / "out" / s)) == sorted(f"{g.split('/')[1]}.wav" for g in good if g.startswith(s))
    outs, wants = [], []
    for name, (sr, x) in good.items():
        rate, data = wavfile.read(tmp_path / "out" / f"{name}.wav")
        assert rate == sr and data.dtype == np.int16 and data.shape == (256 * (x.shape[0] // 256),), name
        outs.append(data)
        wants.append(CO.cdc(CO.decode(str(raw / f"{name}.wav"))[0]))
    _gate("cli", outs, wants)
