"""Trimming silence on the device (svcb_trim_silence_ragged, trim.py, preprocess_trim.py).

The flags are bitwise the oracle's for every fixture clip (tests/golden/trim_synth.npz), including the RMS 184 / 185
stretches, the half-millisecond ties and the zero-filled ends.  Ragged batches in shuffled order equal lone calls,
batches of more than one pass and of mixed rates equal the host cumulative-sum flags, and the CLI end to end on a small
tree writes files byte-equal to the oracle's, skipping what it must."""
import os
import subprocess
import sys
import wave

import numpy as np
import pytest
from scipy.io import wavfile

from oracle import trim_oracle as TO
from tests.test_trim_cpu import random_clip
from tests.util import ROOT
from whisper_vits_svc_b200 import _lib, trim

pytestmark = pytest.mark.gpu

GROUP = 128      # items per launch (csrc/trim_api.cu TRIM_GROUP)
TILE = 1849      # windows per CTA (TRIM_TILE)
RATES = (48000, 44100, 22050, 16000, 8000, 96000, 192000, 11025)


def test_golden_flags_bitwise():
    g = TO.load_golden()
    names = sorted(g)
    flags = trim.trim_batch([g[k][1] for k in names], [g[k][0] for k in names])
    for k, f in zip(names, flags):
        assert f.dtype == np.uint8 and np.array_equal(f, g[k][2]), k


def test_ragged_shuffled_equals_lone():
    rng = np.random.default_rng(3)
    clips = [(sr, x) for sr, x, _ in TO.load_golden().values()]
    for k, n in enumerate((0, 1, 3199, 3200, 9600 + 48 * TILE, 48 * (2 * TILE + 199) + 17, 250000)):
        sr = RATES[k % len(RATES)]
        x = np.clip(rng.standard_normal(n) * rng.choice([100, 190, 3000]), -32768, 32767).astype(np.int16)
        clips.append((sr, x))
    lone = [trim.trim_batch([x], [sr])[0] for sr, x in clips]
    for (sr, x), f in zip(clips, lone):
        assert np.array_equal(f, TO.numpy_flags(x, sr)), (sr, x.shape)
    for _ in range(2):
        order = rng.permutation(len(clips))
        outs = trim.trim_batch([clips[i][1] for i in order], [clips[i][0] for i in order])
        for o, i in zip(outs, order):
            assert np.array_equal(o, lone[i]), (i, clips[i][1].shape)


def test_more_than_one_pass_and_mixed_rates():
    rng = np.random.default_rng(9)
    items = []
    for k in range(2 * GROUP + 9):
        sr = RATES[int(rng.integers(len(RATES)))]
        items.append((sr, random_clip(rng, sr) if k % 3 else
                      np.clip(rng.standard_normal(int(rng.integers(0, sr))) * 184.3, -32768, 32767).astype(np.int16)))
    flags = trim.trim_batch([x for _, x in items], [sr for sr, _ in items])
    assert len(flags) == len(items)
    for (sr, x), f in zip(items, flags):
        assert np.array_equal(f, TO.numpy_flags(x, sr)), (sr, x.shape)
    for i in (0, GROUP - 1, GROUP, 2 * GROUP, len(items) - 1):
        assert np.array_equal(flags[i], trim.trim_batch([items[i][1]], [items[i][0]])[0]), i


def test_bad_rate_rejected():
    with pytest.raises(_lib.SvcbError, match="item 1 has rate 192001"):
        trim.trim_batch([np.zeros(100, np.int16), np.zeros(100, np.int16)], [16000, 192001])
    assert trim.trim_batch([], []) == []


def test_cli_end_to_end(tmp_path):
    raw = tmp_path / "raw"
    for s in ("spk_a", "spk_b"):
        (raw / s).mkdir(parents=True)
    g = TO.load_golden()
    good = {"spk_a/gaps48k": g["gaps48k"], "spk_a/pad44k": g["pad44k"], "spk_a/short16k": g["short16k"],
            "spk_b/level22k": g["level22k"], "spk_b/tie16k_up": g["tie16k_up"], "spk_b/tail44k": g["tail44k"]}
    for name, (sr, x, _) in good.items():
        wavfile.write(raw / f"{name}.wav", sr, x)
    sr, x, _ = g["silent16k"]
    wavfile.write(raw / "spk_b" / "silent.wav", sr, x)
    wavfile.write(raw / "spk_a" / "stereo.wav", 48000, np.stack([g["gaps48k"][1]] * 2, 1))
    with wave.open(str(raw / "spk_b" / "pcm24.wav"), "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(3)
        w.setframerate(48000)
        w.writeframes(bytes(3 * 4800))
    (raw / "spk_a" / "notes.txt").write_text("not audio")
    (tmp_path / "out" / "spk_a").mkdir(parents=True)
    (tmp_path / "out" / "spk_a" / "gaps48k.wav").write_bytes(b"old")   # overwritten
    r = subprocess.run([sys.executable, os.path.join(ROOT, "preprocess_trim.py"), "-i", "raw", "-o", "out", "-t", "2",
                        "--batch", "3"], cwd=tmp_path, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    lines = r.stdout.splitlines()
    assert lines[:2] == ["raw", "out"]
    i = lines.index("list index out of range")
    assert lines[i + 1] == "./raw/spk_b/silent.wav"
    for bad, why in (("stereo.wav", "2 channels"), ("pcm24.wav", "24-bit")):
        line = [s for s in r.stderr.splitlines() if bad in s]
        assert line and line[0].startswith("[!] skipped") and why in line[0], (bad, r.stderr)
    assert "2 of 9 files failed" in r.stderr and "notes.txt" not in r.stderr
    for s in ("spk_a", "spk_b"):
        assert sorted(os.listdir(tmp_path / "out" / s)) == sorted(f"{k.split('/')[1]}.wav" for k in good if k.startswith(s))
    for name, (sr, x, _) in good.items():
        want = tmp_path / "want.wav"
        assert TO.trim_silence(str(raw / f"{name}.wav"), str(want)), name
        assert (tmp_path / "out" / f"{name}.wav").read_bytes() == want.read_bytes(), name
    rate, short = wavfile.read(tmp_path / "out" / "spk_a" / "short16k.wav")
    assert rate == 16000 and short.shape == (2592,) and np.array_equal(short[:2590], g["short16k"][1])
    assert not short[2590:].any()
