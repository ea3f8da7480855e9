"""Resampling of raw recordings without a device: the polyphase formula the kernel evaluates against scipy's
resample_poly, the output length, the oracle's files against the unmodified reference script, the normaliser's
m2 = 0.6 identity, the shared wav decode, the loader's rejections and the CLI's flags, check and walk."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
from scipy.io import wavfile
from scipy.signal import resample_poly

from oracle import ref_import, resample_oracle as RO
from tests.util import ROOT
from whisper_vits_svc_b200 import resample, whisper_infer

CLI = os.path.join(ROOT, "preprocess_a.py")
RATES = [(44100, 16000), (44100, 32000), (48000, 16000), (48000, 32000), (22050, 16000), (22050, 32000),
         (24000, 16000), (8000, 16000), (16000, 32000), (96000, 16000), (44056, 16000)]


def direct(x, up, down, taps, rm):
    """y[j] = sum_k taps[k] xup[(j + rm) down - k], with xup x upsampled by `up` with zeros: the kernel's formula."""
    n, L = x.shape[0], taps.shape[0]
    y = np.empty(-(-n * up // down))
    for j in range(y.shape[0]):
        t = (j + rm) * down
        hi, lo = min(t // up, n - 1), max(0, -(-(t - L + 1) // up))
        i = np.arange(hi, lo - 1, -1)
        y[j] = np.dot(taps[t - i * up], x[i]) if i.size else 0.0
    return y


@pytest.mark.parametrize("sr_in,sr_out", RATES)
def test_formula_equals_resample_poly(sr_in, sr_out):
    up, down = resample.ratio(sr_in, sr_out)
    taps, rm = resample.design(up, down)
    rng = np.random.default_rng(sr_in + sr_out)
    for n in (1, 2, 7, 300, 2000):
        x = rng.uniform(-1, 1, n)
        want = resample_poly(x, up, down)
        got = direct(x, up, down, taps, rm)
        assert got.shape == want.shape and got.shape[0] == resample.out_len(n, sr_in, sr_out), n
        assert np.abs(got - want).max() <= 1e-14, (n, np.abs(got - want).max())


def test_ratio_and_out_len():
    assert resample.ratio(44100, 16000) == (160, 441) and resample.ratio(16000, 16000) == (1, 1)
    assert resample.ratio(44056, 16000) == (2000, 5507)
    for sr_in, sr_out in RATES:
        for n in (1, 2, 3, 441, 1000, 44101):
            assert resample.out_len(n, sr_in, sr_out) == math.ceil(n * sr_out / sr_in) == \
                resample_poly(np.zeros(n), *resample.ratio(sr_in, sr_out)).shape[0]
    with pytest.raises(ValueError):
        resample.ratio(0, 16000)


def test_filter_sizes():
    """The taps the kernel keeps in shared memory (fp64) for the common rates, and the odd rate that does not fit."""
    smem = 200 * 1024   # csrc/resample_api.cu RS_SMEM_MAX, shared with the staged input
    for r, fits in (((44100, 16000), True), ((48000, 16000), True), ((22050, 32000), True), ((44056, 16000), False)):
        up, down = resample.ratio(*r)
        taps, rm = resample.design(up, down)
        half = 10 * max(up, down)
        assert taps.shape[0] == 2 * half + 1 + down - half % down and rm == (half + down - half % down) // down
        assert np.all(taps[:down - half % down] == 0) and taps[down - half % down] != 0
        assert (8 * taps.shape[0] < smem - 32 * 1024) == fits, r


def _sources(tmp_path):
    """Clips the reference decodes alike: 44.1 / 48 / 16 kHz, mono and stereo, int16, int32, uint8 and float32."""
    rng = np.random.default_rng(11)

    def tone(sr, n, f=220.0):
        t = np.arange(n) / sr
        return 0.45 * np.sin(2 * np.pi * f * t) + 0.05 * rng.standard_normal(n)

    srcs = {"a44k_i16.wav": (44100, (tone(44100, 44100 + 37) * 32767).astype(np.int16)),
            "b48k_stereo.wav": (48000, (np.stack([tone(48000, 30011), tone(48000, 30011, 330.0)], 1) * 32767).astype(np.int16)),
            "c44k_i32.wav": (44100, (tone(44100, 20000) * 2 ** 31).astype(np.int32)),
            "d48k_u8.wav": (48000, (tone(48000, 9001) * 127 + 128).astype(np.uint8)),
            "e44k_f32.wav": (44100, tone(44100, 15000).astype(np.float32)),
            "f16k_i16.wav": (16000, (tone(16000, 16003) * 32767).astype(np.int16))}
    for name, (sr, x) in srcs.items():
        wavfile.write(tmp_path / name, sr, x)
    return [str(tmp_path / n) for n in srcs]


@pytest.mark.skipif(not ref_import.available(), reason="reference tree absent")
def test_oracle_files_byte_equal_reference(tmp_path):
    ref = RO.reference_resample_wave()
    for src in _sources(tmp_path):
        for sr in (16000, 32000):
            ref_out, ours = str(tmp_path / f"ref_{sr}.wav"), str(tmp_path / f"ours_{sr}.wav")
            ref(src, ref_out, sr)
            wavfile.write(ours, sr, RO.pcm16(RO.load(src, sr)))
            a, b = open(ref_out, "rb").read(), open(ours, "rb").read()
            assert a == b, (src, sr)
            rate, data = wavfile.read(ours)
            assert rate == sr and data.dtype == np.int16
            assert data.shape[0] == math.ceil(RO.decode(src)[1].shape[0] * sr / RO.decode(src)[0])


def test_m2_is_exactly_0_6():
    rng = np.random.default_rng(2)
    for scale in (1e-30, 3e-5, 0.5, 1.0, 7.0, 1e30):
        for n in (1, 2, 1000):
            y = (rng.standard_normal(n) * scale).astype(np.float32)
            v = y / np.abs(y).max() * 0.6
            assert v.dtype == np.float32 and np.abs(y / np.abs(y).max()).max() == np.float32(1.0)
            assert max(0.01, np.max(np.abs(v))) == np.float32(0.6)


def _load_audio_parent(path, sr):
    """whisper_infer.load_audio as it was before its decode moved into resample.decode_wav."""
    rate, x = wavfile.read(path)
    if x.dtype == np.uint8:
        x = (x.astype(np.float32) - 128.0) / 128.0
    elif x.dtype.kind in "iu":
        x = x.astype(np.float32) / float(np.iinfo(x.dtype).max + 1)
    x = x.astype(np.float32)
    if x.ndim > 1:
        x = x.mean(axis=1)
    if rate != sr:
        g = math.gcd(int(rate), sr)
        x = resample_poly(x, sr // g, int(rate) // g).astype(np.float32)
    return x


def test_shared_decode_keeps_load_audio(tmp_path):
    for src in _sources(tmp_path):
        for sr in (16000, 32000):
            got, want = whisper_infer.load_audio(src, sr), _load_audio_parent(src, sr)
            assert got.dtype == want.dtype == np.float32 and np.array_equal(got, want), (src, sr)
        rate, x = resample.decode_wav(src)
        r2, x2 = RO.decode(src)
        assert rate == r2 and x.dtype == np.float32 and np.array_equal(x, x2), src
        assert np.array_equal(resample.load(src)[0], x) and resample.load(src)[1] == rate


def test_load_rejects_empty_and_non_finite(tmp_path):
    wavfile.write(tmp_path / "empty.wav", 44100, np.zeros(0, np.int16))
    with pytest.raises(ValueError, match="no samples"):
        resample.load(str(tmp_path / "empty.wav"))
    x = np.zeros(100, np.float32)
    x[7] = np.nan
    wavfile.write(tmp_path / "nan.wav", 44100, x)
    with pytest.raises(ValueError, match="non-finite"):
        resample.load(str(tmp_path / "nan.wav"))
    x[7] = np.inf
    wavfile.write(tmp_path / "inf.wav", 44100, x)
    with pytest.raises(ValueError, match="non-finite"):
        resample.load(str(tmp_path / "inf.wav"))


def _cli_module():
    import importlib.util
    spec = importlib.util.spec_from_file_location("preprocess_a_cli", CLI)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_cli_flags_and_rate_check(tmp_path):
    r = subprocess.run([sys.executable, CLI, "-h"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0
    for flag in ("-w WAV, --wav WAV", "-o OUT, --out OUT", "-s SR, --sr SR",
                 "-t THREAD_COUNT, --thread_count THREAD_COUNT", "--batch BATCH"):
        assert flag in r.stdout, flag
    (tmp_path / "raw" / "spk").mkdir(parents=True)
    wavfile.write(tmp_path / "raw" / "spk" / "a.wav", 44100, np.ones(100, np.int16))
    for sr in ("44100", "22050", "0"):
        r = subprocess.run([sys.executable, CLI, "-w", "raw", "-o", "out", "-s", sr], cwd=tmp_path, capture_output=True,
                           text=True, timeout=120)
        assert r.returncode != 0 and "16000 or 32000" in r.stderr, sr
        assert r.stdout.splitlines()[:3] == ["raw", "out", sr]
        assert not (tmp_path / "out" / "spk").exists()


def test_cli_walk_and_loader(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    for s in ("bob", "alice"):
        (tmp_path / "raw" / s).mkdir(parents=True)
        for f in ("b.wav", "a.wav", "notes.txt"):
            (tmp_path / "raw" / s / f).write_bytes(b"")
    (tmp_path / "raw" / "top.wav").write_bytes(b"")            # not in a speaker directory: not taken
    m = _cli_module()
    want = [(f"raw/{s}/{f}.wav", f"out/{s}/{f}.wav") for s in ("alice", "bob") for f in ("a", "b")]
    assert m.resample_jobs("raw", "out") == want
    assert (tmp_path / "out" / "alice").is_dir() and (tmp_path / "out" / "bob").is_dir()
    wavfile.write(tmp_path / "out" / "alice" / "a.wav", 16000, np.ones(10, np.int16))
    assert m.resample_jobs("raw", "out") == want                 # existing outputs are overwritten, not skipped
    wavfile.write(tmp_path / "silent.wav", 48000, np.zeros(500, np.int16))
    with pytest.raises(ValueError, match="silent"):
        m.load_clip(str(tmp_path / "silent.wav"))
    wavfile.write(tmp_path / "ok.wav", 48000, np.arange(500, dtype=np.int16))
    x, rate = m.load_clip(str(tmp_path / "ok.wav"))
    assert rate == 48000 and x.dtype == np.float32 and x.shape == (500,)
    with pytest.raises(ValueError):
        m.load_clip(str(tmp_path / "raw" / "alice" / "a.wav"))   # not a wav at all
