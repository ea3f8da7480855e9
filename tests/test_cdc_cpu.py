"""Cutting the two lowest STFT bins without a device: the oracle's files against the unmodified reference script, the
fixture, the fp64 formula the kernel evaluates against the oracle, the loader's accept / reject rules, the CLI's flags,
walk and output paths, and the C ABI's checks of its offsets before any launch."""
import os
import subprocess
import sys

import numpy as np
import pytest
from scipy.io import wavfile

from oracle import cdc_oracle as CO, ref_import
from tests.util import ROOT
from whisper_vits_svc_b200 import _lib, cdc

CLI = os.path.join(ROOT, "preprocess_cdc.py")


def within_gate(tag, got, want):
    """Every sample within 1 LSB of the oracle; returns how many differ (the callers bound the share)."""
    assert got.dtype == np.int16 and got.shape == want.shape, (tag, got.shape, want.shape)
    d = np.abs(got.astype(np.int32) - want.astype(np.int32))
    assert d.max(initial=0) <= 1, (tag, int(d.max()))
    return int((d > 0).sum())


def formula(x):
    """The kernel's evaluation in numpy fp64: y(p) = xp(p) - sum_f w c_f / sum_f w^2 over the frames covering p, with
    c_f(m) = A0 / 1024 + (A1 cos + S sin)(2 pi m / 1024) / 512 from the frame's reflect-padded samples; then rounded
    to float32, x 32768, clamped and truncated."""
    x = np.asarray(x, np.float64)
    n = x.shape[0]
    H = n // 256
    m = np.arange(1024)
    w = 0.5 - 0.5 * np.cos(2 * np.pi * m / 1024)
    gc, gs = w * np.cos(2 * np.pi * m / 1024), w * np.sin(2 * np.pi * m / 1024)
    frames = np.lib.stride_tricks.sliding_window_view(np.pad(x, 512, mode="reflect"), 1024)[::256][:H + 1]
    c = np.stack([frames @ w / 1024, frames @ gc / 512, frames @ gs / 512], 1)   # [H + 1, 3]
    num, den = np.zeros(256 * H), np.zeros(256 * H)
    p = np.arange(256 * H) + 512
    for j in range(4):   # frame (p // 256) - 3 + j reaches p at m = p % 256 + 256 (3 - j)
        f = p // 256 - 3 + j
        ok = (f >= 0) & (f <= H)
        mm = p % 256 + 256 * (3 - j)
        fc = c[np.clip(f, 0, H)]
        num += ok * (fc[:, 0] * w[mm] + fc[:, 1] * gc[mm] + fc[:, 2] * gs[mm])
        den += ok * w[mm] ** 2
    y = (x[:256 * H] - num / den).astype(np.float32) * np.float32(32768)
    return np.trunc(np.clip(y, -32768, 32767)).astype(np.int16)


@pytest.mark.skipif(not ref_import.available(), reason="reference tree absent")
def test_oracle_files_byte_equal_reference(tmp_path):
    ref = CO.reference_cut_direct_content()
    g = CO.load_golden()
    lens = {x.shape[0] for _, x, _ in g.values()}
    assert 513 in lens and any(n % 256 == 0 for n in lens) and any(n % 256 == 255 for n in lens)
    for name, (sr, x, _) in g.items():
        src, a, b = tmp_path / f"{name}.wav", tmp_path / "ref.wav", tmp_path / "ours.wav"
        wavfile.write(src, sr, x)
        ref(str(src), str(a))
        wavfile.write(b, sr, CO.cdc(CO.decode(str(src))[0]))
        assert a.read_bytes() == b.read_bytes(), name


def test_golden_reproduces_and_hits_both_rails():
    g, clips = CO.load_golden(), CO.synth_clips()
    assert sorted(g) == sorted(clips)
    assert {sr for sr, _, _ in g.values()} == {48000, 22050, 16000}
    lens = {x.shape[0] for _, x, _ in g.values()}
    assert {513, 767, 1024, 48000, 3 * 48000 + 129} <= lens
    both = False
    for name, (sr, x, y) in g.items():
        assert sr == clips[name][0] and np.array_equal(x, clips[name][1]), name
        assert x.dtype == y.dtype == np.int16 and y.shape == (cdc.out_len(x.shape[0]),), name
        assert within_gate(name, CO.cdc(x.astype(np.float32) / np.float32(32768)), y) <= 0.002 * y.size + 1, name
        both |= bool((y == 32767).any() and (y == -32768).any())
    assert both, "no fixture clip reaches both int16 rails"


def test_formula_within_gate_of_oracle():
    """The fp64 formula the kernel evaluates against the oracle's float32 outputs, with the GPU suite's gate."""
    bad = total = 0
    for name, (sr, x, y) in CO.load_golden().items():
        bad += within_gate(name, formula(x.astype(np.float32) / np.float32(32768)), y)
        total += y.size
    print(f"fp64 formula: {bad} of {total} samples differ from the oracle by 1 LSB")
    assert bad <= 0.002 * total


def test_load_accepts_and_rejects(tmp_path):
    rng = np.random.default_rng(3)
    x = np.clip(0.4 * rng.standard_normal(2000), -1, 1)
    for tag, data in (("i16", (x * 32767).astype(np.int16)), ("i32", (x * 2 ** 31 * 0.99).astype(np.int32)),
                      ("u8", (x * 127 + 128).astype(np.uint8)), ("f32", (1.5 * x).astype(np.float32))):
        path = str(tmp_path / f"{tag}.wav")
        wavfile.write(path, 22050, data)
        got, rate = cdc.load(path)
        want, r2 = CO.decode(path)
        assert rate == r2 == 22050 and got.dtype == np.float32 and np.array_equal(got, want[0].numpy()), tag
    for tag, data, why in (("stereo", np.zeros((2000, 2), np.int16), "2 channels"),
                           ("empty", np.zeros(0, np.int16), "0 samples"),
                           ("short", np.ones(512, np.int16), "512 samples"),
                           ("nan", np.where(np.arange(1000) == 7, np.nan, 0.1).astype(np.float32), "non-finite"),
                           ("inf", np.where(np.arange(1000) == 9, -np.inf, 0.1).astype(np.float32), "non-finite")):
        path = str(tmp_path / f"{tag}.wav")
        wavfile.write(path, 48000, data)
        with pytest.raises(ValueError, match=why):
            cdc.load(path)
    wavfile.write(tmp_path / "ok513.wav", 48000, np.ones(513, np.int16))
    assert cdc.load(str(tmp_path / "ok513.wav"))[0].shape == (513,)


@pytest.mark.parametrize("n", [513, 767, 768, 769, 1024, 3 * 48000 + 129])
def test_out_len(n):
    assert cdc.out_len(n) == 256 * (n // 256) == CO.cdc(np.zeros(n, np.float32)).shape[0]


def test_cli_flags():
    r = subprocess.run([sys.executable, CLI, "-h"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0
    for flag in ("-i INPATH", "-o OUTPATH", "-t THREAD_COUNT, --thread_count THREAD_COUNT", "--batch BATCH"):
        assert flag in r.stdout, flag


def test_cli_walk_and_output_paths(tmp_path, monkeypatch):
    import importlib.util
    monkeypatch.chdir(tmp_path)
    for s in ("bob", "alice"):
        (tmp_path / "raw" / s).mkdir(parents=True)
        for f in ("b.wav", "a.wav", "notes.txt", "c.WAV.bak"):
            (tmp_path / "raw" / s / f).write_bytes(b"")
    (tmp_path / "raw" / "top.wav").write_bytes(b"")            # not in a speaker directory: not taken
    spec = importlib.util.spec_from_file_location("preprocess_cdc_cli", CLI)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    jobs = m.cdc_jobs("raw", "out")
    assert jobs == [(f"raw/{s}/{f}.wav", f"out/{s}/{f}.wav") for s in ("alice", "bob") for f in ("a", "b")]
    # the reference's paths: iWave = ./{in}/{spk}/{file}, oWave = ./{out}/{spk}/{file}
    ref = sorted((f"./raw/{s}/{f}", f"./out/{s}/{f}") for s in os.listdir("raw") if os.path.isdir(f"./raw/{s}")
                 for f in os.listdir(f"./raw/{s}") if f.endswith(".wav"))
    assert [(os.path.normpath(a), os.path.normpath(b)) for a, b in jobs] == [(os.path.normpath(a), os.path.normpath(b))
                                                                            for a, b in ref]
    assert (tmp_path / "out" / "alice").is_dir() and (tmp_path / "out" / "bob").is_dir()
    wavfile.write(tmp_path / "out" / "alice" / "a.wav", 16000, np.ones(10, np.int16))
    assert m.cdc_jobs("raw", "out") == jobs                      # existing outputs are overwritten, not skipped


def test_offsets_rejected_before_any_launch():
    # The checks run on the host before the stream or a device pointer is touched: dummy pointers, null stream.
    import ctypes
    lib = _lib.load()
    d = 256

    def rejects(st, *parts):
        msg = lib.svcb_last_error().decode()
        assert st == -1, msg   # SVCB_E_BAD_SHAPE
        for p in parts:
            assert p in msg, msg

    o = _lib.offsets
    rejects(lib.svcb_cdc_ragged(d, o([]), 0, d, None), "svcb_cdc_ragged", "B = 0; need at least one item")
    rejects(lib.svcb_cdc_ragged(d, o([1000, 512]), 2, d, None), "item 1 has 512 samples", "513", "reflect padding")
    dec = (ctypes.c_int64 * 3)(0, 1000, 600)
    rejects(lib.svcb_cdc_ragged(d, dec, 2, d, None), "item 1 has -400 samples", "decrease")
    rejects(lib.svcb_cdc_ragged(d, (ctypes.c_int64 * 2)(-1, 1000), 1, d, None), "negative first offset")
    rejects(lib.svcb_cdc_ragged(None, o([1000]), 1, d, None), "null pointer")
