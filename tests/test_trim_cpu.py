"""Trimming silence without a device: the oracle's RMS against audioop.rms, the files of the unmodified reference
script behind the stub pydub against the CLI's host path fed the oracle's flags, the fixture, trim.py's range rules
against the oracle's, the loader's accept / reject rules, the CLI's flags, walk and output paths, and the C ABI's checks
before any launch."""
import os
import subprocess
import sys
import warnings
import wave

import numpy as np
import pytest
from scipy.io import wavfile

from oracle import ref_import, trim_oracle as TO
from tests.util import ROOT
from whisper_vits_svc_b200 import _lib, trim

CLI = os.path.join(ROOT, "preprocess_trim.py")


def _cli_module():
    import importlib.util
    spec = importlib.util.spec_from_file_location("preprocess_trim_cli", CLI)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def random_clip(rng, rate):
    """A short clip of bursts and quiet stretches of random lengths and levels, some near the threshold."""
    parts = []
    for _ in range(rng.integers(2, 7)):
        kind = rng.choice(["b", "q", "s", "z"], p=[0.4, 0.35, 0.1, 0.15])
        ms = int(rng.integers(40, 600))
        if kind == "b":
            parts.append(("b", ms, float(rng.uniform(500, 20000))))
        elif kind == "q":
            parts.append(("q", ms, float(rng.uniform(5, 260))))
        elif kind == "s":
            parts.append(("s", ms, int(rng.integers(182, 188))))
        else:
            parts.append(("z", ms))
    return TO.compose(rng, rate, parts, n=int(rng.integers(1, 3 * rate)) if rng.random() < 0.3 else None)


def test_oracle_rms_equals_audioop():
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", DeprecationWarning)
        audioop = pytest.importorskip("audioop")
    rng = np.random.default_rng(5)
    cases = [np.zeros(0, np.int16), np.zeros(9600, np.int16), np.full(9600, -32768, np.int16),
             np.full(38400, 32767, np.int16), np.where(np.arange(9600) % 2 == 0, 184, -184).astype(np.int16),
             np.where(np.arange(8820) % 2 == 0, 185, -185).astype(np.int16), np.array([-32768, 32767], np.int16)]
    for _ in range(200):
        n = int(rng.integers(1, 40000))
        scale = float(rng.choice([1, 50, 184.5, 3000, 40000]))
        cases.append(np.clip(rng.standard_normal(n) * scale, -32768, 32767).astype(np.int16))
    for x in cases:
        data = x.astype("<i2").tobytes()
        assert TO.AudioSegment(data, 2, 48000, 1).rms == audioop.rms(data, 2), (x.shape, x[:4])


@pytest.mark.skipif(not ref_import.available(), reason="reference tree absent")
def test_reference_files_byte_equal_host_path(tmp_path, capsys):
    ref = TO.reference_trim_silence()
    g = TO.load_golden()
    silent = set()
    for name, (sr, x, flags) in g.items():
        src, a, b = tmp_path / f"{name}.wav", tmp_path / f"{name}.ref.wav", tmp_path / f"{name}.ours.wav"
        wavfile.write(src, sr, x)
        ref(str(src), str(a))
        ref_out = capsys.readouterr().out
        x2, r2 = trim.load(str(src))
        assert r2 == sr and np.array_equal(x2, x), name
        _cli_module().save_trimmed(f"in/{name}.wav", str(b), x2, r2, flags)
        out = capsys.readouterr().out
        if a.exists():
            assert a.read_bytes() == b.read_bytes(), name
        else:
            silent.add(name)
            assert not b.exists(), name
            assert ref_out.splitlines() == ["list index out of range", str(src)], ref_out
            assert out.splitlines() == ["list index out of range", f"./in/{name}.wav"], out
    assert silent == {"silent16k"}


def test_golden_reproduces_and_covers_the_cases():
    g, clips = TO.load_golden(), TO.synth_clips()
    assert sorted(g) == sorted(clips)
    assert {sr for sr, _, _ in g.values()} == {48000, 44100, 22050, 16000}
    for name, (sr, x, flags) in g.items():
        assert sr == clips[name][0] and np.array_equal(x, clips[name][1]), name
        assert flags.dtype == np.uint8 and flags.shape == (trim.windows(x.shape[0], sr),), name
        assert np.array_equal(TO.window_flags(x, sr), flags), name
        assert np.array_equal(TO.numpy_flags(x, sr), flags), name
    n = {k: v[1].shape[0] for k, v in g.items()}
    assert n["tie16k_down"] == 16008 and trim.length_ms(16008, 16000) == 1000            # 1000.5 -> 1000
    assert n["tie16k_up"] == 16024 and trim.length_ms(16024, 16000) == 1002              # 1001.5 -> 1002
    assert trim.frame(trim.length_ms(n["pad44k"], 44100), 44100) > n["pad44k"]           # the end is zero-filled
    assert g["pad44k"][2][-1] == 0                                                      # ... inside a burst
    assert g["silent16k"][2].all() and g["short16k"][2].size == 0 and g["short48k"][2].size == 0
    # windows wholly inside the 184 stretch are silent and inside the 185 stretch are not, at 48 and 22.05 kHz
    for name in ("level48k", "level22k"):
        sr, x, flags = g[name]
        runs = {}
        for mag in (184, 185):
            on = np.abs(x.astype(np.int32)) == mag
            inside = [i for i in range(flags.size) if on[trim.frame(i, sr):trim.frame(i + 200, sr)].all()]
            runs[mag] = flags[inside]
        assert runs[184].size and runs[184].all() and runs[185].size and not runs[185].any(), name


def test_host_rules_equal_oracle():
    """trim.py's ranges and slicing over the oracle's flags give the oracle's samples: the fixture and seeded random
    clips at four rates."""
    g = TO.load_golden()
    items = [(sr, x, f) for sr, x, f in g.values()]
    rng = np.random.default_rng(21)
    for k in range(60):
        sr = (48000, 44100, 22050, 16000)[k % 4]
        x = random_clip(rng, sr)
        items.append((sr, x, TO.numpy_flags(x, sr)))
    kinds = set()
    for sr, x, flags in items:
        want = TO.trim(x, sr)
        got = trim.trim(x, sr, flags)
        assert (got is None) == (want is None)
        if want is not None:
            assert got.dtype == np.int16 and np.array_equal(got, want), (sr, x.shape)
            kinds.add(len(trim.keep_ranges(flags, trim.length_ms(x.shape[0], sr))))
        else:
            kinds.add(0)
        assert trim.silent_ranges(flags) == TO.detect_silence(TO.AudioSegment(x.tobytes(), 2, sr, 1), 200, -45)
    assert {0, 1, 2, 3} <= kinds


def test_numpy_flags_equal_oracle_loop_on_random_clips():
    rng = np.random.default_rng(8)
    for k in range(24):
        sr = (48000, 44100, 22050, 16000)[k % 4]
        x = random_clip(rng, sr)
        assert np.array_equal(TO.numpy_flags(x, sr), TO.window_flags(x, sr)), (sr, x.shape)


def _write(path, rate, width, channels, frames):
    with wave.open(str(path), "wb") as w:
        w.setnchannels(channels)
        w.setsampwidth(width)
        w.setframerate(rate)
        w.writeframes(frames)


def test_load_accepts_and_rejects(tmp_path):
    x = (np.arange(3000) * 7 % 2000 - 1000).astype(np.int16)
    wavfile.write(tmp_path / "ok.wav", 22050, x)
    got, rate = trim.load(str(tmp_path / "ok.wav"))
    assert rate == 22050 and got.dtype == np.int16 and np.array_equal(got, x)
    wavfile.write(tmp_path / "empty.wav", 16000, np.zeros(0, np.int16))
    assert trim.load(str(tmp_path / "empty.wav"))[0].shape == (0,)
    wavfile.write(tmp_path / "stereo.wav", 48000, np.zeros((100, 2), np.int16))
    _write(tmp_path / "pcm24.wav", 48000, 3, 1, bytes(300))
    wavfile.write(tmp_path / "u8.wav", 48000, np.full(100, 128, np.uint8))
    wavfile.write(tmp_path / "f32.wav", 48000, np.zeros(100, np.float32))
    _write(tmp_path / "fast.wav", 384000, 2, 1, bytes(200))
    (tmp_path / "junk.wav").write_bytes(b"RIFF\x00\x00not a wav")
    for name, why in (("stereo", "2 channels"), ("pcm24", "24-bit"), ("u8", "8-bit"), ("f32", "not a PCM wav"),
                      ("fast", "rate 384000"), ("junk", "not a PCM wav")):
        with pytest.raises(ValueError, match=why):
            trim.load(str(tmp_path / f"{name}.wav"))


@pytest.mark.parametrize("n,rate", [(0, 16000), (3199, 16000), (3200, 16000), (3208, 16000), (16008, 16000),
                                    (16024, 16000), (132323, 44100), (9600, 48000), (9599, 48000), (1, 1)])
def test_windows_match_the_oracle_loop(n, rate):
    seg = TO.AudioSegment(bytes(2 * n), 2, rate, 1)
    assert trim.length_ms(n, rate) == len(seg)
    assert trim.windows(n, rate) == max(len(seg) - 199, 0) == TO.numpy_flags(np.zeros(n, np.int16), rate).size


def test_cli_flags():
    r = subprocess.run([sys.executable, CLI, "-h"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0
    for flag in ("-i INPATH", "-o OUTPATH", "-t THREAD_COUNT, --thread_count THREAD_COUNT", "--batch BATCH"):
        assert flag in r.stdout, flag


def test_cli_walk_and_output_paths(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    for s in ("bob", "alice"):
        (tmp_path / "raw" / s).mkdir(parents=True)
        for f in ("b.wav", "a.wav", "notes.txt", "c.WAV.bak"):
            (tmp_path / "raw" / s / f).write_bytes(b"")
    (tmp_path / "raw" / "top.wav").write_bytes(b"")            # not in a speaker directory: not taken
    m = _cli_module()
    jobs = m.trim_jobs("raw", "out")
    assert jobs == [(f"raw/{s}/{f}.wav", f"out/{s}/{f}.wav") for s in ("alice", "bob") for f in ("a", "b")]
    # the reference's paths: iWave = ./{in}/{spk}/{file}, oWave = ./{out}/{spk}/{file}
    ref = sorted((f"./raw/{s}/{f}", f"./out/{s}/{f}") for s in os.listdir("raw") if os.path.isdir(f"./raw/{s}")
                 for f in os.listdir(f"./raw/{s}") if f.endswith(".wav"))
    assert [(os.path.normpath(a), os.path.normpath(b)) for a, b in jobs] == [(os.path.normpath(a), os.path.normpath(b))
                                                                            for a, b in ref]
    assert (tmp_path / "out" / "alice").is_dir() and (tmp_path / "out" / "bob").is_dir()
    wavfile.write(tmp_path / "out" / "alice" / "a.wav", 16000, np.ones(10, np.int16))
    assert m.trim_jobs("raw", "out") == jobs                     # existing outputs are overwritten, not skipped


def test_offsets_and_rates_rejected_before_any_launch():
    # The checks run on the host before the stream or a device pointer is touched: dummy pointers, null stream.
    import ctypes
    lib = _lib.load()
    d = 256

    def rejects(st, *parts):
        msg = lib.svcb_last_error().decode()
        assert st == -1, msg   # SVCB_E_BAD_SHAPE
        for p in parts:
            assert p in msg, msg

    def rates(*r):
        return (ctypes.c_int32 * len(r))(*r)

    o, f = _lib.offsets, lib.svcb_trim_silence_ragged
    rejects(f(d, o([]), rates(), 0, d, None), "svcb_trim_silence_ragged", "B = 0; need at least one item")
    rejects(f(d, (ctypes.c_int64 * 3)(0, 1000, 600), rates(16000, 16000), 2, d, None), "item 1 has -400 samples",
            "decrease")
    rejects(f(d, (ctypes.c_int64 * 2)(-1, 1000), rates(16000), 1, d, None), "negative first offset")
    rejects(f(d, o([1000, 1000]), rates(16000, 0), 2, d, None), "item 1 has rate 0", "1..192000")
    rejects(f(d, o([1000]), rates(-8000), 1, d, None), "item 0 has rate -8000")
    rejects(f(d, o([1000, 5]), rates(192000, 192001), 2, d, None), "item 1 has rate 192001", "2^53")
    rejects(f(None, o([1000]), rates(16000), 1, d, None), "null pointer")
    rejects(f(d, o([1000]), None, 1, d, None), "null pointer")
