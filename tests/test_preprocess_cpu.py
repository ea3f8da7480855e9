"""Dataset feature preparation without a device: pad_or_trim against the reference, the PPG row rule, the ragged
batch plan, the CLIs' walk and skip rule, and the shared loader's retry path."""
import contextlib
import importlib.util
import io
import os

import numpy as np
import pytest

from oracle import preprocess_oracle as PO, ref_import
from tests.util import ROOT
from whisper_vits_svc_b200 import dataset, whisper_infer

S15, S30 = 240000, 480000
LENGTHS = [1, 319, 320, 16000 * 5 + 7, S15 - 1, S15, S15 + 1, S15 + 161, 16000 * 27 + 3, S30 - 1, S30, S30 + 1, 16000 * 41]


def _cli(name):
    spec = importlib.util.spec_from_file_location(name.replace(".py", "_cli"), os.path.join(ROOT, name))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


@pytest.mark.parametrize("n", LENGTHS)
def test_pad_or_trim_constructed(n):
    """Under 15 s -> exactly 15 s (zeros appended), 15-30 s unchanged, over 30 s -> the first 30 s."""
    x = np.random.default_rng(n).standard_normal(n).astype(np.float32)
    for f in (whisper_infer.pad_or_trim, PO.pad_or_trim):
        y = f(x)
        assert y.dtype == np.float32
        assert y.shape[0] == min(max(n, S15), S30)
        k = min(n, S30)
        assert np.array_equal(y[:k], x[:k]) and not y[k:].any()


@pytest.mark.skipif(not ref_import.available(), reason="reference tree absent")
@pytest.mark.parametrize("n", LENGTHS)
def test_pad_or_trim_matches_reference_live(n):
    ref = PO.reference_pad_or_trim()
    x = np.random.default_rng(n).standard_normal(n).astype(np.float32)
    want = ref(x)
    assert np.array_equal(whisper_infer.pad_or_trim(x), want) and np.array_equal(PO.pad_or_trim(x), want)


@pytest.mark.parametrize("n", LENGTHS)
def test_ppg_row_rule(n):
    """rows = min(audln // 320, encoder positions of the pad_or_trim-ed audio)."""
    F = PO.pad_or_trim(np.zeros(n, np.float32)).shape[0] // 160
    want = min(n // 320, (F - 1) // 2 + 1)
    assert whisper_infer.ppg_rows(n) == want
    assert want == (1500 if n >= S30 else n // 320)


def test_plan_window_caps_and_coverage():
    rng = np.random.default_rng(3)
    sizes = [int(s) for s in rng.integers(2 * 16000, 28 * 16000, 300)] + [S30 * 40]   # one file over the budget
    max_items, budget = 16, 16 * 10 * 16000
    plan = dataset.plan_window(sizes, max_items, budget)
    flat = sorted(i for g in plan for i in g)
    assert flat == list(range(len(sizes)))                          # every file exactly once
    for g in plan:
        assert 1 <= len(g) <= max_items
        assert len(g) == 1 or len(g) * max(sizes[i] for i in g) <= budget
    assert [len(sizes) - 1] in plan                                 # over the budget: alone
    padded = sum(len(g) * max(sizes[i] for i in g) for g in plan[:-1])
    assert padded / sum(sizes[:-1]) < 1.1                           # sorted windows keep the padding small


def test_run_batched_bounded_lookahead_and_stats():
    """Loads never run more than one window ahead of the batch being processed; every key is processed once."""
    state = {"loaded": 0, "ran": 0, "max_ahead": 0}
    keys = list(range(100))

    def load(k):
        state["loaded"] += 1
        return np.zeros(1000 + 37 * (k % 11), np.float32)

    def run(items):
        state["max_ahead"] = max(state["max_ahead"], state["loaded"] - state["ran"])
        state["ran"] += len(items)
        return [a.shape[0] for a in items]

    saved = {}
    st = dataset.run_batched(keys, load, run, saved.__setitem__, 3, 4, size=lambda a: a.shape[0], max_padded=10_000, window=8)
    assert sorted(saved) == keys and st["failed"] == 0
    assert all(saved[k] == 1000 + 37 * (k % 11) for k in keys)
    assert state["max_ahead"] <= 2 * 8
    assert st["samples"] == sum(saved.values()) and st["samples"] <= st["padded"]


def test_run_batched_retries_a_failing_batch_one_by_one():
    """A device batch that fails is retried file by file: only the culprit is lost and named; unreadable files are
    reported and skipped."""
    def load(k):
        if k == "bad.wav":
            raise ValueError("unreadable")
        return np.full(100 + len(k), float(k[1]), np.float32)

    def run(items):
        if any(a[0] == 4 for a in items):
            raise RuntimeError("device rejected item 4")
        return [float(a[0]) for a in items]

    keys = [f"f{i}.wav" for i in range(7)] + ["bad.wav"]
    saved = {}
    err = io.StringIO()
    with contextlib.redirect_stderr(err):
        st = dataset.run_batched(keys, load, run, saved.__setitem__, 2, 3, size=len, max_padded=10_000)
    assert st["failed"] == 2
    assert "bad.wav: unreadable" in err.getvalue() and "f4.wav: device rejected" in err.getvalue()
    assert sorted(saved) == sorted(f"f{i}.wav" for i in (0, 1, 2, 3, 5, 6))
    assert saved["f5.wav"] == 5.0


def test_cli_walk_paths_and_skip_existing(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    for s in ("alice", "bob"):
        (tmp_path / "wav" / s).mkdir(parents=True)
        for f in ("a.wav", "b.wav", "notes.txt"):
            (tmp_path / "wav" / s / f).write_bytes(b"")
    (tmp_path / "wav" / "top.wav").write_bytes(b"")            # not in a speaker directory: not taken
    ppg = _cli("preprocess_ppg.py")
    hub = _cli("preprocess_hubert.py")
    want = [(f"wav/{s}/{f}.wav", f"out/{s}/{f}") for s in ("alice", "bob") for f in ("a", "b")]
    assert ppg.ppg_jobs("wav", "out") == [(w, p + ".ppg") for w, p in want]
    assert hub.vec_jobs("wav", "vec") == [(w, p.replace("out/", "vec/") + ".vec") for w, p in want]
    assert (tmp_path / "out" / "alice").is_dir() and (tmp_path / "vec" / "bob").is_dir()
    np.save(tmp_path / "out" / "alice" / "b.ppg.npy", np.zeros((1, 1280), np.float32))
    assert [w for w, _ in ppg.ppg_jobs("wav", "out")] == ["wav/alice/a.wav", "wav/bob/a.wav", "wav/bob/b.wav"]
    np.save(tmp_path / "vec" / "alice" / "b.vec.npy", np.zeros((1, 256), np.float32))
    assert len(hub.vec_jobs("wav", "vec")) == 4                 # preprocess_hubert.py overwrites existing outputs
