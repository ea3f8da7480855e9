"""The host steps of svc_preprocessing.py without a device: the speaker average, the training lists and the loader
check against the unmodified reference scripts and classes, and the pipeline's refusal to start without a GPU."""
import contextlib
import importlib.util
import io
import os
import random
import runpy
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import ref_import
from tests.util import ROOT

needs_ref = pytest.mark.skipif(not ref_import.available(), reason="reference tree absent")


def _cli(name):
    spec = importlib.util.spec_from_file_location(name.replace(".py", "_cli"), os.path.join(ROOT, name))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


@contextlib.contextmanager
def _cwd(path):
    old = os.getcwd()
    os.chdir(path)
    try:
        yield
    finally:
        os.chdir(old)


def _run_ref(script, argv):
    """prepare/<script> run as __main__ with argv, in the current directory; its stdout."""
    out = io.StringIO()
    old = sys.argv
    sys.argv = [script] + list(argv)
    try:
        with contextlib.redirect_stdout(out), contextlib.redirect_stderr(io.StringIO()):
            runpy.run_path(os.path.join(ref_import.REF_ROOT, "prepare", script), run_name="__main__")
    finally:
        sys.argv = old
    return out.getvalue()


def _files(root):
    return {os.path.relpath(os.path.join(d, f), root): open(os.path.join(d, f), "rb").read()
            for d, _, fs in os.walk(root) for f in fs}


# ------------------------------------------------------------------------------------------------ step 7
@needs_ref
def test_speaker_ave_matches_reference(tmp_path):
    g = np.random.default_rng(7)
    spk = tmp_path / "data_svc" / "speaker"
    for name, n in (("alto", 5), ("tenor", 3), ("empty", 0)):
        (spk / name).mkdir(parents=True)
        for i in range(n):
            np.save(spk / name / f"{i:03d}.spk.npy", (g.standard_normal(256) * (1 + i)).astype(np.float32))
    (spk / "tenor" / "notes.txt").write_text("not an embedding")
    with _cwd(tmp_path):
        _run_ref("preprocess_speaker_ave.py", ["data_svc/speaker/", "singer_ref"])
        assert _cli("preprocess_speaker_ave.py").main(["data_svc/speaker/", "singer_new"]) == 0
    ref, new = _files(tmp_path / "singer_ref"), _files(tmp_path / "singer_new")
    assert sorted(ref) == ["alto.spk.npy", "tenor.spk.npy"]
    assert new == ref


# ------------------------------------------------------------------------------------------------ step 9
FEATURES = ("speaker/{s}/{f}.spk.npy", "waves-32k/{s}/{f}.wav", "specs/{s}/{f}.pt", "pitch/{s}/{f}.pit.npy",
            "hubert/{s}/{f}.vec.npy", "whisper/{s}/{f}.ppg.npy")


def _train_tree(root):
    """16 items in two speakers; four of them lack one feature file each (never the wave, which the walk starts
    from), and one stray file sits beside the speakers."""
    missing = {3: 0, 6: 2, 9: 4, 12: 5}
    for i in range(16):
        s, f = ("bass", "soprano")[i % 2], f"clip{i:02d}"
        for k, pat in enumerate(FEATURES):
            if missing.get(i) == k:
                continue
            p = root / "data_svc" / pat.format(s=s, f=f)
            p.parent.mkdir(parents=True, exist_ok=True)
            p.write_bytes(b"x")
    (root / "data_svc" / "waves-32k" / "readme.txt").write_text("not a speaker")


@needs_ref
@pytest.mark.parametrize("seed", [0, 1, 1234])
def test_train_lists_match_reference(tmp_path, seed):
    _train_tree(tmp_path)
    train = _cli("preprocess_train.py")
    with _cwd(tmp_path):
        random.seed(seed)
        ref_out = _run_ref("preprocess_train.py", [])
        ref = _files(tmp_path / "files")
        shutil.rmtree(tmp_path / "files")
        random.seed(seed)
        out = io.StringIO()
        with contextlib.redirect_stdout(out):
            assert train.main([]) == 0
    assert out.getvalue() == ref_out and ref_out.count("File isn't existed") == 4
    assert _files(tmp_path / "files") == ref
    assert len(ref["valid.txt"].splitlines()) == 10 and len(ref["train.txt"].splitlines()) == 2


# ------------------------------------------------------------------------------------------------ step 10
HOP = 320


def _zzz_tree(root, rate_of=lambda i: 32000):
    """Items whose useful lengths (pitch frames - 1) fall below 1 s, in both sampler buckets, at and past the 4 s cap,
    and at the sampler's lower boundary, plus one with a missing ppg.  vec and ppg rows are set so that either can be
    the shorter after the x2 repeat, and so that some items are cropped at random."""
    from scipy.io import wavfile
    g = np.random.default_rng(3)
    frames = [50, 120, 151, 160, 230, 301, 340, 401, 420, 650, 800, 260]
    lines = []
    for i, n in enumerate(frames):
        d = root / "data_svc" / f"s{i % 3}"
        d.mkdir(parents=True, exist_ok=True)
        stem = str(d / f"c{i:02d}")
        rate = rate_of(i)
        wav = (g.standard_normal(n * HOP * rate // 32000 + 77) * 3000).astype(np.int16)
        wavfile.write(stem + ".wav", rate, wav)
        torch.save(torch.from_numpy(g.standard_normal((513, n)).astype(np.float32)), stem + ".pt")
        np.save(stem + ".pit.npy", (g.random(n) * 400).astype(np.float32))
        np.save(stem + ".vec.npy", g.standard_normal((n // 2 + (2 if i % 2 else 0), 16)).astype(np.float32))
        if i != len(frames) - 1:
            np.save(stem + ".ppg.npy", g.standard_normal((n // 2 + (0 if i % 2 else 3), 24)).astype(np.float32))
        np.save(stem + ".spk.npy", g.standard_normal(256).astype(np.float32))
        lines.append("|".join(f"{stem}{e}" for e in (".wav", ".pt", ".pit.npy", ".vec.npy", ".ppg.npy", ".spk.npy")))
    (root / "files").mkdir()
    (root / "files" / "valid.txt").write_text("".join(f"{ln}\n" for ln in lines), encoding="utf-8")


def _ref_data_utils():
    ref_import._ensure_path()
    from vits import data_utils
    return data_utils


def _equal(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert x.dtype == y.dtype and x.shape == y.shape and torch.equal(x, y)


@needs_ref
@pytest.mark.parametrize("seed", [0, 5])
def test_loader_check_matches_reference(tmp_path, seed):
    """The reference's loop (every item, then a DataLoader over the bucket sampler) and the restatement, under the same
    seeds: the same filtered items and lengths, the same items, batches and collated tensors."""
    from torch.utils.data import DataLoader
    _zzz_tree(tmp_path)
    R, Z = _ref_data_utils(), _cli("preprocess_zzz.py")
    hp = ref_import.load_hp(os.path.join(ROOT, "configs", "base.yaml"))
    lists = str(tmp_path / "files" / "valid.txt")

    def seeded_set(cls):
        random.seed(seed)
        torch.manual_seed(seed)
        out = io.StringIO()
        with contextlib.redirect_stdout(out):
            ds = cls(lists, hp.data)
        return ds, out.getvalue()

    ref, ref_out = seeded_set(R.TextAudioSpeakerSet)
    ref_items = list(ref)
    sampler = R.DistributedBucketSampler(ref, 4, [150, 300, 450], num_replicas=1, rank=0, shuffle=True)
    ref_batches = list(DataLoader(ref, num_workers=0, shuffle=False, collate_fn=R.TextAudioSpeakerCollate(),
                                  batch_sampler=sampler))

    ds, out = seeded_set(Z.TextAudioSpeakerSet)
    items = [ds[i] for i in range(len(ds))]
    plan = Z.bucket_batches(ds.lengths)
    batches = [Z.collate([ds[i] for i in b]) for b in plan]

    assert out == ref_out == "----------10----------\n"
    assert ds.items == ref.items and ds.lengths == ref.lengths
    assert min(ds.lengths) >= 100 and max(ds.lengths) == 400
    assert plan == sampler.batches and len(plan) == 3
    assert len(items) == len(ref_items) == 10
    for a, b in zip(items, ref_items):
        _equal(a, b)
    assert len(batches) == len(ref_batches)
    for a, b in zip(batches, ref_batches):
        _equal(a, b)


@needs_ref
def test_loader_check_rejects_a_wrong_rate_like_reference(tmp_path):
    _zzz_tree(tmp_path, rate_of=lambda i: 16000 if i == 4 else 32000)
    R, Z = _ref_data_utils(), _cli("preprocess_zzz.py")
    hp = ref_import.load_hp(os.path.join(ROOT, "configs", "base.yaml"))
    lists = str(tmp_path / "files" / "valid.txt")
    with contextlib.redirect_stdout(io.StringIO()):
        sets = [R.TextAudioSpeakerSet(lists, hp.data), Z.TextAudioSpeakerSet(lists, hp.data)]
    k = [i for i, it in enumerate(sets[0].items) if it[0].endswith("c04.wav")][0]
    for ds in sets:
        with pytest.raises(AssertionError, match="sample rate of .*c04.wav is 16000"):
            ds[k]
    (tmp_path / "configs").mkdir()
    shutil.copy(os.path.join(ROOT, "configs", "base.yaml"), tmp_path / "configs")
    with _cwd(tmp_path), pytest.raises(AssertionError):
        Z.main([])


def test_loader_check_main_reads_every_item(tmp_path, capsys):
    _zzz_tree(tmp_path)
    (tmp_path / "configs").mkdir()
    shutil.copy(os.path.join(ROOT, "configs", "base.yaml"), tmp_path / "configs")
    with _cwd(tmp_path):
        assert _cli("preprocess_zzz.py").main([]) == 0
    assert capsys.readouterr().out == "----------10----------\n"


def test_bucket_batches_without_items():
    Z = _cli("preprocess_zzz.py")
    assert Z.bucket_batches([]) == [] and Z.bucket_batches([120, 100]) == []


# ------------------------------------------------------------------------------------------------ the pipeline
@pytest.mark.parametrize("argv", [[], ["-t", "2"], ["-h"]])
def test_pipeline_needs_a_gpu(tmp_path, argv):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "svc_preprocessing.py"), *argv], cwd=tmp_path, env=env,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode != 0
    assert "You need GPU to Train!" in r.stderr and "AssertionError" in r.stderr
    assert r.stdout == ""
    assert os.listdir(tmp_path) == []


@needs_ref
def test_pipeline_runs_the_reference_commands_in_order():
    """The ten commands of the reference's svc_preprocessing.py, with prepare/ dropped and the same arguments."""
    import re
    with open(os.path.join(ref_import.REF_ROOT, "svc_preprocessing.py"), encoding="utf-8") as f:
        ref = re.findall(r'"python prepare/([^"]+)"', f.read())
    P = _cli("svc_preprocessing.py")
    assert len(ref) == 10 and P.STEPS == ref
    for step in P.STEPS:
        run, argv = P.step_main(step)
        assert callable(run) and argv == step.split()[1:]
