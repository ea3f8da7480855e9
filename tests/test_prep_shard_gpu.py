"""Data preparation under torchrun on the device: two ranks on one card, each CLI and svc_preprocessing.py against
one-process runs of the same steps on the same tree, a corrupt wav in one rank's share, and a missing model file."""
import importlib.util
import os
import random
import shutil

import numpy as np
import pytest
import torch

from tests.ranks import RANK_PID_LINES, torchrun
from tests.test_speaker_gpu import CONFIG as SPEAKER_CONFIG
from tests.util import ROOT
from whisper_vits_svc_b200 import synth

pytestmark = pytest.mark.gpu

SEED = 1234
TIMEOUT = 1200
# speaker/file: (seconds, rate), mixed lengths and rates so that the two shares differ in size and count
CLIPS = {"alto/a00": (0.6, 44100), "alto/a01": (1.7, 48000), "alto/a02": (2.6, 16000), "alto/a03": (3.3, 48000),
         "alto/a04": (7.4, 44100), "bass/b00": (1.1, 32000), "bass/b01": (4.9, 48000), "tenor/t00": (1.2, 48000),
         "tenor/t01": (2.1, 44100), "tenor/t02": (5.6, 44100), "tenor/t03": (0.9, 48000)}
BROKEN = "tenor/broken"
# the CLIs svc_preprocessing.py does not run, each on the raw tree: (script, arguments, output directory)
SINGLE = [("preprocess_cdc.py", ["-i", "dataset_raw", "-o", "out/cdc"], "out/cdc"),
          ("preprocess_trim.py", ["-i", "dataset_raw", "-o", "out/trim"], "out/trim"),
          ("preprocess_f0.py", ["-w", "dataset_raw", "-p", "out/world"], "out/world"),
          ("preprocess_f0_mouth.py", ["-w", "dataset_raw", "-p", "out/praat"], "out/praat"),
          ("preprocess_f0_salience.py", ["-w", "dataset_raw", "-p", "out/salience"], "out/salience")]
# runs a script as __main__ and writes its exit status to status.<RANK> in the working directory
WRAPPER = ("import runpy, sys\n"
           "sys.argv = sys.argv[1:]\n"
           "code = 1\n"
           "try:\n"
           "    runpy.run_path(sys.argv[0], run_name='__main__')\n"
           "    code = 0\n"
           "except SystemExit as e:\n"
           "    code = 0 if e.code is None else e.code if isinstance(e.code, int) else 1\n"
           "finally:\n"
           "    open(f\"status.{os.environ['RANK']}\", 'w').write(str(code))\n"
           "sys.exit(code)\n")


def _cli(name):
    spec = importlib.util.spec_from_file_location(name.replace(".py", "_cli"), os.path.join(ROOT, name))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


@pytest.fixture(scope="module")
def models(tmp_path_factory):
    """The five model files at the reference's relative paths (Whisper at a reduced width), and configs/base.yaml."""
    d = tmp_path_factory.mktemp("models")
    dims = dict(synth.WHISPER_LARGE_V2_DIMS, n_audio_state=256, n_audio_head=4, n_audio_layer=4)
    for rel, obj in (("whisper_pretrain/large-v2.pt", synth.whisper_checkpoint(dims, seed=11)),
                     ("hubert_pretrain/hubert-soft-0d54a1f4.pt", synth.hubert_checkpoint(31)),
                     ("speaker_pretrain/best_model.pth.tar", synth.speaker_checkpoint(5)),
                     ("crepe/assets/full.pth", synth.crepe_checkpoint(11, "full"))):
        (d / rel).parent.mkdir(parents=True, exist_ok=True)
        torch.save(obj, d / rel)
    (d / "speaker_pretrain" / "config.json").write_text(SPEAKER_CONFIG)
    (d / "configs").mkdir()
    shutil.copy(os.path.join(ROOT, "configs", "base.yaml"), d / "configs")
    return d


def _tree(root, models, broken=True):
    from scipy.io import wavfile
    shutil.copytree(models, root, dirs_exist_ok=True)
    for i, (rel, (sec, rate)) in enumerate(CLIPS.items()):
        n = int(sec * rate)
        t = np.arange(n) / rate
        g = np.random.default_rng(i)
        x = 0.3 * np.sin(2 * np.pi * (130.0 + 20 * i) * t) * (1 + 0.4 * np.sin(2 * np.pi * 3 * t))
        x = x * (t > 0.3) + 0.02 * g.standard_normal(n)   # a quiet lead-in for the silence trim
        p = root / "dataset_raw" / f"{rel}.wav"
        p.parent.mkdir(parents=True, exist_ok=True)
        wavfile.write(p, rate, (x * 32767).astype(np.int16))
    if broken:
        (root / "dataset_raw" / f"{BROKEN}.wav").write_bytes(b"not a wav file")
    return root


def _torchrun(cwd, script, args):
    """`python -m torch.distributed.run --nproc-per-node 2 script args` in cwd, both ranks on the first visible
    device, with one host thread each (torchrun's default); the ranks are stopped if they outlive TIMEOUT
    (tests/ranks.py).  -> (statuses of ranks 0 and 1, stdout, stderr)."""
    (cwd / "wrapper.py").write_text(RANK_PID_LINES + WRAPPER)
    env = dict(os.environ, CUDA_VISIBLE_DEVICES=os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0],
               OMP_NUM_THREADS="1")
    code, out, err = torchrun(["wrapper.py", os.path.join(ROOT, script), *args], 2, cwd, env, TIMEOUT, cwd)
    if code is None:
        pytest.fail(f"{script}: the ranks did not finish in {TIMEOUT} s")
    status = []
    for r in (0, 1):
        s = cwd / f"status.{r}"
        status.append(int(s.read_text()) if s.exists() else None)
        s.unlink(missing_ok=True)
    return status, out, err


def _in(root, fn):
    cwd = os.getcwd()
    try:
        os.chdir(root)
        return fn()
    finally:
        os.chdir(cwd)


def _files(root, tops):
    return {os.path.relpath(os.path.join(d, f), root): os.path.join(d, f)
            for top in tops for d, _, fs in os.walk(root / top) for f in fs}


def _same(a, b, shape_only=()):
    """Byte-equal files, except those under `shape_only` (drawn from the global RNG): dtype and shape."""
    assert sorted(a) == sorted(b)
    bad = []
    for k in sorted(a):
        if k.startswith(shape_only):
            x, y = np.load(a[k]), np.load(b[k])
            if not (x.dtype == y.dtype and x.shape == y.shape):
                bad.append(k)
        else:
            with open(a[k], "rb") as f, open(b[k], "rb") as g:
                if f.read() != g.read():
                    bad.append(k)
                    if k.endswith(".npy"):
                        print(f"{k}: max-abs {np.abs(np.load(a[k]) - np.load(b[k])).max():.3e}")
    assert not bad, bad


def test_each_cli_on_two_ranks_equals_one_process(tmp_path, models, capfd):
    """cdc, trim and the WORLD, Praat and salience F0 on two ranks write what one process writes; the corrupt wav
    falls in one rank's share, is reported there, counted once in rank 0's summed line, and both ranks exit 0."""
    two = _tree(tmp_path / "two", models)
    one = _tree(tmp_path / "one", models)
    for script, args, out in SINGLE:
        status, _, err = _torchrun(two, script, args)
        assert status == [0, 0], (script, err[-3000:])
        assert err.count(f"[!] skipped dataset_raw/{BROKEN}.wav") == 1, (script, err[-3000:])
        assert err.count(f"1 of {len(CLIPS) + 1} files failed") == 1, (script, err[-3000:])
        capfd.readouterr()
        assert _in(one, lambda: _cli(script).main(args)) == 0, script
        assert f"1 of {len(CLIPS) + 1} files failed" in capfd.readouterr().err
        got, want = _files(two, [out]), _files(one, [out])
        assert len(want) == len(CLIPS), script
        _same(got, want)


def test_pipeline_on_two_ranks_equals_one_process(tmp_path, models):
    """svc_preprocessing.py on two ranks: the same data_svc/ tree and list entries as one process.  CREPE's noise and
    the list shuffle are drawn from the global RNG, so pitch files are compared by dtype and shape and the lists by
    their entries; everything else byte for byte.  torchrun starts its ranks with OMP_NUM_THREADS=1, and the host
    reduction that folds HuBERT's positional-conv weight norm at load sums in an order that follows torch's thread
    count, so the one-process run uses one thread too."""
    P = _cli("svc_preprocessing.py")
    two = _tree(tmp_path / "two", models, broken=False)
    one = _tree(tmp_path / "one", models, broken=False)
    status, out, err = _torchrun(two, "svc_preprocessing.py", ["-t", "2"])
    assert status == [0, 0], out[-3000:] + err[-3000:]
    assert [ln for ln in out.splitlines() if ln.startswith("Command: ")] == [f"Command: python {s}" for s in P.STEPS]

    def seeded():
        torch.manual_seed(SEED)
        random.seed(SEED)
        np.random.seed(SEED)
        threads = torch.get_num_threads()
        torch.set_num_threads(1)   # as torchrun starts its ranks: HuBERT's weight-norm fold follows the thread count
        try:
            return P.main([])
        finally:
            torch.set_num_threads(threads)
    assert _in(one, seeded) == 0
    got, want = _files(two, ["data_svc"]), _files(one, ["data_svc"])
    assert len([k for k in want if k.endswith(".spk.npy")]) == len(CLIPS) + 3   # and one average per speaker
    _same(got, want, shape_only=os.path.join("data_svc", "pitch"))
    for name in ("train.txt", "valid.txt"):
        assert (two / "files" / name).exists()
    entries = [sorted(ln for n in ("train.txt", "valid.txt") for ln in (r / "files" / n).read_text().splitlines())
               for r in (two, one)]
    assert entries[0] == entries[1] and len(entries[0]) == len(CLIPS)


def test_missing_model_file_fails_both_ranks(tmp_path, models):
    root = _tree(tmp_path / "nowhisper", models)
    os.remove(root / "whisper_pretrain" / "large-v2.pt")
    status, out, err = _torchrun(root, "preprocess_ppg.py", ["-w", "dataset_raw", "-p", "ppg"])
    assert status == [1, 1], out[-3000:] + err[-3000:]
    assert err.count("Traceback") >= 2 and "large-v2.pt" in err   # each rank's, and the launcher's summary
