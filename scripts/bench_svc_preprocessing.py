#!/usr/bin/env python
"""Data preparation end to end: the ten steps of svc_preprocessing.py as ten processes of the individual CLIs (the
reference's structure) against one svc_preprocessing.py process, on the same tree.

A seeded synthetic `dataset_raw` of --files clips of 2 to 28 s at 44.1 and 48 kHz in four speaker directories, and
full-size seeded weights for the five models (Whisper large-v2 geometry with 24 kept layers, HuBERT-Soft, the LSTM
speaker encoder, CREPE full), as bench_preprocess.py and bench_crepe.py make them.  One untimed warm-up process comes
first, so that the first torch import on a fresh machine is charged to neither arm; then the arms alternate, --reps
times each, each run on a fresh `data_svc/`.

Every process is the CLI or svc_preprocessing.py run as `__main__` by a two-line wrapper that records
torch.cuda.max_memory_allocated at exit.  A step of the ten-process arm is the wall time of its process; in the
one-process arm a step runs from its `Command:` line to the next one (the first is preceded by the process start-up,
reported apart).  The outputs of the two arms are compared: byte-equal, except the pitch files (CREPE's noise and
dither are unseeded, so shape and dtype only) and the two lists (the shuffle is unseeded, so the set of lines).  The
card name, power limit and max SM clock are read in the same run.  Prints one JSON line.

    python scripts/bench_svc_preprocessing.py [--files 512] [--reps 2]"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

RATES = (44100, 48000)
# runs a script as __main__ and writes the process's peak device memory to $PEAK_OUT at exit
WRAPPER = ("import atexit, runpy, sys, torch\n"
           "atexit.register(lambda: open(__import__('os').environ['PEAK_OUT'], 'w').write("
           "str(torch.cuda.max_memory_allocated() if torch.cuda.is_initialized() else 0)))\n"
           "sys.argv = sys.argv[1:]\n"
           "runpy.run_path(sys.argv[0], run_name='__main__')\n")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True, check=True).stdout.strip()
    name, pl, clk = [s.strip() for s in q.splitlines()[0].split(",")]
    return name, float(pl), int(clk)


def make_tree(d, files, seed):
    """dataset_raw/spk<k>/<i>.wav and the five model files at the reference's relative paths; seconds of audio."""
    from scipy.io import wavfile
    from tests.test_speaker_gpu import CONFIG
    from whisper_vits_svc_b200 import synth
    rng = np.random.default_rng(seed)
    total = 0.0
    for i in range(files):
        rate = RATES[i % 2]
        n = int(rng.uniform(2.0, 28.0) * rate)
        t = np.arange(n) / rate
        x = 0.3 * np.sin(2 * np.pi * (120.0 + 5 * (i % 40)) * t) + 0.05 * rng.standard_normal(n)
        spk = os.path.join(d, "dataset_raw", f"spk{i % 4}")
        os.makedirs(spk, exist_ok=True)
        wavfile.write(os.path.join(spk, f"{i:04d}.wav"), rate, (np.clip(x, -1, 1) * 32767).astype(np.int16))
        total += n / rate
    for rel, make in (("whisper_pretrain/large-v2.pt", lambda: synth.whisper_checkpoint(seed=7)),
                      ("hubert_pretrain/hubert-soft-0d54a1f4.pt", lambda: synth.hubert_checkpoint(7)),
                      ("speaker_pretrain/best_model.pth.tar", lambda: synth.speaker_checkpoint(7)),
                      ("crepe/assets/full.pth", lambda: synth.crepe_checkpoint(7, "full"))):
        os.makedirs(os.path.join(d, os.path.dirname(rel)), exist_ok=True)
        torch.save(make(), os.path.join(d, rel))
    with open(os.path.join(d, "speaker_pretrain", "config.json"), "w") as f:
        f.write(CONFIG)
    os.makedirs(os.path.join(d, "configs"))
    shutil.copy(os.path.join(ROOT, "configs", "base.yaml"), os.path.join(d, "configs"))
    return total


def clean(d):
    for top in ("data_svc", "files"):
        shutil.rmtree(os.path.join(d, top), ignore_errors=True)


def wrapped(d, script, args):
    """Run ROOT/script as __main__ in d -> (exit code, peak bytes, stdout lines with their arrival times, stderr)."""
    peak = os.path.join(d, "peak.txt")
    env = dict(os.environ, PEAK_OUT=peak)
    with tempfile.TemporaryFile("w+") as err:
        p = subprocess.Popen([sys.executable, "-c", WRAPPER, os.path.join(ROOT, script), *args], cwd=d, env=env,
                             stdout=subprocess.PIPE, stderr=err, text=True)
        lines = [(time.perf_counter(), ln) for ln in p.stdout]
        code = p.wait()
        err.seek(0)
        tail = err.read()[-3000:]
    with open(peak) as f:
        return code, int(f.read() or 0), lines, tail


def run_steps(d, steps):
    """The reference's structure: one process per step."""
    clean(d)
    times, peak = {}, 0
    for step in steps:
        script, *args = step.split()
        t0 = time.perf_counter()
        code, pk, _, err = wrapped(d, script, args)
        times[script if script not in times else script + " (2)"] = round(time.perf_counter() - t0, 2)
        if code:
            raise SystemExit(f"{step} failed ({code}):\n{err}")
        peak = max(peak, pk)
    return dict(steps=times, total_s=round(sum(times.values()), 2), peak_gib=round(peak / 2 ** 30, 2))


def run_one(d, steps):
    """One svc_preprocessing.py process; a step runs from its Command line to the next."""
    clean(d)
    t0 = time.perf_counter()
    code, peak, lines, err = wrapped(d, "svc_preprocessing.py", ["-t", "2"])
    t1 = time.perf_counter()
    if code:
        raise SystemExit(f"svc_preprocessing.py failed ({code}):\n{err}")
    marks = [t for t, ln in lines if ln.startswith("Command: ")] + [t1]
    assert len(marks) == len(steps) + 1
    times = {}
    for step, a, b in zip(steps, marks, marks[1:]):
        script = step.split()[0]
        times[script if script not in times else script + " (2)"] = round(b - a, 2)
    return dict(startup_s=round(marks[0] - t0, 2), steps=times, total_s=round(t1 - t0, 2),
                peak_gib=round(peak / 2 ** 30, 2))


def snapshot(d):
    out = {}
    for top in ("data_svc", "files"):
        for r, _, fs in os.walk(os.path.join(d, top)):
            for f in fs:
                p = os.path.join(r, f)
                out[os.path.relpath(p, d)] = p
    return out


def compare(a, b):
    """The paths whose outputs disagree between two runs (see the module docstring)."""
    bad = sorted(set(a) ^ set(b))
    lists = [k for k in a if k.startswith("files")]
    if sorted(ln for k in lists for ln in open(a[k]).read().splitlines()) != sorted(
            ln for k in lists if k in b for ln in open(b[k]).read().splitlines()):
        bad += lists
    for k in sorted(set(a) & set(b)):
        if k.startswith("files"):
            continue
        if k.startswith(os.path.join("data_svc", "pitch")):
            x, y = np.load(a[k]), np.load(b[k])
            same = x.dtype == y.dtype and x.shape == y.shape
        else:
            with open(a[k], "rb") as f, open(b[k], "rb") as g:
                same = f.read() == g.read()
        if not same:
            bad.append(k)
    return bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=512)
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_svc_preprocessing needs a CUDA device (an H100)")
    import svc_preprocessing
    name, power, clock = gpu_info()
    res = dict(metric="svc_preprocessing", gpu=name, power_limit_w=power, max_sm_clock_mhz=clock, files=args.files)
    with tempfile.TemporaryDirectory() as d:
        res["audio_s"] = round(make_tree(d, args.files, 2026), 1)
        subprocess.run([sys.executable, "-c", "import torch, whisper_vits_svc_b200; torch.zeros(1, device='cuda')"],
                       cwd=ROOT, check=True)   # warm-up, untimed
        runs = {"ten_processes": [], "one_process": []}
        outs = {}
        for _ in range(args.reps):
            for arm, fn in (("ten_processes", run_steps), ("one_process", run_one)):
                runs[arm].append(fn(d, svc_preprocessing.STEPS))
                print(json.dumps({arm: runs[arm][-1]}), file=sys.stderr, flush=True)
                keep = os.path.join(d, f"out_{arm}")
                shutil.rmtree(keep, ignore_errors=True)
                os.makedirs(keep)
                for top in ("data_svc", "files"):
                    shutil.move(os.path.join(d, top), os.path.join(keep, top))
                outs[arm] = snapshot(keep)
        res["runs"] = runs
        res["outputs_differ"] = compare(outs["ten_processes"], outs["one_process"])
        res["output_files"] = len(outs["one_process"])
        for arm, rs in runs.items():
            tot = [r["total_s"] for r in rs]
            res[f"{arm}_total_s"] = dict(min=min(tot), max=max(tot))
        res["speedup_min_over_min"] = round(res["ten_processes_total_s"]["min"] / res["one_process_total_s"]["min"], 3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
