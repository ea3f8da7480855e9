#!/usr/bin/env python
"""Data preparation at 1 rank and at --ranks ranks under torchrun: svc_preprocessing.py end to end, and two single
CLIs (preprocess_ppg.py, bound by the device, and preprocess_spec.py, bound by host file I/O) on the waves it wrote.

The tree is bench_svc_preprocessing.py's: --files seeded synthetic clips of 2 to 28 s at 44.1 and 48 kHz in four
speaker directories, and full-size seeded weights for the five models.  One untimed warm-up process comes first, then
the two arms alternate, --reps times each, each on a fresh `data_svc/`.  The 1-rank arm is the plain command; the
N-rank arm is `python -m torch.distributed.run --standalone --nproc-per-node N` of it.  Ranks take
cuda:(LOCAL_RANK % device count): with fewer visible GPUs than ranks, several ranks share a card, and the result says
how many GPUs were used.  A step of svc_preprocessing.py runs from rank 0's `Command:` line to the next, which rank 0
prints once every rank has finished the step; a single CLI is the wall time of its command, start-up included.
The N-rank outputs are compared with the 1-rank ones as bench_svc_preprocessing.py compares its arms.  The card
name, power limit and max SM clock are read in the same run.  Prints a DESIGN.md table, a README line and, last, one
JSON line.

    python scripts/bench_prep_shard.py [--files 512] [--ranks 2] [--reps 2]"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import torch  # noqa: E402

import bench_svc_preprocessing as B  # noqa: E402

# one host thread per process in both arms, as torchrun starts its ranks: HuBERT's weight-norm fold at load is a host
# reduction whose order follows the thread count, and the arms' outputs are compared byte for byte
ENV = dict(os.environ, OMP_NUM_THREADS=os.environ.get("OMP_NUM_THREADS", "1"))
TIMEOUT = 1800   # seconds any one command may take before it is stopped (SIGTERM, which torchrun passes to its ranks)
CLIS = (("preprocess_ppg.py", ["-w", "data_svc/waves-16k/", "-p", "bench_ppg"], "bench_ppg"),
        ("preprocess_spec.py", ["-w", "data_svc/waves-32k/", "-s", "bench_specs"], "bench_specs"))


def command(ranks, script, args):
    if ranks == 1:
        return [sys.executable, os.path.join(ROOT, script), *args]
    return [sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc-per-node", str(ranks),
            os.path.join(ROOT, script), *args]


def timed(d, cmd):
    """Run cmd in d -> (its stdout lines with their arrival times, start time, end time), perf_counter seconds.  A
    command that fails, or runs longer than TIMEOUT and is stopped, stops the benchmark."""
    with tempfile.TemporaryFile("w+") as err:
        t0 = time.perf_counter()
        p = subprocess.Popen(cmd, cwd=d, env=ENV, stdout=subprocess.PIPE, stderr=err, text=True)
        stop = threading.Timer(TIMEOUT, p.terminate)
        stop.start()
        try:
            lines = [(time.perf_counter(), ln) for ln in p.stdout]
            code = p.wait()
        finally:
            stop.cancel()
        t1 = time.perf_counter()
        if code:
            err.seek(0)
            raise SystemExit(f"{' '.join(cmd)} failed ({code}):\n{err.read()[-3000:]}")
    return lines, t0, t1


def label(step):
    """A step's row in the table: its script, the rate for the two resampling steps, and "(rank 0)" for the steps
    that rank 0 runs alone."""
    import svc_preprocessing
    script, *argv = step.split()
    if script == "preprocess_a.py":
        return f"{script} {int(argv[argv.index('-s') + 1]) // 1000} kHz"
    return f"{script} (rank 0)" if script in svc_preprocessing.HOST_STEPS else script


def run_arm(d, ranks, steps):
    """svc_preprocessing.py, then each CLI of CLIS on its waves, on a fresh tree."""
    B.clean(d)
    lines, t0, t1 = timed(d, command(ranks, "svc_preprocessing.py", ["-t", "2"]))
    marks = [t for t, ln in lines if ln.startswith("Command: ")] + [t1]
    assert len(marks) == len(steps) + 1, len(marks)
    times = {label(step): round(b - a, 2) for step, a, b in zip(steps, marks, marks[1:])}
    res = dict(startup_s=round(marks[0] - t0, 2), steps=times, total_s=round(t1 - t0, 2), clis={})
    for script, args, out in CLIS:
        shutil.rmtree(os.path.join(d, out), ignore_errors=True)
        _, a, b = timed(d, command(ranks, script, args))
        res["clis"][script] = round(b - a, 2)
    return res


def outputs(d):
    snap = B.snapshot(d)
    for _, _, out in CLIS:
        for r, _, fs in os.walk(os.path.join(d, out)):
            for f in fs:
                p = os.path.join(r, f)
                snap[os.path.relpath(p, d)] = p
    return snap


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=512)
    ap.add_argument("--ranks", type=int, default=2)
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_prep_shard needs a CUDA device (an H100)")
    import svc_preprocessing
    name, power, clock = B.gpu_info()
    gpus = min(args.ranks, torch.cuda.device_count())
    res = dict(metric="prep_shard", gpu=name, power_limit_w=power, max_sm_clock_mhz=clock, files=args.files,
               ranks=args.ranks, gpus_used=gpus)
    arms = {"1_rank": 1, f"{args.ranks}_ranks": args.ranks}
    with tempfile.TemporaryDirectory() as d:
        res["audio_s"] = round(B.make_tree(d, args.files, 2026), 1)
        subprocess.run([sys.executable, "-c", "import torch, whisper_vits_svc_b200; torch.zeros(1, device='cuda')"],
                       cwd=ROOT, check=True)   # warm-up, untimed
        runs = {arm: [] for arm in arms}
        outs = {}
        for _ in range(args.reps):
            for arm, ranks in arms.items():
                runs[arm].append(run_arm(d, ranks, svc_preprocessing.STEPS))
                print(json.dumps({arm: runs[arm][-1]}), file=sys.stderr, flush=True)
                keep = os.path.join(d, f"out_{arm}")
                shutil.rmtree(keep, ignore_errors=True)
                os.makedirs(keep)
                for top in ("data_svc", "files") + tuple(out for _, _, out in CLIS):
                    shutil.move(os.path.join(d, top), os.path.join(keep, top))
                outs[arm] = outputs(keep)
        one, many = arms
        res["runs"] = runs
        res["outputs_differ"] = B.compare(outs[one], outs[many])
        res["output_files"] = len(outs[one])
    best = {arm: min(r["total_s"] for r in rs) for arm, rs in runs.items()}
    res["speedup_min_over_min"] = round(best[one] / best[many], 3)

    where = f"{args.ranks} ranks on {gpus} GPU{'s' if gpus > 1 else ''}"
    print(f"Measured on an {name} at a {power:.0f} W power limit, max SM clock {clock} MHz, {args.files} clips "
          f"({res['audio_s']:.0f} s of audio); seconds, wall clock, the {args.reps} runs of each arm:\n")
    print(f"| step | 1 rank | {where} |\n|---|---|---|")
    fmt = lambda arm, get: " / ".join(f"{get(r):.1f}" for r in runs[arm])   # noqa: E731
    print(f"| start-up before the first step | {fmt(one, lambda r: r['startup_s'])} | "
          f"{fmt(many, lambda r: r['startup_s'])} |")
    for step in runs[one][0]["steps"]:
        script, _, note = step.partition(" ")
        print(f"| `{script}`{' ' + note if note else ''} | {fmt(one, lambda r: r['steps'][step])} | "
              f"{fmt(many, lambda r: r['steps'][step])} |")
    print(f"| `svc_preprocessing.py` total | {fmt(one, lambda r: r['total_s'])} | "
          f"{fmt(many, lambda r: r['total_s'])} |")
    for script, _, _ in CLIS:
        print(f"| `{script}` alone, as a command | {fmt(one, lambda r: r['clis'][script])} | "
              f"{fmt(many, lambda r: r['clis'][script])} |")
    if gpus < args.ranks:
        print(f"| {args.ranks} ranks on {args.ranks} GPUs | | not measured |")
    if args.ranks < 8:
        print("| 8 ranks on 8 GPUs | | not measured |")
    print(f"\nREADME: `svc_preprocessing.py` on {args.files} clips: {best[one]:.1f} s at 1 rank, {best[many]:.1f} s at "
          f"{where} ({res['speedup_min_over_min']:.2f}x), {name}, {power:.0f} W.\n")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
