#!/usr/bin/env python
"""Dataset feature preparation (preprocess_ppg.py, preprocess_hubert.py) on the device: ragged batches against one file
at a time.

A seeded synthetic dataset of --files clips with lengths drawn uniformly from 2 to 28 s, and full-size synthetic
checkpoints (Whisper large-v2 geometry with 24 kept layers, HuBERT-Soft with 12 layers).  For each encoder the
library calls the CLIs make (whisper_infer.ppg_batch, hubert_infer.units_batch) run over the whole dataset, in the
CLIs' batch plan and one file per call, alternated, after one warm pass of each (every shape is warmed); a pass is a
host clock around calls that end in a device synchronise, so it includes the host padding and the copies.  Then the
padding overhead of the plan, the per-kernel split from svcb_timing_report (a separate ragged pass), and the
end-to-end time of both CLIs on the same dataset written to disk as 16-bit wavs.  The card name, power limit and max
SM clock are read in the same run.  Prints one JSON line.

    python scripts/bench_preprocess.py [--files 512] [--reps 2] [--no-cli]"""
import argparse
import importlib.util
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

SR = 16000


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True, check=True).stdout.strip()
    name, pl, clk = [s.strip() for s in q.splitlines()[0].split(",")]
    return name, float(pl), int(clk)


def dataset(n, seed):
    rng = np.random.default_rng(seed)
    lens = rng.integers(2 * SR, 28 * SR + 1, n)
    out = []
    for i, m in enumerate(lens):
        t = np.arange(m) / SR
        x = 0.3 * np.sin(2 * np.pi * (120.0 + 5 * (i % 40)) * t) + 0.05 * rng.standard_normal(m)
        out.append(x.astype(np.float32))
    return out


def cli_module(name):
    spec = importlib.util.spec_from_file_location(name[:-3] + "_cli", os.path.join(ROOT, name))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def plan(audios, size, batch, max_padded):
    """The CLIs' plan: windows of 8 x batch files in dataset order, each sorted and cut by dataset.plan_window."""
    from whisper_vits_svc_b200 import dataset as D
    groups, padded, real = [], 0, 0
    w = 8 * batch
    for s in range(0, len(audios), w):
        sizes = [size(a) for a in audios[s:s + w]]
        for g in D.plan_window(sizes, batch, max_padded):
            groups.append([s + i for i in g])
            real += sum(sizes[i] for i in g)
            padded += len(g) * max(sizes[i] for i in g)
    return groups, padded / real


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def kernel_split(lib, fn):
    lib.svcb_timing_enable(1)
    fn()
    torch.cuda.synchronize()
    rep = lib.svcb_timing_report().decode()
    lib.svcb_timing_enable(0)
    ks = {}
    for line in rep.strip().splitlines():
        k, cnt, kms, fl, _by, *_ = line.split()
        ks[k] = dict(launches=int(cnt), ms=round(float(kms), 1),
                     tflops=round(float(fl) / (float(kms) * 1e-3) / 1e12, 1) if float(fl) > 0 else None)
    return dict(sorted(ks.items(), key=lambda kv: -kv[1]["ms"]))


def compare(lib, audios, run, groups, reps):
    """Ragged passes (the plan's groups) and one-file passes, alternated after one warm pass of each."""
    ragged = lambda: [run([audios[i] for i in g]) for g in groups]  # noqa: E731
    single = lambda: [run([a]) for a in audios]  # noqa: E731
    ragged(); single()
    t_r, t_s = [], []
    for _ in range(reps):
        t_r.append(timed(ragged))
        t_s.append(timed(single))
    audio_s = sum(a.shape[0] for a in audios) / SR

    def arm(ts):
        best = min(ts)
        return dict(seconds=[round(t, 3) for t in ts], files_per_s=round(len(audios) / best, 1),
                    audio_s_per_s=round(audio_s / best, 1))
    return dict(ragged=arm(t_r), one_file=arm(t_s), speedup=round(min(t_s) / min(t_r), 2),
                kernels_ragged=kernel_split(lib, ragged))


def run_clis(audios, ck_whisper, sd_hubert, threads):
    from scipy.io import wavfile
    out = {}
    with tempfile.TemporaryDirectory() as d:
        os.makedirs(os.path.join(d, "whisper_pretrain"))
        os.makedirs(os.path.join(d, "hubert_pretrain"))
        torch.save(ck_whisper, os.path.join(d, "whisper_pretrain", "large-v2.pt"))
        torch.save(sd_hubert, os.path.join(d, "hubert_pretrain", "hubert-soft-0d54a1f4.pt"))
        for i, a in enumerate(audios):
            spk = os.path.join(d, "wav", f"spk{i % 4}")
            os.makedirs(spk, exist_ok=True)
            wavfile.write(os.path.join(spk, f"{i:04d}.wav"), SR, (np.clip(a, -1, 1) * 32767).astype(np.int16))
        for script, flag, dst in (("preprocess_ppg.py", "-p", "whisper"), ("preprocess_hubert.py", "-v", "hubert")):
            t0 = time.perf_counter()
            r = subprocess.run([sys.executable, os.path.join(ROOT, script), "-w", "wav", flag, dst, "-t", str(threads)],
                               cwd=d, capture_output=True, text=True)
            dt = time.perf_counter() - t0
            if r.returncode != 0:
                raise SystemExit(r.stdout[-2000:] + r.stderr[-3000:])
            over = [ln for ln in r.stdout.splitlines() if ln.startswith("padding overhead")]
            out[script] = dict(seconds=round(dt, 1), files_per_s=round(len(audios) / dt, 1), padding=over[-1] if over else None)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=512)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--no-cli", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_preprocess needs a CUDA device (an H100)")
    from whisper_vits_svc_b200 import _lib, hubert_infer, synth, whisper_infer
    lib = _lib.load()
    name, power, clock = gpu_info()
    audios = dataset(args.files, 2026)
    ppg_cli, hub_cli = cli_module("preprocess_ppg.py"), cli_module("preprocess_hubert.py")
    res = dict(metric="dataset_preprocess", gpu=name, power_limit_w=power, max_sm_clock_mhz=clock, files=args.files,
               audio_s=round(sum(a.shape[0] for a in audios) / SR, 1))

    ck = synth.whisper_checkpoint(seed=7)
    wm = whisper_infer.WhisperB200(ck, "cuda")
    groups, pad = plan(audios, lambda a: min(max(a.shape[0], 240000), 480000), 32, ppg_cli.MAX_PADDED)
    res["whisper"] = dict(padding_overhead=round(pad, 3), batches=len(groups),
                          **compare(lib, audios, lambda a: whisper_infer.ppg_batch(wm, a), groups, args.reps))
    del wm
    torch.cuda.empty_cache()

    sd = synth.hubert_checkpoint(7)
    hm = hubert_infer.HubertSoftB200(sd, "cuda")
    groups, pad = plan(audios, lambda a: a.shape[0], 32, hub_cli.MAX_PADDED)
    res["hubert"] = dict(padding_overhead=round(pad, 3), batches=len(groups),
                         **compare(lib, audios, lambda a: hubert_infer.units_batch(hm, a), groups, args.reps))
    del hm
    torch.cuda.empty_cache()

    print(json.dumps(res), file=sys.stderr, flush=True)   # the library numbers, before the slower CLI runs
    if not args.no_cli:
        res["cli"] = run_clis(audios, ck, sd, args.threads)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
