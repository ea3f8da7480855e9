#!/usr/bin/env python
"""Praat autocorrelation F0 (svcb_praat_f0_ragged, preprocess_f0_mouth.py) on 512 seeded clips of 2 to 28 s at 16 kHz:
the clips of scripts/bench_f0.py (harmonic tones gliding across 80-800 Hz in voiced runs of 0.1-1.5 s, between pauses
of low room noise).  Prints one JSON line: the card and its power limit (read in the same run), then
  device   the kernel time of the CLI's plan per pass (CUDA events around --reps passes over every batch's svcb call,
           after a warm-up pass) and, from the library's per-kernel timing of one pass, each kernel family's time:
           peak (mean and global peak), frame (local mean, windowed frame, direct autocorrelation, candidates) and
           viterbi.  The frame kernel's share is of the fp64 FMA bounds of the data sheet (H100 SXM at 700 W): 34
           TFLOP/s on the CUDA cores and 67 TFLOP/s on the tensor cores; the other kernels' of the HBM bound (3.35 TB/s);
  cli      preprocess_f0_mouth.py end to end on a temporary dataset (wall clock), and the same work split into phases run
           one after another in this process: read (load_audio on -t threads), device (padded F0 per batch: copies
           and kernels, synchronised) and write (np.save);
  cpu      the numpy oracle per file on -t processes over --cpu-files files, scaled to the whole set by frames.

    python scripts/bench_praat_f0.py [-t 8] [--batch 64] [--cpu-files 16] [--reps 3]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ProcessPoolExecutor, ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

N_CLIPS, SPEAKERS, SR = 512, 4, 16000
FP64_CUDA_CORE_FLOPS = 34e12
FP64_TENSOR_FLOPS = 67e12
HBM_BPS = 3.35e12


def parse_timing(report):
    """name -> (ms, flops) of svcb_timing_report()'s lines "name launches total_ms flops bytes"."""
    out = {}
    for line in report.decode().splitlines():
        f = line.split()
        if len(f) >= 4 and f[0].startswith("praat_"):
            out[f[0]] = (float(f[2]), float(f[3]))
    return out


def device_arm(data, plan, reps):
    from whisper_vits_svc_b200 import _lib, praat_f0
    lib = _lib.load()
    calls, n_in, n_fr = [], 0, 0
    ws_need = 0
    for g in plan:
        lin = [data[i].shape[0] for i in g]
        x = torch.from_numpy(np.concatenate([data[i] for i in g]).astype(np.float64)).cuda()
        fr = sum(praat_f0.frames_of(n) for n in lin)
        out = torch.empty(fr, dtype=torch.float64, device="cuda")
        calls.append((x, _lib.offsets(lin), len(g), out))
        ws_need = max(ws_need, lib.svcb_praat_f0_workspace_bytes(sum(lin), len(g)))
        n_in, n_fr = n_in + sum(lin), n_fr + fr
    ws = torch.empty(ws_need, dtype=torch.uint8, device="cuda")

    def run(c):
        x, so, b, out = c
        _lib.call("praat_f0_ragged", x.data_ptr(), so, b, out.data_ptr(), ws.data_ptr(), ws.numel())

    for c in calls:
        run(c)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        for c in calls:
            run(c)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    lib.svcb_timing_enable(1)
    for c in calls:
        run(c)
    torch.cuda.synchronize()
    phases = parse_timing(lib.svcb_timing_report())
    lib.svcb_timing_enable(0)
    ph = {}
    for k, (t, fl) in phases.items():
        if k == "praat_frame":
            ph[k] = dict(ms=round(t, 3), tflops=round(fl / (t / 1e3) / 1e12, 2),
                         share_of_fp64_cuda_core_bound=round(fl / FP64_CUDA_CORE_FLOPS / (t / 1e3), 3),
                         share_of_fp64_tensor_bound=round(fl / FP64_TENSOR_FLOPS / (t / 1e3), 3))
        else:
            b = 8.0 * n_in if k == "praat_peak" else 8.0 * 31 * n_fr
            ph[k] = dict(ms=round(t, 3), share_of_hbm_bound=round(b / HBM_BPS / (t / 1e3), 3))
    del calls, ws
    torch.cuda.empty_cache()
    return dict(device_calls=len(plan), reps=reps, ms_per_pass=round(ms, 2), samples=n_in, frames=n_fr, phases=ph)


def _oracle_file(x):
    from oracle import praat_f0_oracle as O
    return O.praat_f0(x)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("-t", "--threads", type=int, default=8)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--cpu-files", type=int, default=16)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_praat_f0 needs a CUDA device (an H100)")
    from bench_f0 import clips
    from bench_retrieval import gpu_info
    from scipy.io import wavfile
    from whisper_vits_svc_b200 import dataset, hubert_infer, praat_f0
    import preprocess_f0_mouth as CLI
    name, power = gpu_info()
    data = clips()
    audio_s = sum(x.shape[0] for x in data) / SR
    plan = dataset.plan_window([x.shape[0] for x in data], args.batch, CLI.MAX_PADDED)
    dev = device_arm(data, plan, args.reps)
    with tempfile.TemporaryDirectory() as tmp:
        for i, x in enumerate(data):
            d = os.path.join(tmp, "wav", f"spk{i % SPEAKERS}")
            os.makedirs(d, exist_ok=True)
            wavfile.write(os.path.join(d, f"{i:03d}.wav"), SR, np.rint(x * 32768).astype(np.int16))
        t0 = time.perf_counter()
        r = subprocess.run([sys.executable, os.path.join(ROOT, "preprocess_f0_mouth.py"), "-w", "wav", "-p", "pit", "-t",
                            str(args.threads), "--batch", str(args.batch)], cwd=tmp, capture_output=True, text=True)
        cli_s = time.perf_counter() - t0
        if r.returncode != 0 or "failed" in r.stderr:
            raise SystemExit(r.stderr[-3000:])
        cwd = os.getcwd()
        os.chdir(tmp)
        jobs = [(os.path.join(tmp, w), os.path.join(tmp, p)) for w, p in CLI.pit_jobs("wav", "pit-phases")]
        os.chdir(cwd)
        t0 = time.perf_counter()
        with ThreadPoolExecutor(args.threads) as pool:
            loaded = list(pool.map(lambda j: hubert_infer.load_audio(j[0], SR), jobs))
        t1 = time.perf_counter()
        f0 = [None] * len(jobs)
        ex = praat_f0.Extractor("cuda")
        for g in dataset.plan_window([x.shape[0] for x in loaded], args.batch, CLI.MAX_PADDED):
            for i, f in zip(g, ex.f0_batch([loaded[i] for i in g])):
                f0[i] = f
        torch.cuda.synchronize()
        ex.close()
        t2 = time.perf_counter()
        for (_, p), f in zip(jobs, f0):
            np.save(p, f, allow_pickle=False)
        t3 = time.perf_counter()
        same = all(np.array_equal(np.load(p + ".npy"), np.load(p.replace("pit-phases", "pit") + ".npy"))
                   for _, p in jobs[::17])
        voiced = float(np.mean(np.concatenate(f0) > 0))
        cli = dict(end_to_end_s=round(cli_s, 2), files_per_s=round(N_CLIPS / cli_s, 1),
                   audio_s_per_s=round(audio_s / cli_s), voiced_share=round(voiced, 3),
                   phases_s=dict(read=round(t1 - t0, 2), device=round(t2 - t1, 2), write=round(t3 - t2, 2)),
                   phase_files_equal_cli=same)
        sub = list(range(0, len(loaded), max(1, len(loaded) // args.cpu_files)))[:args.cpu_files]
        t0 = time.perf_counter()
        with ProcessPoolExecutor(args.threads) as pool:
            res = list(pool.map(_oracle_file, [loaded[i] for i in sub]))
        cpu_sub = time.perf_counter() - t0
        vu_equal = all(np.array_equal(r_ > 0, f0[i] > 0) for r_, i in zip(res, sub))
        rel = [np.abs(r_ - f0[i])[r_ > 0] / r_[r_ > 0] for r_, i in zip(res, sub)]
        sub_frames = sum(f0[i].shape[0] for i in sub)
        cpu = dict(kind=f"numpy oracle per file, {args.threads} processes", files=len(sub), seconds=round(cpu_sub, 2),
                   scaled_to_all_s=round(cpu_sub * sum(f.shape[0] for f in f0) / sub_frames, 1),
                   voiced_unvoiced_equal_device=vu_equal,
                   max_rel_diff_voiced=float(max((float(v.max()) for v in rel if v.size), default=0.0)))
    print(json.dumps(dict(metric="praat_f0", gpu=name, power_limit_w=power, clips=N_CLIPS, batches=len(plan),
                          audio_s=round(audio_s, 1), device=dev, cli=cli, cpu=cpu)))


if __name__ == "__main__":
    main()
