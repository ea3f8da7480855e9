#!/usr/bin/env python
"""Salience-based F0 (svcb_salience_f0_ragged, preprocess_f0_salience.py) on 512 seeded clips of 2 to 28 s at 16 kHz:
the clips of scripts/bench_f0.py (harmonic tones gliding across 80-800 Hz in voiced runs of 0.1-1.5 s, between pauses
of low room noise).  Prints one JSON line: the card and its power limit (read in the same run), then
  device   the kernel time of the CLI's plan per pass (CUDA events around --reps passes over every batch's svcb call,
           after a warm-up pass) and, from the library's per-kernel timing of one pass, each phase's time: stft (the
           direct DFT of bins 0-231; its share is of the data sheet's fp64 CUDA-core FMA bound, 34 TFLOP/s on an H100
           SXM at 700 W), bin (instantaneous frequency, binning and smoothing), harm (threshold and harmonic
           summation) and dp (the max-plus recursion: 636 x 636 additions and comparisons per frame);
  cli      preprocess_f0_salience.py end to end on a temporary dataset (wall clock), and the same work split into phases
           run one after another in this process: read (load_audio on -t threads), device (F0 per batch: copies,
           kernels and the host's repeat and average, synchronised) and write (np.save);
  cpu      the float32 oracle with the DP as the reference runs it (a scan over every predecessor, compiled by numba
           once per worker and warmed up) per file on -t processes over --cpu-files files: the per-file work alone
           (no pool start-up, imports or compiles), summed, scaled to the whole set by frames and divided by the
           processes, and the share of their frames on the device's bin.

    python scripts/bench_salience_f0.py [-t 8] [--batch 64] [--cpu-files 16] [--reps 3]"""
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


def parse_timing(report):
    """name -> (ms, flops) of svcb_timing_report()'s lines "name launches total_ms flops bytes"."""
    out = {}
    for line in report.decode().splitlines():
        f = line.split()
        if len(f) >= 4 and f[0].startswith("salience_"):
            out[f[0]] = (float(f[2]), float(f[3]))
    return out


def device_arm(data, plan, reps):
    from whisper_vits_svc_b200 import _lib, salience_f0
    lib = _lib.load()
    calls, n_in, n_fr = [], 0, 0
    ws_need = 0
    for g in plan:
        lin = [data[i].shape[0] for i in g]
        x = torch.from_numpy(np.concatenate([data[i] for i in g]).astype(np.float32)).cuda()
        fr = sum(salience_f0.frames_of(n) for n in lin)
        out = torch.empty(fr, dtype=torch.float64, device="cuda")
        calls.append((x, _lib.offsets(lin), len(g), out))
        ws_need = max(ws_need, lib.svcb_salience_f0_workspace_bytes(sum(lin), len(g)))
        n_in, n_fr = n_in + sum(lin), n_fr + fr
    ws = torch.empty(ws_need, dtype=torch.uint8, device="cuda")

    def run(c):
        x, so, b, out = c
        _lib.call("salience_f0_ragged", x.data_ptr(), so, b, out.data_ptr(), None, None, None, ws.data_ptr(), ws.numel())

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
        ph[k] = dict(ms=round(t, 3))
        if k == "salience_stft":
            ph[k].update(tflops=round(fl / (t / 1e3) / 1e12, 2),
                         share_of_fp64_cuda_core_bound=round(fl / FP64_CUDA_CORE_FLOPS / (t / 1e3), 3))
        if k == "salience_dp":
            ph[k].update(gadds_per_s=round(fl / 2 / (t / 1e3) / 1e9, 1))
    del calls, ws
    torch.cuda.empty_cache()
    return dict(device_calls=len(plan), reps=reps, ms_per_pass=round(ms, 2), samples=n_in, frames=n_fr, phases=ph)


def _dp_loops(Zl, tl):
    """The max-plus DP as the reference runs it: per frame and bin, a scan over every predecessor."""
    B, F = Zl.shape
    D = Zl[:, 0].copy()
    E = np.zeros((F, B), np.int64)
    for n in range(1, F):
        Dn = np.empty(B)
        for b in range(B):
            best, arg = -np.inf, 0
            for q in range(B):
                s = tl[b, q] + D[q]
                if s > best:
                    best, arg = s, q
            Dn[b] = best + Zl[b, n]
            E[n - 1, b] = arg
        D = Dn
    eta = np.zeros(F, np.int64)
    eta[F - 1] = np.argmax(D)
    for n in range(F - 2, -1, -1):
        eta[n] = E[n, eta[n + 1]]
    return eta


_DP = None


def _cpu_init():
    """Per worker: compile the DP with numba once and run it on a tiny input, so no file pays for the compile."""
    global _DP
    from oracle import salience_oracle as O
    try:
        import numba
        _DP = numba.njit(cache=False)(_dp_loops)
        _DP(np.zeros((O.B, 2)), O.transition_log())
    except ImportError:
        _DP = None


def _cpu_file(x):
    """The float32 oracle's salience and path of one file and the seconds that work took in this worker."""
    from oracle import salience_oracle as O
    t0 = time.perf_counter()
    with np.errstate(all="ignore"):
        Z = O.salience_rep(x, np.float32)
    eta = _DP(np.log(Z + O.EPS32), O.transition_log()) if _DP is not None else O.dp(Z)
    return eta, "numba" if _DP is not None else "numpy", time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("-t", "--threads", type=int, default=8)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--cpu-files", type=int, default=16)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_salience_f0 needs a CUDA device (an H100)")
    from bench_f0 import clips
    from bench_retrieval import gpu_info
    from scipy.io import wavfile
    from whisper_vits_svc_b200 import dataset, hubert_infer, salience_f0
    import preprocess_f0_salience as CLI
    name, power = gpu_info()
    data = [x.astype(np.float32) for x in clips()]
    audio_s = sum(x.shape[0] for x in data) / SR
    plan = dataset.plan_window([x.shape[0] for x in data], args.batch, CLI.MAX_PADDED)
    dev = device_arm(data, plan, args.reps)
    with tempfile.TemporaryDirectory() as tmp:
        for i, x in enumerate(data):
            d = os.path.join(tmp, "wav", f"spk{i % SPEAKERS}")
            os.makedirs(d, exist_ok=True)
            wavfile.write(os.path.join(d, f"{i:03d}.wav"), SR, np.rint(x * 32768).astype(np.int16))
        t0 = time.perf_counter()
        r = subprocess.run([sys.executable, os.path.join(ROOT, "preprocess_f0_salience.py"), "-w", "wav", "-p", "pit",
                            "-t", str(args.threads), "--batch", str(args.batch)], cwd=tmp, capture_output=True, text=True)
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
        ex = salience_f0.Extractor("cuda")
        for g in dataset.plan_window([x.shape[0] for x in loaded], args.batch, CLI.MAX_PADDED):
            for i, f in zip(g, ex.f0_batch([loaded[i] for i in g])):
                f0[i] = f
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        for (_, p), f in zip(jobs, f0):
            np.save(p, f, allow_pickle=False)
        t3 = time.perf_counter()
        same = all(np.array_equal(np.load(p + ".npy"), np.load(p.replace("pit-phases", "pit") + ".npy"))
                   for _, p in jobs[::17])
        cli = dict(end_to_end_s=round(cli_s, 2), files_per_s=round(N_CLIPS / cli_s, 1),
                   audio_s_per_s=round(audio_s / cli_s),
                   phases_s=dict(read=round(t1 - t0, 2), device=round(t2 - t1, 2), write=round(t3 - t2, 2)),
                   phase_files_equal_cli=same)
        sub = list(range(0, len(loaded), max(1, len(loaded) // args.cpu_files)))[:args.cpu_files]
        with ProcessPoolExecutor(args.threads, initializer=_cpu_init) as pool:
            res = list(pool.map(_cpu_file, [loaded[i] for i in sub]))
        cpu_sub = sum(r_[2] for r_ in res)   # per-file work only: no pool start-up, imports or compiles
        paths = ex.raw([loaded[i] for i in sub], taps=True)
        ex.close()
        agree = [np.mean(r_[0] == p[3].cpu().numpy()) for r_, p in zip(res, paths)]
        sub_frames = sum(salience_f0.frames_of(loaded[i].shape[0]) for i in sub)
        all_frames = sum(salience_f0.frames_of(x.shape[0]) for x in loaded)
        cpu = dict(kind=f"float32 oracle + {res[0][1]} DP per file", files=len(sub), processes=args.threads,
                   work_s=round(cpu_sub, 2), scaled_to_all_cpu_s=round(cpu_sub * all_frames / sub_frames, 1),
                   scaled_to_all_s_on_processes=round(cpu_sub * all_frames / sub_frames / args.threads, 1),
                   same_bin_as_device=round(float(np.mean(agree)), 4), worst_file_same_bin=round(float(min(agree)), 4))
    print(json.dumps(dict(metric="salience_f0", gpu=name, power_limit_w=power, clips=N_CLIPS, batches=len(plan),
                          audio_s=round(audio_s, 1), device=dev, cli=cli, cpu=cpu)))


if __name__ == "__main__":
    main()
