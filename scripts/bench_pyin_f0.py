#!/usr/bin/env python
"""pYIN F0 (svcb_pyin_f0_ragged, preprocess_f0_pyin.py) on 512 seeded clips of 2 to 28 s at 16 kHz: the clips of
scripts/bench_f0.py (harmonic tones gliding across 80-800 Hz in voiced runs of 0.1-1.5 s, between pauses of low room
noise).  Prints one JSON line: the card and its power limit (read in the same run), then
  device   the device calls of the CLI's plan with their host-to-device and device-to-host copies (CUDA events around
           --reps passes over every batch, after a warm-up pass) and, from the library's per-kernel timing of one pass,
           each phase's kernel time: cmndf (the direct difference function: 3 fp64 operations per term, its share of
           the data sheet's fp64 CUDA-core bound, 34 TFLOP/s on an H100 SXM at 700 W), thresh (minima, thresholds,
           observations), viterbi (one CTA per item over its frames) and tail (conf and refinement);
  cli      preprocess_f0_pyin.py -t THREADS end to end on a temporary dataset (wall clock), and the same work split into
           phases run one after another in this process: read (load_audio on -t threads), device (F0 per batch,
           synchronised) and write (np.save);
  cpu      the reference's work per file over --cpu-files files on -t processes, as the reference runs it on a CPU: the
           CMNDF by explicit loops and the dense Viterbi as a scan over all 1036 predecessors per state and frame,
           both compiled with numba (once per worker, warmed up), the thresholding by the numpy oracle; the per-file
           work summed and scaled to the whole set by frames.  The reference's own functions are not run here.

    python scripts/bench_pyin_f0.py [-t 8] [--batch 64] [--cpu-files 16] [--reps 3]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

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
        if len(f) >= 4 and f[0].startswith("pyin_"):
            out[f[0]] = (float(f[2]), float(f[3]))
    return out


def device_arm(data, plan, reps):
    from whisper_vits_svc_b200 import _lib, pyin_f0
    lib = _lib.load()
    ex = pyin_f0.Extractor("cuda")
    batches = [[data[i] for i in g] for g in plan]

    def run():
        for b in batches:
            for f, c in ex.raw(b):
                f.cpu(), c.cpu()

    run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        run()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    lib.svcb_timing_enable(1)
    run()
    torch.cuda.synchronize()
    phases = parse_timing(lib.svcb_timing_report())
    lib.svcb_timing_enable(0)
    ex.close()
    ph = {}
    for k, (t, fl) in phases.items():
        ph[k] = dict(ms=round(t, 3))
        if k == "pyin_cmndf":
            ph[k].update(tflops=round(fl / (t / 1e3) / 1e12, 2),
                         share_of_fp64_cuda_core_bound=round(fl / FP64_CUDA_CORE_FLOPS / (t / 1e3), 3))
    torch.cuda.empty_cache()
    frames = sum(pyin_f0.frames_of(x.shape[0]) for x in data)
    return dict(device_calls=len(plan), reps=reps, ms_per_pass_with_copies=round(ms, 2), frames=frames,
                kernel_ms=round(sum(v["ms"] for v in ph.values()), 2), phases=ph)


def _cmndf_frames(fr, lags):
    """[M, lags] CMNDF of the frames by explicit loops: each lag's squared differences added sample by sample, the
    running mean of the differences so far, and their ratio (the work of the reference's per-frame CMNDF)."""
    M, n = fr.shape
    out = np.empty((M, lags))
    for m in range(M):
        out[m, 0] = 1.0
        mean = 0.0
        for tau in range(1, lags):
            acc = 0.0
            for j in range(n - tau):
                e = fr[m, j] - fr[m, j + tau]
                acc += e * e
            mean = mean * (tau - 1) / tau + acc / tau
            out[m, tau] = acc / (mean + 2.220446049250313e-16)
    return out


def _dense_scan(at, ol, init):
    """The HMM path by the dense recursion the reference runs: for every frame and state a scan over all predecessors
    (at[j, k] the log transition k -> j), the first index of the largest sum; then the trace back."""
    S, F = ol.shape
    d = init + ol[:, 0]
    bp = np.zeros((F, S), np.int32)
    for n in range(1, F):
        dn = np.empty(S)
        for j in range(S):
            best, arg = -np.inf, 0
            for k in range(S):
                v = at[j, k] + d[k]
                if v > best:
                    best, arg = v, k
            dn[j] = best + ol[j, n]
            bp[n - 1, j] = arg
        d = dn
    path = np.zeros(F, np.int32)
    path[F - 1] = np.argmax(d)
    for n in range(F - 2, -1, -1):
        path[n] = bp[n, path[n + 1]]
    return path


_CPU = None


def _cpu_init():
    """Per worker: compile the two loops with numba once and run them on tiny inputs, so no file pays for a compile."""
    global _CPU
    import numba
    from oracle import pyin_oracle as O
    cm, scan = numba.njit(_cmndf_frames), numba.njit(_dense_scan)
    at = np.ascontiguousarray(np.log(O.transition_matrix() + O.TINY).T)
    cm(np.zeros((1, O.N)), O.LAGS)
    scan(at, np.zeros((O.S, 2)), O.log_init())
    _CPU = (cm, scan, at)


def _cpu_file(x):
    """(CMNDF, thresholding, Viterbi) seconds of one file in this worker."""
    from oracle import pyin_oracle as O
    cm, scan, at = _CPU
    thr, beta, fa = O.thresholds(), O.beta_distr(), O.f_axis()
    fr = O.frames(x)
    t0 = time.perf_counter()
    c = cm(fr, O.LAGS)
    t1 = time.perf_counter()
    Obs = np.zeros((O.S, fr.shape[0]))
    for m in range(fr.shape[0]):
        Obs[:, m] = O.threshold_frame(c[m], thr, beta, fa)[0]
    Obs[:O.B] *= 0.5
    Obs[O.B:] = 0.5 * (1 - Obs[:O.B].sum(0)) / O.B
    t2 = time.perf_counter()
    scan(at, np.log(Obs + O.TINY), O.log_init())
    return t1 - t0, t2 - t1, time.perf_counter() - t2


def cpu_arm(loaded, sub, processes):
    from concurrent.futures import ProcessPoolExecutor
    from oracle import pyin_oracle as O
    with ProcessPoolExecutor(processes, initializer=_cpu_init) as pool:
        res = list(pool.map(_cpu_file, [loaded[i] for i in sub]))
    t_cm, t_th, t_vit = (sum(r[j] for r in res) for j in range(3))
    scale = sum(O.n_frames(x.shape[0]) for x in loaded) / sum(O.n_frames(loaded[i].shape[0]) for i in sub)
    total = t_cm + t_th + t_vit   # per-file work only: no pool start-up, imports or compiles
    return dict(kind="numba-compiled loops doing the reference's CMNDF and dense Viterbi work, numpy thresholding, "
                     "one core per file",
                files=len(sub), work_s=round(total, 2), s_per_file=round(total / len(sub), 2),
                phases_s=dict(cmndf=round(t_cm, 2), thresh=round(t_th, 2), viterbi=round(t_vit, 2)),
                scaled_to_all_cpu_s=round(total * scale, 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("-t", "--threads", type=int, default=8)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--cpu-files", type=int, default=16)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pyin_f0 needs a CUDA device (an H100)")
    from bench_f0 import clips
    from bench_retrieval import gpu_info
    from scipy.io import wavfile
    from whisper_vits_svc_b200 import dataset, hubert_infer, pyin_f0
    import preprocess_f0_pyin as CLI
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
        r = subprocess.run([sys.executable, os.path.join(ROOT, "preprocess_f0_pyin.py"), "-w", "wav", "-p", "pit",
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
        ex = pyin_f0.Extractor("cuda")
        for g in dataset.plan_window([x.shape[0] for x in loaded], args.batch, CLI.MAX_PADDED):
            for i, f in zip(g, ex.f0_batch([loaded[i] for i in g])):
                f0[i] = f
        torch.cuda.synchronize()
        ex.close()
        t2 = time.perf_counter()
        for (_, p), f in zip(jobs, f0):
            os.makedirs(os.path.dirname(p), exist_ok=True)
            np.save(p, f, allow_pickle=False)
        t3 = time.perf_counter()
        same = all(np.array_equal(np.load(p + ".npy"), np.load(p.replace("pit-phases", "pit") + ".npy"))
                   for _, p in jobs[::17])
        cli = dict(end_to_end_s=round(cli_s, 2), files_per_s=round(N_CLIPS / cli_s, 1),
                   audio_s_per_s=round(audio_s / cli_s),
                   phases_s=dict(read=round(t1 - t0, 2), device=round(t2 - t1, 2), write=round(t3 - t2, 2)),
                   phase_files_equal_cli=same)
        sub = list(range(0, len(loaded), max(1, len(loaded) // args.cpu_files)))[:args.cpu_files]
        cpu = cpu_arm(loaded, sub, args.threads)
    print(json.dumps(dict(metric="pyin_f0", gpu=name, power_limit_w=power, clips=N_CLIPS, batches=len(plan),
                          audio_s=round(audio_s, 1), device=dev, cli=cli, cpu=cpu)))


if __name__ == "__main__":
    main()
