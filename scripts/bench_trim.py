#!/usr/bin/env python
"""Trimming silence out of raw recordings (svcb_trim_silence_ragged, preprocess_trim.py) on 512 seeded clips of 2 to
28 s at 48 kHz with speech-like bursts and silences.  Prints one JSON line: the card and its power limit (read in the
same run), then
  device   the kernel time of the CLI's plan (CUDA events around --reps passes over every batch's svcb call, after a
           warm-up pass), per pass, and the achieved bytes / s against the HBM bound (data sheet, H100 SXM at 700 W:
           3.35 TB/s).  Bytes are 2 read per sample and 1 written per window;
  cli      preprocess_trim.py end to end on a temporary dataset (wall clock), and the same work split into phases run
           one after another in this process: read (trim.load on -t threads), device (trim_batch per batch: copies and
           kernel, synchronised), rules (trim.trim per file: ranges and slicing on the host) and write (trim.write_wav);
  cpu      the oracle's pydub loop (AudioSegment.from_wav, split_on_silence with one 200 ms slice and rms per ms, the
           join and export, as trim_silence runs them) per file on -t threads over a subset of the files, scaled to the
           whole set by samples, and whether its files equal the CLI's;
  numpy    the same flags on the host as one int64 cumulative sum per clip (oracle numpy_flags), then trim.trim, on -t
           threads over every file, against the device phase plus the rules phase, and whether all flags equal the
           device's.

    python scripts/bench_trim.py [-t 8] [--batch 64] [--cpu-files 48] [--reps 20]"""
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

N_CLIPS, SPEAKERS, SR = 512, 4, 48000
HBM_BPS = 3.35e12


def clips(seed=0):
    """512 int16 clips of 2 to 28 s at 48 kHz: voiced bursts of 80-900 ms (a gliding partial pair and noise under
    20 ms ramps, peaks of 1,000-12,000) between pauses of 40-1,200 ms of room noise at RMS 5-120, with leading and
    trailing pauses."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(N_CLIPS):
        n = int(rng.uniform(2, 28) * SR)
        x = np.empty(n, np.float32)
        p, voiced = 0, False
        while p < n:
            m = min(n - p, int(SR * (rng.uniform(0.08, 0.9) if voiced else rng.uniform(0.04, 1.2))))
            if voiced:
                t = np.arange(m, dtype=np.float32) / SR
                ph = 2 * np.pi * rng.uniform(90, 350) * (t + 0.1 * t * t)
                seg = np.sin(ph) + 0.5 * np.sin(2 * ph + 1.0) + 0.3 * rng.standard_normal(m, dtype=np.float32)
                r = min(m // 2, SR // 50)
                if r:
                    ramp = (0.5 - 0.5 * np.cos(np.pi * np.arange(r) / r)).astype(np.float32)
                    seg[:r] *= ramp
                    seg[m - r:] *= ramp[::-1]
                x[p:p + m] = rng.uniform(1000, 12000) / 1.8 * seg
            else:
                x[p:p + m] = rng.uniform(5, 120) * rng.standard_normal(m, dtype=np.float32)
            p, voiced = p + m, not voiced
        out.append(np.clip(np.rint(x), -32768, 32767).astype(np.int16))
    return out


def device_arm(data, plan, reps):
    """Kernel time of every batch of the plan, one svcb_trim_silence_ragged call each, over reps passes."""
    from ctypes import c_int32
    from whisper_vits_svc_b200 import _lib, trim
    calls, n_in, n_win = [], 0, 0
    for g in plan:
        lin = [data[i].shape[0] for i in g]
        win = sum(trim.windows(n, SR) for n in lin)
        x = torch.from_numpy(np.concatenate([data[i] for i in g])).cuda()
        out = torch.empty(max(win, 1), dtype=torch.uint8, device="cuda")
        calls.append((x, _lib.offsets(lin), (c_int32 * len(g))(*([SR] * len(g))), len(g), out))
        n_in, n_win = n_in + sum(lin), n_win + win

    def run(c):
        x, so, rates, b, out = c
        _lib.call("trim_silence_ragged", x.data_ptr(), so, rates, b, out.data_ptr())

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
    nbytes = 2.0 * n_in + n_win
    t_bytes = nbytes / HBM_BPS
    return dict(device_calls=len(calls), reps=reps, ms_per_pass=round(ms, 3), samples=n_in, windows=n_win,
                gb_per_s=round(nbytes / (ms / 1e3) / 1e9, 1), bound="bytes", bound_ms=round(1e3 * t_bytes, 3),
                share_of_bound=round(t_bytes / (ms / 1e3), 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("-t", "--threads", type=int, default=8)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--cpu-files", type=int, default=48)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_trim needs a CUDA device (an H100)")
    from bench_retrieval import gpu_info
    from oracle import trim_oracle as TO
    from whisper_vits_svc_b200 import dataset, trim
    import preprocess_trim as CLI
    name, power = gpu_info()
    data = clips()
    audio_s = sum(x.shape[0] for x in data) / SR
    plan = dataset.plan_window([x.shape[0] for x in data], args.batch, CLI.MAX_PADDED)
    dev = device_arm(data, plan, args.reps)
    torch.cuda.empty_cache()
    with tempfile.TemporaryDirectory() as tmp:
        for i, x in enumerate(data):
            d = os.path.join(tmp, "raw", f"spk{i % SPEAKERS}")
            os.makedirs(d, exist_ok=True)
            trim.write_wav(os.path.join(d, f"{i:03d}.wav"), x, SR)
        t0 = time.perf_counter()
        r = subprocess.run([sys.executable, os.path.join(ROOT, "preprocess_trim.py"), "-i", "raw", "-o", "trim", "-t",
                            str(args.threads), "--batch", str(args.batch)], cwd=tmp, capture_output=True, text=True)
        cli_s = time.perf_counter() - t0
        if r.returncode != 0 or "failed" in r.stderr:
            raise SystemExit(r.stderr[-3000:])
        cwd = os.getcwd()
        os.chdir(tmp)   # the reference's walk takes paths relative to the working directory
        jobs = [(os.path.join(tmp, w), os.path.join(tmp, p)) for w, p in CLI.trim_jobs("raw", "trim-phases")]
        os.chdir(cwd)
        t0 = time.perf_counter()
        with ThreadPoolExecutor(args.threads) as pool:
            loaded = list(pool.map(lambda j: trim.load(j[0]), jobs))
        t1 = time.perf_counter()
        flags = [None] * len(jobs)
        for g in dataset.plan_window([x.shape[0] for x, _ in loaded], args.batch, CLI.MAX_PADDED):
            for i, f in zip(g, trim.trim_batch([loaded[i][0] for i in g], [loaded[i][1] for i in g])):
                flags[i] = f
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        pcm = [trim.trim(x, rate, f) for (x, rate), f in zip(loaded, flags)]
        t3 = time.perf_counter()
        for (_, p), y, (_, rate) in zip(jobs, pcm, loaded):
            if y is not None:
                trim.write_wav(p, y, rate)
        t4 = time.perf_counter()
        written = [p for _, p in jobs if os.path.exists(p)]
        same = all(open(p, "rb").read() == open(p.replace("trim-phases", "trim"), "rb").read() for p in written[::29])
        kept = sum(y.shape[0] for y in pcm if y is not None)
        cli = dict(end_to_end_s=round(cli_s, 2), files_per_s=round(N_CLIPS / cli_s, 1),
                   audio_s_per_s=round(audio_s / cli_s), files_written=len(written), kept_share=round(kept / sum(
                       x.shape[0] for x in data), 3),
                   phases_s=dict(read=round(t1 - t0, 2), device=round(t2 - t1, 2), rules=round(t3 - t2, 2),
                                 write=round(t4 - t3, 2)), phase_files_equal_cli=same)
        # numpy arm: the flags from one int64 cumulative sum per clip, then the same rules, over every file
        t0 = time.perf_counter()
        with ThreadPoolExecutor(args.threads) as pool:
            host = list(pool.map(lambda xr: _numpy_arm(TO, trim, *xr), loaded))
        np_s = time.perf_counter() - t0
        flags_equal = all(np.array_equal(f, h[0]) for f, h in zip(flags, host))
        pcm_equal = all((y is None and h[1] is None) or (y is not None and h[1] is not None and np.array_equal(y, h[1]))
                        for y, h in zip(pcm, host))
        numpy_arm = dict(kind=f"int64 cumsum flags + trim.trim per file, {args.threads} threads", seconds=round(np_s, 2),
                         device_plus_rules_s=round(t3 - t1, 2), flags_equal_device=flags_equal,
                         samples_equal_device=pcm_equal)
        del host
        # CPU arm: the oracle's pydub loop per file on a subset, its files against the CLI's
        sub = jobs[:: max(1, len(jobs) // args.cpu_files)][:args.cpu_files]
        idx = [jobs.index(j) for j in sub]
        sub_samples = sum(data[i].shape[0] for i in idx)
        os.makedirs(os.path.join(tmp, "oracle"), exist_ok=True)
        dsts = [os.path.join(tmp, "oracle", f"{k}.wav") for k in range(len(sub))]
        t0 = time.perf_counter()
        with ThreadPoolExecutor(args.threads) as pool:
            res = list(pool.map(lambda jd: TO.trim_silence(jd[0][0], jd[1]), zip(sub, dsts)))
        cpu_sub = time.perf_counter() - t0
        equal = all((not r and not os.path.exists(j[1].replace("trim-phases", "trim"))) or
                    (r and open(d, "rb").read() == open(j[1].replace("trim-phases", "trim"), "rb").read())
                    for r, j, d in zip(res, sub, dsts))
        cpu = dict(kind=f"oracle pydub loop (slice + rms per ms) per file, {args.threads} threads", files=len(sub),
                   seconds=round(cpu_sub, 2), scaled_to_all_s=round(cpu_sub * sum(x.shape[0] for x in data) / sub_samples, 1),
                   files_equal_cli=equal)
    print(json.dumps(dict(metric="trim", gpu=name, power_limit_w=power, clips=N_CLIPS, batches=len(plan),
                          audio_s=round(audio_s, 1), device=dev, cli=cli, numpy=numpy_arm, cpu=cpu)))


def _numpy_arm(TO, trim, x, rate):
    f = TO.numpy_flags(x, rate)
    return f, trim.trim(x, rate, f)


if __name__ == "__main__":
    main()
