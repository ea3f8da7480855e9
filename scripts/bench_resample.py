#!/usr/bin/env python
"""Resampling of raw recordings (svcb_resample_ragged + svcb_pcm16_normalise_ragged, preprocess_a.py) on 512 seeded
clips of 2 to 28 s, three quarters at 44.1 kHz and one quarter at 48 kHz, to 16 and 32 kHz.  Prints one JSON line: the
card and its power limit (read in the same run), then per target rate
  device   the kernel time of each batch of the CLI's plan (CUDA events around the device calls only, one per input
           rate in the batch, after a warm-up pass over every batch): in total, and the achieved bytes / s and FP64
           FMA / s against their bounds (data sheet, H100 SXM at 700 W: 3.35 TB/s HBM3, 34 TFLOP/s FP64 without
           tensor cores = 17 T FMA / s), naming the bound that applies;
  cli      preprocess_a.py end to end on a temporary dataset (wall clock), and the same work split into phases run one
           after another in this process: read (resample.load on -t threads), device (pcm16_batch per rate: copies,
           kernels, synchronised) and write (scipy.io.wavfile.write);
  cpu      the oracle (scipy resample_poly in float64 and the numpy normalisation) per file on -t threads over a subset
           of the files, scaled to the whole set by samples.

    python scripts/bench_resample.py [-t 8] [--batch 64] [--cpu-files 48]"""
import argparse
import ctypes
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

N_CLIPS, SPEAKERS = 512, 4
HBM_BPS, FP64_FMA_PS = 3.35e12, 17e12


def clips(seed=0):
    """512 (rate, int16 clip) of 2 to 28 s: partials with vibrato over a little noise; every fourth clip at 48 kHz."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(N_CLIPS):
        sr = 48000 if i % 4 == 3 else 44100
        n = int(rng.uniform(2, 28) * sr)
        t = np.arange(n, dtype=np.float64) / sr
        ph = 2 * np.pi * rng.uniform(90, 400) * (t + 0.02 * np.sin(2 * np.pi * 5.0 * t))
        x = sum(0.25 / k * np.sin(k * ph) for k in (1, 2, 3, 5)) + 0.02 * rng.standard_normal(n)
        out.append((sr, (np.clip(x, -1, 1) * 32767).astype(np.int16)))
    return out


def device_arm(audio, rates, sr_out, plan):
    """Kernel time of every batch of the plan, one resample + normalise per input rate in the batch."""
    from whisper_vits_svc_b200 import _lib, resample as R
    calls, n_in, n_out, fmas, taps_bytes = [], 0, 0, 0.0, 0.0
    for g in plan:
        for rate in sorted({rates[i] for i in g}):
            idx = [i for i in g if rates[i] == rate]
            up, down = R.ratio(rate, sr_out)
            taps, rm = R._device_taps(up, down, torch.device("cuda"))
            lin = [audio[i].shape[0] for i in idx]
            lout = [R.out_len(n, rate, sr_out) for n in lin]
            so, oo = np.cumsum([0] + lin), np.cumsum([0] + lout)
            x = torch.from_numpy(np.concatenate([audio[i] for i in idx])).cuda()
            y = torch.empty(int(oo[-1]), device="cuda")
            p16 = torch.empty(int(oo[-1]), dtype=torch.int16, device="cuda")
            peak = torch.empty(len(idx), device="cuda")
            calls.append((x, y, p16, peak, (ctypes.c_int64 * len(so))(*[int(v) for v in so]),
                          (ctypes.c_int64 * len(oo))(*[int(v) for v in oo]), len(idx), up, down, taps, rm))
            n_in, n_out = n_in + sum(lin), n_out + sum(lout)
            fmas += sum(lout) * -(-taps.numel() // up)
            taps_bytes += 8.0 * taps.numel()

    def run(c):
        x, y, p16, peak, so, oo, n, up, down, taps, rm = c
        _lib.call("resample_ragged", x.data_ptr(), so, n, up, down, taps.data_ptr(), taps.numel(), rm, y.data_ptr())
        _lib.call("pcm16_normalise_ragged", y.data_ptr(), oo, n, p16.data_ptr(), peak.data_ptr())

    for c in calls:
        run(c)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = 0.0
    for c in calls:
        e0.record()
        run(c)
        e1.record()
        torch.cuda.synchronize()
        ms += e0.elapsed_time(e1)
    s = ms / 1e3
    # algorithmic bytes: fp32 input read, fp32 output written by the FIR and read twice by the normaliser, int16 out
    nbytes = 4.0 * n_in + 4.0 * 3 * n_out + 2.0 * n_out + taps_bytes
    t_bytes, t_fma = nbytes / HBM_BPS, fmas / FP64_FMA_PS
    return dict(device_calls=len(calls), ms_total=round(ms, 2), outputs=n_out,
                gb_per_s=round(nbytes / s / 1e9, 1), fp64_tfma_per_s=round(fmas / s / 1e12, 3),
                bound="bytes" if t_bytes >= t_fma else "fp64",
                bound_ms=round(1e3 * max(t_bytes, t_fma), 3), share_of_bound=round(max(t_bytes, t_fma) / s, 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("-t", "--threads", type=int, default=8)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--cpu-files", type=int, default=48)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_resample needs a CUDA device (an H100)")
    from scipy.io import wavfile
    from bench_retrieval import gpu_info
    from oracle import resample_oracle as RO
    from whisper_vits_svc_b200 import dataset, resample as R
    import preprocess_a as CLI
    name, power = gpu_info()
    data = clips()
    rates = [sr for sr, _ in data]
    audio = [x.astype(np.float32) / np.float32(32768) for _, x in data]
    audio_s = sum(x.shape[0] / sr for sr, x in data)
    plan = dataset.plan_window([x.shape[0] for x in audio], args.batch, CLI.MAX_PADDED)
    res = {}
    with tempfile.TemporaryDirectory() as tmp:
        for i, (sr, x) in enumerate(data):
            d = os.path.join(tmp, "raw", f"spk{i % SPEAKERS}")
            os.makedirs(d, exist_ok=True)
            wavfile.write(os.path.join(d, f"{i:03d}.wav"), sr, x)
        for sr_out in (16000, 32000):
            dev = device_arm(audio, rates, sr_out, plan)
            torch.cuda.empty_cache()
            out = f"waves-{sr_out // 1000}k"
            t0 = time.perf_counter()
            r = subprocess.run([sys.executable, os.path.join(ROOT, "preprocess_a.py"), "-w", "raw", "-o", out, "-s",
                                str(sr_out), "-t", str(args.threads), "--batch", str(args.batch)], cwd=tmp,
                               capture_output=True, text=True)
            cli_s = time.perf_counter() - t0
            if r.returncode != 0 or "failed" in r.stderr:
                raise SystemExit(r.stderr[-3000:])
            cwd = os.getcwd()
            os.chdir(tmp)   # the reference's walk takes paths relative to the working directory
            jobs = [(os.path.join(tmp, w), os.path.join(tmp, p)) for w, p in CLI.resample_jobs("raw", out + "-phases")]
            os.chdir(cwd)
            t0 = time.perf_counter()
            with ThreadPoolExecutor(args.threads) as pool:
                loaded = list(pool.map(lambda j: R.load(j[0]), jobs))
            t1 = time.perf_counter()
            pcm = [None] * len(jobs)
            for g in dataset.plan_window([x.shape[0] for x, _ in loaded], args.batch, CLI.MAX_PADDED):
                for rate in sorted({loaded[i][1] for i in g}):
                    idx = [i for i in g if loaded[i][1] == rate]
                    for i, p in zip(idx, R.pcm16_batch([loaded[i][0] for i in idx], rate, sr_out)[0]):
                        pcm[i] = p
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            for (_, p), y in zip(jobs, pcm):
                wavfile.write(p, sr_out, y)
            t3 = time.perf_counter()
            same = all(open(p, "rb").read() == open(p.replace(out + "-phases", out), "rb").read() for _, p in jobs[::37])
            cli = dict(end_to_end_s=round(cli_s, 2), files_per_s=round(N_CLIPS / cli_s, 1),
                       audio_s_per_s=round(audio_s / cli_s), phases_s=dict(read=round(t1 - t0, 2),
                                                                           device=round(t2 - t1, 2),
                                                                           write=round(t3 - t2, 2)),
                       phase_files_equal_cli=same)
            del loaded, pcm
            sub = jobs[:: max(1, len(jobs) // args.cpu_files)][:args.cpu_files]
            sub_samples = sum(RO.decode(w)[1].shape[0] for w, _ in sub)
            t0 = time.perf_counter()
            with ThreadPoolExecutor(args.threads) as pool:
                list(pool.map(lambda j: RO.pcm16(RO.load(j[0], sr_out)), sub))
            cpu_sub = time.perf_counter() - t0
            cpu = dict(kind=f"oracle (scipy resample_poly, float64) per file, {args.threads} threads", files=len(sub),
                       seconds=round(cpu_sub, 2),
                       scaled_to_all_s=round(cpu_sub * sum(x.shape[0] for x in audio) / sub_samples, 1))
            res[str(sr_out)] = dict(device=dev, cli=cli, cpu=cpu)
    print(json.dumps(dict(metric="resample", gpu=name, power_limit_w=power, clips=N_CLIPS, batches=len(plan),
                          audio_s=round(audio_s, 1), **res)))


if __name__ == "__main__":
    main()
