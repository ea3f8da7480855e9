#!/usr/bin/env python
"""Cutting the two lowest STFT bins out of raw recordings (svcb_cdc_ragged, preprocess_cdc.py) on 512 seeded clips of
2 to 28 s at 48 kHz.  Prints one JSON line: the card and its power limit (read in the same run), then
  device   the kernel time of each batch of the CLI's plan (CUDA events around the device calls only, after a warm-up
           pass over every batch): in total, and the achieved bytes / s and FP64 FMA / s against their bounds (data
           sheet, H100 SXM at 700 W: 3.35 TB/s HBM3, 34 TFLOP/s FP64 without tensor cores = 17 T FMA / s), naming the
           bound that applies.  Bytes are 4 read and 2 written per sample; FMAs are 3 x 1024 per frame and 12 per
           output sample;
  cli      preprocess_cdc.py end to end on a temporary dataset (wall clock), and the same work split into phases run
           one after another in this process: read (cdc.load on -t threads), device (cdc_batch per batch: copies and
           kernels, synchronised) and write (scipy.io.wavfile.write);
  cpu      the oracle (torch.stft / istft in float32, one torch thread each) per file on -t threads over a subset of
           the files, scaled to the whole set by samples.

    python scripts/bench_cdc.py [-t 8] [--batch 64] [--cpu-files 48]"""
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
HBM_BPS, FP64_FMA_PS = 3.35e12, 17e12


def clips(seed=0):
    """512 int16 clips of 2 to 28 s at 48 kHz: partials with vibrato, a DC offset, mains hum and a little noise."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(N_CLIPS):
        n = int(rng.uniform(2, 28) * SR)
        t = np.arange(n, dtype=np.float64) / SR
        ph = 2 * np.pi * rng.uniform(90, 400) * (t + 0.02 * np.sin(2 * np.pi * 5.0 * t))
        x = sum(0.25 / k * np.sin(k * ph) for k in (1, 2, 3, 5)) + rng.uniform(-0.05, 0.05)
        x = x + 0.05 * np.sin(2 * np.pi * rng.choice([50.0, 60.0]) * t) + 0.02 * rng.standard_normal(n)
        out.append((np.clip(x, -1, 1) * 32767).astype(np.int16))
    return out


def device_arm(audio, plan):
    """Kernel time of every batch of the plan, one svcb_cdc_ragged call each."""
    from whisper_vits_svc_b200 import _lib, cdc
    calls, n_in, n_out, frames = [], 0, 0, 0
    for g in plan:
        lin = [audio[i].shape[0] for i in g]
        lout = [cdc.out_len(n) for n in lin]
        x = torch.from_numpy(np.concatenate([audio[i] for i in g])).cuda()
        out = torch.empty(sum(lout), dtype=torch.int16, device="cuda")
        calls.append((x, _lib.offsets(lin), len(g), out))
        n_in, n_out, frames = n_in + sum(lin), n_out + sum(lout), frames + sum(n // 256 + 1 for n in lin)

    def run(c):
        x, so, b, out = c
        _lib.call("cdc_ragged", x.data_ptr(), so, b, out.data_ptr())

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
    nbytes = 4.0 * n_in + 2.0 * n_out
    fmas = 3.0 * 1024 * frames + 12.0 * n_out
    t_bytes, t_fma = nbytes / HBM_BPS, fmas / FP64_FMA_PS
    return dict(device_calls=len(calls), ms_total=round(ms, 2), samples=n_in,
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
        raise SystemExit("bench_cdc needs a CUDA device (an H100)")
    from scipy.io import wavfile
    from bench_retrieval import gpu_info
    from oracle import cdc_oracle as CO
    from whisper_vits_svc_b200 import cdc, dataset
    import preprocess_cdc as CLI
    name, power = gpu_info()
    data = clips()
    audio = [x.astype(np.float32) / np.float32(32768) for x in data]
    audio_s = sum(x.shape[0] for x in data) / SR
    plan = dataset.plan_window([x.shape[0] for x in audio], args.batch, CLI.MAX_PADDED)
    dev = device_arm(audio, plan)
    torch.cuda.empty_cache()
    with tempfile.TemporaryDirectory() as tmp:
        for i, x in enumerate(data):
            d = os.path.join(tmp, "raw", f"spk{i % SPEAKERS}")
            os.makedirs(d, exist_ok=True)
            wavfile.write(os.path.join(d, f"{i:03d}.wav"), SR, x)
        t0 = time.perf_counter()
        r = subprocess.run([sys.executable, os.path.join(ROOT, "preprocess_cdc.py"), "-i", "raw", "-o", "cdc", "-t",
                            str(args.threads), "--batch", str(args.batch)], cwd=tmp, capture_output=True, text=True)
        cli_s = time.perf_counter() - t0
        if r.returncode != 0 or "failed" in r.stderr:
            raise SystemExit(r.stderr[-3000:])
        cwd = os.getcwd()
        os.chdir(tmp)   # the reference's walk takes paths relative to the working directory
        jobs = [(os.path.join(tmp, w), os.path.join(tmp, p)) for w, p in CLI.cdc_jobs("raw", "cdc-phases")]
        os.chdir(cwd)
        t0 = time.perf_counter()
        with ThreadPoolExecutor(args.threads) as pool:
            loaded = list(pool.map(lambda j: cdc.load(j[0]), jobs))
        t1 = time.perf_counter()
        pcm = [None] * len(jobs)
        for g in dataset.plan_window([x.shape[0] for x, _ in loaded], args.batch, CLI.MAX_PADDED):
            for i, p in zip(g, cdc.cdc_batch([loaded[i][0] for i in g])):
                pcm[i] = p
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        for (_, p), y, (_, rate) in zip(jobs, pcm, loaded):
            wavfile.write(p, rate, y)
        t3 = time.perf_counter()
        same = all(open(p, "rb").read() == open(p.replace("cdc-phases", "cdc"), "rb").read() for _, p in jobs[::37])
        cli = dict(end_to_end_s=round(cli_s, 2), files_per_s=round(N_CLIPS / cli_s, 1),
                   audio_s_per_s=round(audio_s / cli_s), phases_s=dict(read=round(t1 - t0, 2), device=round(t2 - t1, 2),
                                                                       write=round(t3 - t2, 2)),
                   phase_files_equal_cli=same)
        # parity of the timed outputs: every sample within 1 LSB of the oracle on a subset, and the share that differs
        sub = jobs[:: max(1, len(jobs) // args.cpu_files)][:args.cpu_files]
        idx = [jobs.index(j) for j in sub]
        del loaded
        sub_samples = sum(data[i].shape[0] for i in idx)
        torch_threads = torch.get_num_threads()
        torch.set_num_threads(1)
        t0 = time.perf_counter()
        with ThreadPoolExecutor(args.threads) as pool:
            want = list(pool.map(lambda j: CO.cdc(CO.decode(j[0])[0]), sub))
        cpu_sub = time.perf_counter() - t0
        torch.set_num_threads(torch_threads)
        d = [np.abs(pcm[i].astype(np.int32) - w) for i, w in zip(idx, want)]
        parity = dict(files=len(idx), max_lsb=int(max(x.max() for x in d)),
                      share_differing=round(sum(int((x > 0).sum()) for x in d) / sum(x.size for x in d), 5))
        cpu = dict(kind=f"oracle (torch.stft / istft, float32) per file, {args.threads} threads", files=len(sub),
                   seconds=round(cpu_sub, 2), scaled_to_all_s=round(cpu_sub * sum(x.shape[0] for x in data) / sub_samples, 1))
    print(json.dumps(dict(metric="cdc", gpu=name, power_limit_w=power, clips=N_CLIPS, batches=len(plan),
                          audio_s=round(audio_s, 1), device=dev, cli=cli, cpu=cpu, parity=parity)))


if __name__ == "__main__":
    main()
