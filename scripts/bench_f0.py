#!/usr/bin/env python
"""WORLD DIO + StoneMask F0 (svcb_world_f0_ragged, preprocess_f0.py) on 512 seeded clips of 2 to 28 s at 16 kHz:
harmonic tones gliding across 80-800 Hz in voiced runs of 0.1-1.5 s, between pauses of low room noise.  Prints one
JSON line: the card and its power limit (read in the same run), then
  device   the kernel time of the CLI's plan per pass (CUDA events around --reps passes over every batch's svcb call,
           after a warm-up pass) and, from the library's per-kernel timing of one pass, each phase's time: bands (mean,
           centring, low-cut and band FIRs), events, candidates, fix and StoneMask.  The bands' share is of the fp64
           FMA bound (data sheet, H100 SXM at 700 W: 67 TFLOP/s), the other phases' of the HBM bound (3.35 TB/s);
  cli      preprocess_f0.py end to end on a temporary dataset (wall clock), and the same work split into phases run one
           after another in this process: read (load_audio on -t threads), device (raw F0 per batch: copies and
           kernels, synchronised), round (Python's round per value) and write (np.save);
  cpu      the numpy oracle (dio + stonemask) per file on -t processes over --cpu-files files, scaled to the whole set
           by samples.

    python scripts/bench_f0.py [-t 8] [--batch 64] [--cpu-files 48] [--reps 5]"""
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
FP64_FLOPS = 67e12
HBM_BPS = 3.35e12


def clips(seed=0):
    """512 float32 clips of 2 to 28 s at 16 kHz, 16-bit quantised as a wav holds them."""
    from oracle import f0_oracle as O
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(N_CLIPS):
        n = int(rng.uniform(2, 28) * SR)
        tr = np.zeros(n)
        p, voiced = 0, False
        while p < n:
            m = min(n - p, int(SR * (rng.uniform(0.1, 1.5) if voiced else rng.uniform(0.05, 0.8))))
            if voiced:
                a, b = rng.uniform(80, 800, 2)
                tr[p:p + m] = np.geomspace(a, b, m)
            p, voiced = p + m, not voiced
        x = O.tone(tr, rng, amp=rng.uniform(0.05, 0.5)) + 10 ** rng.uniform(-4, -2.5) * rng.standard_normal(n)
        out.append((np.clip(np.rint(x * 32767), -32768, 32767) / 32768).astype(np.float32))
    return out


def parse_timing(report):
    """name -> ms of svcb_timing_report()'s lines "name launches total_ms flops bytes"."""
    out = {}
    for line in report.decode().splitlines():
        f = line.split()
        if len(f) >= 3 and f[0].startswith("f0_"):
            out[f[0]] = float(f[2])
    return out


def device_arm(data, plan, reps):
    from whisper_vits_svc_b200 import _lib, world_f0
    lib = _lib.load()
    calls, n_in, n_fr = [], 0, 0
    ws_need = 0
    for g in plan:
        lin = [data[i].shape[0] for i in g]
        x = torch.from_numpy(np.concatenate([data[i] for i in g]).astype(np.float64)).cuda()
        fr = sum(world_f0.frames_of(n) for n in lin)
        out = torch.empty(fr, dtype=torch.float64, device="cuda")
        calls.append((x, _lib.offsets(lin), len(g), out))
        ws_need = max(ws_need, lib.svcb_world_f0_workspace_bytes(sum(lin), len(g)))
        n_in, n_fr = n_in + sum(lin), n_fr + fr
    ws = torch.empty(ws_need, dtype=torch.uint8, device="cuda")

    def run(c):
        x, so, b, out = c
        _lib.call("world_f0_ragged", x.data_ptr(), so, b, out.data_ptr(), ws.data_ptr(), ws.numel())

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
    taps = 641 + 4 * (80 + 56 + 40 + 28 + 20 + 14 + 10 + 7)
    flops = 2.0 * n_in * taps
    bound = dict(f0_bands=flops / FP64_FLOPS, f0_events=8.0 * 8 * n_in / HBM_BPS,
                 f0_candidates=8.0 * 8 * n_fr / HBM_BPS, f0_fix=8.0 * 12 * n_fr / HBM_BPS,
                 f0_stonemask=(8.0 * 2 * n_fr + 8.0 * n_in) / HBM_BPS)
    ph = {k: dict(ms=round(v, 3), share_of_bound=round(bound[k] / (v / 1e3), 3) if v > 0 else None)
          for k, v in phases.items()}
    del calls, ws
    torch.cuda.empty_cache()
    return dict(device_calls=len(plan), reps=reps, ms_per_pass=round(ms, 2), samples=n_in, frames=n_fr,
                band_fir_tflops=round(flops / (phases.get("f0_bands", ms) / 1e3) / 1e12, 2), phases=ph)


def _oracle_file(x):
    from oracle import f0_oracle as O
    return O.round1(O.world_f0(x))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("-t", "--threads", type=int, default=8)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--cpu-files", type=int, default=48)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_f0 needs a CUDA device (an H100)")
    from bench_retrieval import gpu_info
    from scipy.io import wavfile
    from whisper_vits_svc_b200 import dataset, hubert_infer, world_f0
    import preprocess_f0 as CLI
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
        r = subprocess.run([sys.executable, os.path.join(ROOT, "preprocess_f0.py"), "-w", "wav", "-p", "pit", "-t",
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
        raw = [None] * len(jobs)
        ex = world_f0.Extractor("cuda")
        for g in dataset.plan_window([x.shape[0] for x in loaded], args.batch, CLI.MAX_PADDED):
            for i, f in zip(g, ex.raw([loaded[i] for i in g])):
                raw[i] = f.cpu().numpy()
        torch.cuda.synchronize()
        ex.close()
        t2 = time.perf_counter()
        rounded = [world_f0.round1(f) for f in raw]
        t3 = time.perf_counter()
        for (_, p), f in zip(jobs, rounded):
            np.save(p, f, allow_pickle=False)
        t4 = time.perf_counter()
        same = all(np.array_equal(np.load(p + ".npy"), np.load(p.replace("pit-phases", "pit") + ".npy"))
                   for _, p in jobs[::17])
        voiced = float(np.mean(np.concatenate(rounded) > 0))
        cli = dict(end_to_end_s=round(cli_s, 2), files_per_s=round(N_CLIPS / cli_s, 1),
                   audio_s_per_s=round(audio_s / cli_s), voiced_share=round(voiced, 3),
                   phases_s=dict(read=round(t1 - t0, 2), device=round(t2 - t1, 2), round=round(t3 - t2, 2),
                                 write=round(t4 - t3, 2)), phase_files_equal_cli=same)
        sub = list(range(0, len(loaded), max(1, len(loaded) // args.cpu_files)))[:args.cpu_files]
        sub_samples = sum(loaded[i].shape[0] for i in sub)
        t0 = time.perf_counter()
        with ProcessPoolExecutor(args.threads) as pool:
            res = list(pool.map(_oracle_file, [loaded[i] for i in sub]))
        cpu_sub = time.perf_counter() - t0
        vu_equal = all(np.array_equal(r_ > 0, rounded[i] > 0) for r_, i in zip(res, sub))
        d = np.concatenate([np.abs(r_ - rounded[i]) for r_, i in zip(res, sub)])
        cpu = dict(kind=f"numpy oracle (dio + stonemask) per file, {args.threads} processes", files=len(sub),
                   seconds=round(cpu_sub, 2),
                   scaled_to_all_s=round(cpu_sub * sum(x.shape[0] for x in loaded) / sub_samples, 1),
                   voiced_unvoiced_equal_device=vu_equal, frames_differing=int(np.count_nonzero(d)),
                   frames=int(d.shape[0]), max_abs_diff_hz=round(float(d.max()), 3))
    print(json.dumps(dict(metric="world_f0", gpu=name, power_limit_w=power, clips=N_CLIPS, batches=len(plan),
                          audio_s=round(audio_s, 1), device=dev, cli=cli, cpu=cpu)))


if __name__ == "__main__":
    main()
