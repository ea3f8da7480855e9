#!/usr/bin/env python
"""Silero VAD on the device (svcb_vad_probs) on two workloads: one 50 s clip (the latency of svc_inference_post.py)
and 256 clips of 2 to 28 s in one ragged call (throughput).  Prints one JSON line: the card and its power limit (read
in the same run), ms per call (CUDA events, warmed up), windows / s and audio seconds / s, the split between the front
end (vad_front) and the recurrence (vad_rec) from svcb_timing_report (a separate pass), and the CPU arm: the oracle's
torch restatement run window by window as the reference's loop calls the model (an oracle port, not the live
TorchScript model), on the 50 s clip at 8 threads, timed in the same run.

    python scripts/bench_vad.py [--iters 10] [--warmup 3]"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

SR = 16000


def clip(rng, base, n):
    """Speech-like audio of n samples: the test.wav excerpt tiled at a random gain, with a little noise."""
    x = np.resize(np.roll(base, int(rng.integers(base.shape[0]))), n) * np.float32(rng.uniform(0.3, 1.5))
    return (x + 1e-3 * rng.standard_normal(n)).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cpu-threads", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vad needs a CUDA device (an H100)")
    from bench_retrieval import gpu_info
    from oracle import vad_oracle as VO
    from whisper_vits_svc_b200 import _lib
    from whisper_vits_svc_b200 import vad_infer as V
    lib = _lib.load()
    name, power = gpu_info()
    sd = VO.load_tensors()
    vad = V.VadB200(sd, "cuda")
    base = VO.load_golden("vad_test10s")["test10s.wav"]
    rng = np.random.default_rng(0)
    workloads = {"one_50s_clip": [clip(rng, base, 50 * SR)],
                 "ragged_256_clips_2_to_28s": [clip(rng, base, int(rng.uniform(2, 28) * SR)) for _ in range(256)]}
    results = {}
    for wl, wavs in workloads.items():
        flat = torch.from_numpy(np.concatenate(wavs))
        windows = sum(V.windows(w.shape[0]) for w in wavs)
        seconds = flat.numel() / SR
        # the call as the CLI makes it, minus the host-to-device copy of the audio
        dev = [flat[a:b].cuda() for a, b in zip(np.cumsum([0] + [w.shape[0] for w in wavs[:-1]]), np.cumsum([w.shape[0] for w in wavs]))]
        for _ in range(args.warmup):
            vad.speech_probs_device(dev)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            vad.speech_probs_device(dev)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.iters
        lib.svcb_timing_enable(1)
        vad.speech_probs_device(dev)
        torch.cuda.synchronize()
        rep = lib.svcb_timing_report().decode()
        lib.svcb_timing_enable(0)
        kernels = {}
        for line in rep.strip().splitlines():
            k, cnt, kms, fl, by, _ = line.split()
            kernels[k] = dict(launches=int(cnt), ms=round(float(kms), 3),
                              tflops=round(float(fl) / (float(kms) * 1e-3) / 1e12, 2) if float(fl) > 0 else None)
        longest = max(V.windows(w.shape[0]) for w in wavs)
        rec = kernels.get("vad_rec", {})
        results[wl] = dict(items=len(wavs), windows=windows, audio_s=round(seconds, 1), ms_per_call=round(ms, 3),
                           windows_per_s=round(windows / (ms * 1e-3)), audio_s_per_s=round(seconds / (ms * 1e-3)),
                           rec_us_per_step_longest_item=round(rec.get("ms", 0) * 1e3 / longest, 3) if rec else None,
                           kernels=kernels)
    torch.set_num_threads(args.cpu_threads)
    x = workloads["one_50s_clip"][0]
    t0 = time.perf_counter()
    VO.speech_probs(sd, x, per_window=True)
    cpu_s = time.perf_counter() - t0
    print(json.dumps(dict(metric="silero_vad", gpu=name, power_limit_w=power, results=results,
                          cpu=dict(kind=f"oracle port (torch CPU, per-window loop), {args.cpu_threads} threads",
                                   clip_s=50, seconds=round(cpu_s, 3)))))


if __name__ == "__main__":
    main()
