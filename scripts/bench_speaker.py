#!/usr/bin/env python
"""LSTM speaker encoder on the device (svcb_speaker_mel + svcb_speaker_embed) for B = 1, 8, 32 and 128 utterances of
10 s (T = 626 mel frames: the encoder's work is fixed once T >= 250).  Prints one JSON line: the card and its power
limit (read in the same run), ms per call and utterances / s (CUDA events, warmed up), the per-kernel split from
svcb_timing_report (a separate pass; the recurrence also per step, kernel time / 250), achieved TFLOP/s from the
algorithmic counts of the reference's fp32 form, and the CPU arm: the oracle's fp32 torch restatement of one
utterance at 16 threads, timed in the same run.

    python scripts/bench_speaker.py [--batches 1,8,32,128] [--iters 5]"""
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

SECONDS, SR = 10.0, 16000
# launch_gemm_tc / launch_ivf_pack book each launch under these names as well as under the spk_gemm_* / spk_pack scope
# around them; they are left out so that the kernels below sum to the call
NESTED = ("whisper_gemm_tc", "ivf_pack")
AUDIO = dict(preemphasis=0.98, ref_level_db=20.0, min_level_db=-100.0, max_norm=4.0, trim_db=60.0)


def utterance_flops():
    """Algorithmic FLOPs of one compute_embedding at T >= 250 (10 windows x 250 steps) in the reference's fp32 form."""
    rows = 10 * 250
    inp = 2 * rows * 4 * 768 * (80 + 256 + 256)
    rec = 3 * 2 * rows * 4 * 768 * 768
    proj = 3 * 2 * rows * 768 * 256
    return inp + rec + proj, rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,8,32,128")
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_speaker needs a CUDA device (an H100)")
    from bench_retrieval import gpu_info
    from oracle import speaker_oracle as SO
    from whisper_vits_svc_b200 import _lib, synth
    from whisper_vits_svc_b200 import speaker_infer as S
    lib = _lib.load()
    name, power = gpu_info()
    sd = synth.speaker_checkpoint(1)["model"]
    enc = S.SpeakerEncoderB200(sd, AUDIO, "cuda")
    n = int(SECONDS * SR)
    rng = np.random.default_rng(0)
    pool = [(0.3 * rng.standard_normal(n)).astype(np.float32) for _ in range(8)]
    f_utt, f_rec = utterance_flops()
    results = []
    for B in [int(b) for b in args.batches.split(",")]:
        wavs = [pool[i % len(pool)] for i in range(B)]
        for _ in range(args.warmup):
            enc.embed(wavs)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            enc.embed(wavs)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.iters
        lib.svcb_timing_enable(1)
        enc.embed(wavs)
        torch.cuda.synchronize()
        rep = lib.svcb_timing_report().decode()
        lib.svcb_timing_enable(0)
        kernels = {}
        for line in rep.strip().splitlines():
            k, cnt, kms, fl, by, _ = line.split()
            if k in NESTED:
                continue
            kernels[k] = dict(launches=int(cnt), ms=round(float(kms), 3),
                              tflops=round(float(fl) / (float(kms) * 1e-3) / 1e12, 1) if float(fl) > 0 else None)
        rec = kernels.get("spk_lstm_rec", {})
        results.append(dict(B=B, ms_per_call=round(ms, 2), utt_per_s=round(B / (ms * 1e-3), 1),
                            tflops_algorithmic=round(B * f_utt / (ms * 1e-3) / 1e12, 2),
                            rec_us_per_step=round(rec.get("ms", 0) * 1e3 / (rec.get("launches", 1) * 250), 2),
                            rec_tflops_algorithmic=round(B * f_rec / (rec.get("ms", 1) * 1e-3) / 1e12, 2), kernels=kernels))
    torch.set_num_threads(16)
    x = SO.prepare(pool[0])
    t0 = time.perf_counter()
    mel = SO.melspectrogram(x).T
    SO.compute_embedding(sd, mel)
    cpu_ms = (time.perf_counter() - t0) * 1e3
    print(json.dumps(dict(metric="speaker_encoder", gpu=name, power_limit_w=power, seconds=SECONDS,
                          gflop_per_utterance=round(f_utt / 1e9, 1), results=results,
                          cpu=dict(kind="oracle fp32 torch, 16 threads", ms_per_utterance=round(cpu_ms, 1)))))


if __name__ == "__main__":
    main()
