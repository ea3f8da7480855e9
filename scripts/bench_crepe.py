#!/usr/bin/env python
"""Measures the CREPE-full pitch extractor on the device: 512 clips of 2 to 28 s (the length mix of bench_preprocess.py)
at hop 320 (`pitch_inference.py`) and hop 160 (`preprocess_crepe.py`), with seeded weights.

Reports CUDA-event time of the probabilities and of the decoder after a warm-up pass over the same shapes, the
per-kernel split of `svcb_timing_report` (taken in a pass of its own, since its events serialise the stream), frames/s,
audio seconds per second, and the convolutions' TFLOP/s against the bf16 dense peak of the card as found (name, power
limit and SM clock are printed beside it).  The CPU arm runs the fp32 oracle on 64 frames at the host's thread count and
scales it to the frame count: it is labelled as scaled.  Nothing here changes a device setting."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.append(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

MAC_PER_FRAME = 256 * 1024 * 512 + 64 * (128 * 128 * 1024 + 64 * 128 * 128 + 32 * 128 * 128 + 16 * 256 * 128 + 8 * 512 * 256) + 2048 * 360
H100_BF16_DENSE_TFLOPS = 989.0   # NVIDIA data sheet, H100 SXM at 700 W


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=512)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--cpu-frames", type=int, default=64)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_crepe.py measures the device path; there is no CPU path"
    from oracle import crepe_oracle as O
    from whisper_vits_svc_b200 import _lib, crepe_infer as C, synth

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    sd = synth.crepe_checkpoint(1234, "full")
    model = C.CrepeB200(sd, "cuda", "full")
    g = np.random.default_rng(0)
    lengths = (g.uniform(2.0, 28.0, args.clips) * 16000).astype(np.int64)
    clips = [torch.from_numpy((g.standard_normal(n) * 0.1).astype(np.float32)).cuda() for n in lengths]
    noises = [torch.randn(int(n), device="cuda") for n in lengths]
    lib = _lib.load()
    out = {"card": card, "clips": args.clips, "audio_s": float(lengths.sum() / 16000), "gflop_per_frame": 2 * MAC_PER_FRAME / 1e9}

    def run(hop, timing=False):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        t_probs = t_dec = 0.0
        frames = 0
        for i in range(0, args.clips, args.batch):
            ev[0].record()
            probs, fo = model.probs_device(clips[i:i + args.batch], hop, noises[i:i + args.batch])
            ev[1].record()
            C.decode_device(probs, fo, torch.zeros(fo[-1]))
            ev[2].record()
            torch.cuda.synchronize()
            t_probs += ev[0].elapsed_time(ev[1]) / 1e3
            t_dec += ev[1].elapsed_time(ev[2]) / 1e3
            frames += fo[-1]
        return t_probs, t_dec, frames

    for hop in (320, 160):
        run(hop)   # warm-up: every shape of the timed pass
        t0 = time.perf_counter()
        t_probs, t_dec, frames = run(hop)
        wall = time.perf_counter() - t0
        lib.svcb_timing_enable(1)
        run(hop)
        report = lib.svcb_timing_report().decode()
        lib.svcb_timing_enable(0)
        out[f"hop{hop}"] = {
            "frames": int(frames), "probs_s": t_probs, "decode_s": t_dec, "wall_s": wall,
            "frames_per_s": frames / (t_probs + t_dec), "audio_s_per_s": out["audio_s"] / (t_probs + t_dec),
            "decoder_share": t_dec / (t_probs + t_dec),
            "network_tflops": frames * 2 * MAC_PER_FRAME / t_probs / 1e12,
            "share_of_data_sheet_bf16_peak": frames * 2 * MAC_PER_FRAME / t_probs / 1e12 / H100_BF16_DENSE_TFLOPS,
        }
        print(f"--- hop {hop}: per-kernel timing\n{report}")

    fr = O.frames(clips[0].cpu()[:args.cpu_frames * 320], 320)[:args.cpu_frames]
    O.network(sd, fr[:4])
    t0 = time.perf_counter()
    O.network(sd, fr)
    cpu = (time.perf_counter() - t0) / fr.shape[0]
    out["cpu_oracle"] = {"threads": torch.get_num_threads(), "s_per_frame": cpu,
                         "hop320_s_scaled_from_%d_frames" % fr.shape[0]: cpu * out["hop320"]["frames"]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
