#!/usr/bin/env python
"""The dense Conv1d shapes of the headline step (csrc/conv_tc.cu) at B = 32, T = 1000, one at a time through
svcb_op_conv_tc: channel-major input, pre-packed weights, the epilogue each call site uses (gate for the flow's
`in`, ReLU for `ffn1`, Mish for the generator's `conv_pre`).  The prior's `pre` / `hub` read a time-major input in
the step; here they read a channel-major one.  The generator's `comb` / noise convs take the combined upsampler's
second input and are not timed here.

Prints one JSON line: the card, its power limit and max SM clock (read in the same run) and, per shape, ms per call
(CUDA events over --iters calls, warmed up), algorithmic TFLOP/s (2 Cin Cout K B T over the time) and the tensor
work's share of the 989 TFLOP/s dense bf16 data-sheet peak (bf16x3 issues 3 bf16 products per algorithmic one).

    python scripts/bench_conv_tc.py [--batch 32] [--frames 1000] [--iters 20] [--precision 3]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

PEAK_BF16 = 989e12
# name, Cin, Cout, K, flags, act, launches per step (CONV_GATE = 4; ACT_RELU = 1, ACT_MISH = 2)
SHAPES = [
    ("prior.pre", 1280, 192, 5, 0, 0, 1),
    ("prior.hub", 256, 192, 5, 0, 0, 1),
    ("prior.qkv", 192, 576, 1, 0, 0, 6),
    ("prior.o", 192, 192, 1, 0, 0, 6),
    ("prior.ffn1", 192, 640, 3, 0, 1, 6),
    ("prior.ffn2", 640, 192, 3, 0, 0, 6),
    ("prior.proj", 192, 384, 1, 0, 0, 1),
    ("flow.pre", 96, 192, 1, 0, 0, 4),
    ("flow.in", 192, 384, 5, 4, 0, 16),
    ("flow.rs", 192, 384, 1, 0, 0, 16),
    ("flow.post", 192, 96, 1, 0, 0, 4),
    ("gen.conv_pre", 192, 320, 7, 0, 2, 1),
]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                        "-i", str(torch.cuda.current_device())], capture_output=True, text=True, check=True).stdout
    name, pl, clk = [s.strip() for s in q.strip().splitlines()[0].split(",")]
    return name, float(pl), float(clk)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--precision", type=int, default=3, choices=[1, 3])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_conv_tc.py needs a CUDA device")
    from whisper_vits_svc_b200 import _lib, pack
    lib = _lib.load()
    name, power, clk = gpu_info()
    B, T, ns = args.batch, args.frames, args.precision
    g = torch.Generator().manual_seed(0)
    rows = []
    for sname, cin, cout, k, flags, act, per_step in SHAPES:
        x = torch.randn(B, cin, T, generator=g).cuda()
        w = torch.randn(cout, cin, k, generator=g) / (cin * k) ** 0.5
        wtc = pack.pack_conv_tc_general(w).cuda()
        b = (torch.randn(cout, generator=g) * 0.1).cuda()
        y = torch.empty(B, cout // 2 if flags & 4 else cout, T, device="cuda")
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

        def call():
            st = lib.svcb_op_conv_tc(x.data_ptr(), wtc.data_ptr(), b.data_ptr(), y.data_ptr(), None, None,
                                     B, cin, cout, T, k, 1, ns, flags, act, stream)
            _lib.check(st, "svcb_op_conv_tc")

        for _ in range(args.warmup):
            call()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            call()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.iters
        flop = 2.0 * cin * cout * k * B * T
        tflops = flop / (ms * 1e-3) / 1e12
        rows.append({"shape": sname, "cin": cin, "cout": cout, "k": k, "launches_per_step": per_step,
                     "ms": round(ms, 4), "ms_per_step": round(ms * per_step, 3), "tflops": round(tflops, 1),
                     "tensor_share_of_peak": round(tflops * 1e12 * (3 if ns == 3 else 1) / PEAK_BF16, 3)})
    print(json.dumps({"gpu": name, "power_limit_w": power, "max_sm_clock_mhz": clk, "batch": B, "frames": T,
                      "precision": ns, "iters": args.iters,
                      "family_ms_per_step": round(sum(r["ms_per_step"] for r in rows), 3), "shapes": rows}))


if __name__ == "__main__":
    main()
