#!/usr/bin/env python
"""The AMP-link convolutions of generator stages 0-1 (csrc/amp_conv_tc.cu) at B = 32, T = 1000, one shape at a time
through ops.amp_conv_tc.  A shape is (C, k, dilation, residual, accumulate, divide).  Per stage and block (k = 3, 7,
11) the step runs three c1 links (dilation 1, 3, 5, no residual, into a temporary) and three c2 links (dilation 1,
with the residual); the third c2 link of the second and third block adds into the stage sum, and the very last one
also divides it by 3.  So each stage has 18 links over 14 distinct shapes.

ops.amp_conv_tc also runs snake_pack; only the `amp_conv_tc_*` launches are counted (svcb_timing_enable /
svcb_timing_report: CUDA events around each launch).

Prints one JSON line: the card, its power limit and max SM clock (read in the same run) and, per shape, ms per
launch, the launches per step, the tensor work's share of the 989 TFLOP/s dense bf16 data-sheet peak (3 bf16
products per tap and output row), and the HBM bytes a launch must move with their share of the 3.35 TB/s data-sheet
bandwidth: per element 4 B of bf16 hi/lo image read and 4 B of y written, plus 4 B each of residual and stage sum read.

    python scripts/bench_amp_conv_tc.py [--batch 32] [--frames 1000] [--iters 20]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

PEAK_BF16 = 989e12
PEAK_HBM = 3.35e12
STAGES = [(160, 5), (80, 20)]   # (C, samples per frame) of generator stages 0-1
KERNELS = (3, 7, 11)
DILATIONS = (1, 3, 5)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                        "-i", str(torch.cuda.current_device())], capture_output=True, text=True, check=True).stdout
    name, pl, clk = [s.strip() for s in q.strip().splitlines()[0].split(",")]
    return name, float(pl), float(clk)


def conv_ms(lib, call, iters):
    """Summed duration and count of the amp_conv_tc_* launches of `iters` calls."""
    lib.svcb_timing_enable(1)
    for _ in range(iters):
        call()
    torch.cuda.synchronize()
    rep = lib.svcb_timing_report().decode()
    lib.svcb_timing_enable(0)
    ms, n = 0.0, 0
    for line in rep.strip().splitlines():
        f = line.split()
        if f[0].startswith("amp_conv_tc_"):
            n += int(f[1]); ms += float(f[2])
    assert n == iters, (n, iters, rep)
    return ms / n


def stage_shapes(k):
    """(dilation, residual, accumulate, divide, launches per step) of block k's links"""
    c1 = [(d, False, False, False, 1) for d in DILATIONS]
    if k == 3:
        return c1 + [(1, True, False, False, 3)]
    if k == 7:
        return c1 + [(1, True, False, False, 2), (1, True, True, False, 1)]
    return c1 + [(1, True, False, False, 2), (1, True, True, True, 1)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_amp_conv_tc.py needs a CUDA device")
    from whisper_vits_svc_b200 import _lib, ops
    lib = _lib.load()
    name, power, clk = gpu_info()
    B = args.batch
    g = torch.Generator().manual_seed(0)
    gd = torch.Generator(device="cuda").manual_seed(0)
    fu = (torch.randn(12, generator=g) * 0.1).cuda()
    fd = (torch.randn(12, generator=g) * 0.1).cuda()
    rows = []
    for C, up in STAGES:
        L = args.frames * up
        x = torch.randn(B, C, L, device="cuda", generator=gd)
        res = torch.randn(B, C, L, device="cuda", generator=gd)
        acc = torch.randn(B, C, L, device="cuda", generator=gd)
        alpha, beta = (torch.randn(C, generator=g) * 0.3 for _ in range(2))
        bias = (torch.randn(C, generator=g) * 0.1).cuda()
        for k in KERNELS:
            w = torch.randn(C, C, k, generator=g) / (C * k) ** 0.5
            for d, with_res, accum, div, per_step in stage_shapes(k):
                def call():
                    ops.amp_conv_tc(x, alpha, beta, fu, fd, w, bias, dilation=d, res=res if with_res else None,
                                    acc=acc if accum else None, out_div=3.0 if div else 0.0)

                for _ in range(args.warmup):
                    call()
                ms = conv_ms(lib, call, args.iters)
                tensor_flop = 3 * 2.0 * C * C * k * B * L
                hbm_bytes = (8 + 4 * with_res + 4 * accum) * B * C * L
                rows.append({"C": C, "k": k, "dilation": d, "res": with_res, "accum": accum, "div": div,
                             "launches_per_step": per_step, "ms": round(ms, 4),
                             "tensor_share_of_peak": round(tensor_flop / (ms * 1e-3) / PEAK_BF16, 3),
                             "hbm_bytes": hbm_bytes, "hbm_share_of_peak": round(hbm_bytes / (ms * 1e-3) / PEAK_HBM, 3)})
        del x, res, acc
        torch.cuda.empty_cache()
    per_stage = {C: round(sum(r["ms"] * r["launches_per_step"] for r in rows if r["C"] == C), 3) for C, _ in STAGES}
    print(json.dumps({"gpu": name, "power_limit_w": power, "max_sm_clock_mhz": clk, "batch": B, "frames": args.frames,
                      "iters": args.iters, "launches_per_step": sum(r["launches_per_step"] for r in rows),
                      "family_ms_per_step": round(sum(per_stage.values()), 3),
                      "stage_ms_per_step": {f"c{C}": v for C, v in per_stage.items()}, "shapes": rows}))


if __name__ == "__main__":
    main()
