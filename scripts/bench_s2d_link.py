#!/usr/bin/env python
"""The space-to-depth AMP links of generator stages 2-4 (csrc/amp_s2d.cu) at B = 32, T = 1000, one shape at a time
through ops.amp_s2d_link.  A shape is (C, k, dilation, Snake output or not, residual or not); the step runs 54
links over 15 distinct shapes per stage, each c1 link without a residual, each c2 link with one, every link but a
block's last with the next SnakeAlias in its epilogue.  A c1 link of dilation d runs on the fold pack.s2d_fold
picks (its input image permuted inside blocks of r*d samples, the undilated conv's taps), and a c2 link writes the
image in the fold of the c1 link after it; each row reports the folds, taps and tile rows.  The c2 shapes are timed
writing the standard image and both folded images, and without the Snake output: that link is the MMA side plus a
plain fp32 store, so the differences are what the Snake epilogue and the folded store cost.

ops.amp_s2d_link also clears the images, runs snake_pack_s2d and unpacks the output image; only the
`amp_s2d_link_*` launches are counted (svcb_timing_enable / svcb_timing_report: CUDA events around each launch).
ops.amp_s2d_link always writes the fp32 result, which the step's c1 links do not.

Prints one JSON line: the card, its power limit and max SM clock (read in the same run) and, per shape, ms per
launch, the launches per step, the tensor work's share of the 989 TFLOP/s dense bf16 data-sheet peak (3 bf16
products per tap column and tile row, halo rows included, edge taps counted over their reached columns), and the HBM bytes a launch must move with their share of the
3.35 TB/s data-sheet bandwidth: per element 4 B of bf16 hi/lo input image read and 4 B of y written, plus 4 B of
residual read and 4 B of bf16 hi/lo output image written when the shape has them.  The weights are read from L2.

    python scripts/bench_s2d_link.py [--batch 32] [--frames 1000] [--iters 20]"""
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
STAGES = [(40, 80), (20, 160), (10, 320)]   # (C, samples per frame) of generator stages 2-4
KERNELS = (3, 7, 11)
DILATIONS = (1, 3, 5)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                        "-i", str(torch.cuda.current_device())], capture_output=True, text=True, check=True).stdout
    name, pl, clk = [s.strip() for s in q.strip().splitlines()[0].split(",")]
    return name, float(pl), float(clk)


def link_ms(lib, call, iters):
    """Summed duration and count of the amp_s2d_link_* launches of `iters` calls."""
    lib.svcb_timing_enable(1)
    for _ in range(iters):
        call()
    torch.cuda.synchronize()
    rep = lib.svcb_timing_report().decode()
    lib.svcb_timing_enable(0)
    ms, n = 0.0, 0
    for line in rep.strip().splitlines():
        f = line.split()
        if f[0].startswith("amp_s2d_link_"):
            n += int(f[1]); ms += float(f[2])
    assert n == iters, (n, iters, rep)
    return ms / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_s2d_link.py needs a CUDA device")
    from whisper_vits_svc_b200 import _lib, ops, pack
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
        r = pack.s2d_factor(C)
        x = torch.randn(B, C, L, device="cuda", generator=gd)
        res = torch.randn(B, C, L, device="cuda", generator=gd)
        a_in, b_in, a_out, b_out = (torch.randn(C, generator=g) * 0.3 for _ in range(4))
        bias = (torch.randn(C, generator=g) * 0.1).cuda()
        for k in KERNELS:
            # (dilation, residual, output fold, launches per step with Snake output, without): c1 links read the fold
            # pack.s2d_fold picks; c2 links write the next c1 link's fold (c2[0] for d = 3, c2[1] for d = 5), and
            # each c2 shape is also timed writing the standard image and both folds, so that the folded store's cost
            # shows on its own
            nxt = [pack.s2d_fold(k, d, r) for d in DILATIONS[1:]]
            shapes = [(d, False, 1, 1, 0) for d in DILATIONS]
            shapes += [(1, True, f, sum(n == f for n in nxt), 1 if f == 1 else 0) for f in (1, 3, 5)]
            for d, with_res, fout, n_snake, n_plain in shapes:
                w = torch.randn(C, C, k, generator=g) / (C * k) ** 0.5
                fin = pack.s2d_fold(k, d, r)
                mlo, mhi = pack.s2d_taps(k, 1 if fin > 1 else d, r)
                for snake, per_step in ((True, n_snake), (False, n_plain)):
                    if not snake and fout > 1:
                        continue
                    halo, S, _ = pack.s2d_tile(r, fin, fout if snake else 1, mlo, mhi)
                    ntiles = B * ((L // r + 4 + S - 1) // S)

                    def call():
                        ops.amp_s2d_link(x, a_in, b_in, fu, fd, w, bias, dilation=d, res=res if with_res else None,
                                         alpha_out=a_out if snake else None, beta_out=b_out if snake else None,
                                         out_dilation=fout if snake else 1)

                    for _ in range(args.warmup):
                        call()
                    ms = link_ms(lib, call, args.iters)
                    cols = sum(n1 - n0 for n0, n1 in pack.s2d_tap_cols(k, 1 if fin > 1 else d, r))
                    tensor_flop = 3 * 2.0 * 160 * cols * ntiles * 128
                    hbm_bytes = (8 + 4 * with_res + 4 * snake) * B * C * L
                    rows.append({"C": C, "r": r, "k": k, "dilation": d, "fold_in": fin, "fold_out": fout,
                                 "ntaps": mlo + mhi + 1, "tile_rows": S + 2 * halo, "useful_rows": S, "snake": snake,
                                 "res": with_res, "launches_per_step": per_step, "ms": round(ms, 4),
                                 "tensor_share_of_peak": round(tensor_flop / (ms * 1e-3) / PEAK_BF16, 3),
                                 "hbm_bytes": hbm_bytes, "hbm_share_of_peak": round(hbm_bytes / (ms * 1e-3) / PEAK_HBM, 3)})
        del x, res
        torch.cuda.empty_cache()
    print(json.dumps({"gpu": name, "power_limit_w": power, "max_sm_clock_mhz": clk, "batch": B, "frames": args.frames,
                      "iters": args.iters, "launches_per_step": sum(r["launches_per_step"] for r in rows),
                      "family_ms_per_step": round(sum(r["ms"] * r["launches_per_step"] for r in rows), 3),
                      "shapes": rows}))


if __name__ == "__main__":
    main()
