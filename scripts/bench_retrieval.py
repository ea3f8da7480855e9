#!/usr/bin/env python
"""Feature retrieval on the device (svcb_ivf_retrieve) at the headline batch: M = 32,000 feature rows (BASELINE
configs[3]: 32 x 1000 frames), k = 3, nprobe = 1, over synthetic clustered IVF-Flat indexes built on the device:

    compressed    10,000 vectors, nlist = min(16 sqrt(N), N / 39) = 256    (svc_train_retrieval.py's k-means path)
    uncompressed 200,000 vectors, nlist = 5,128

each at d = 1280 (PPG) and d = 256 (HuBERT).  Prints one JSON line: the card and its power limit (read in the same
run), ms per call (CUDA events, warmed up), the per-kernel split (svcb_timing_report, a separate pass), the coarse
GEMM's TFLOP/s (algorithmic fp32 FLOPs 2 M nlist d; the bf16x3 GEMM executes 3x that on the tensor cores) against the
peak bench.py uses, the scan's GB/s (bytes booked at the average list size), and the numpy oracle's CPU time on
1,000 rows (`kind: "port"`: the oracle restatement, not faiss).

    python scripts/bench_retrieval.py [--rows 32000] [--iters 20]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

WORKLOADS = [("compressed", 10_000, 256), ("uncompressed", 200_000, 5_128)]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True, check=True).stdout.strip()
    name, pl = [s.strip() for s in q.splitlines()[0].split(",")]
    return name, float(pl)


def build_index(ntotal, nlist, d, seed):
    """Clustered vectors around nlist random centroids, listed by centroid, built with torch on the device."""
    from whisper_vits_svc_b200.retrieval import IVFFlat
    g = torch.Generator(device="cuda").manual_seed(seed)
    cen = torch.randn(nlist, d, device="cuda", generator=g)
    lst = torch.randint(0, nlist, (ntotal,), device="cuda", generator=g)
    order = torch.argsort(lst, stable=True)
    lst = lst[order]
    vec = cen[lst] + 0.35 * torch.randn(ntotal, d, device="cuda", generator=g)
    off = torch.zeros(nlist + 1, dtype=torch.int64, device="cuda")
    off[1:] = torch.cumsum(torch.bincount(lst, minlength=nlist), 0)
    ix = IVFFlat(d=d, nlist=nlist, nprobe=1, metric=1, centroids=cen.cpu().numpy(), list_offsets=off.cpu().numpy(),
                 vectors=vec.cpu().numpy(), ids=order.cpu().numpy().astype(np.int64))
    return ix, cen


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=32_000)
    ap.add_argument("--k", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--port-rows", type=int, default=1000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_retrieval needs a CUDA device (an H100)")
    import bench
    from oracle import retrieval_oracle as RO
    from whisper_vits_svc_b200 import _lib, retrieval as R
    lib = _lib.load()
    name, power = gpu_info()
    peaks = bench.load_peaks()
    results = []
    for wl, ntotal, nlist in WORKLOADS:
        for d in (1280, 256):
            ix, cen = build_index(ntotal, nlist, d, seed=d + nlist)
            g = torch.Generator(device="cuda").manual_seed(7)
            x = cen[torch.randint(0, nlist, (args.rows,), device="cuda", generator=g)] + \
                0.4 * torch.randn(args.rows, d, device="cuda", generator=g)
            dev = R.DeviceIVFIndex(ix, 0.5, args.k, "cuda")
            for _ in range(args.warmup):
                dev.retriv(x)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                dev.retriv(x)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / args.iters
            lib.svcb_timing_enable(1)
            for _ in range(args.iters):
                dev.retriv(x)
            torch.cuda.synchronize()
            rep = lib.svcb_timing_report().decode()
            lib.svcb_timing_enable(0)
            rows, table, _ = bench.kernel_families(rep, args.iters)
            by = {r["name"]: r for r in rows}
            co, sc = by["ivf_coarse_tc"], by["ivf_scan_blend"]
            coarse_tf = co["flops"] / (co["ms"] * 1e-3) / 1e12
            xs = x[:args.port_rows].cpu().numpy()
            t0 = time.perf_counter()
            dist, _, _, vecs = RO.search(ix, xs, args.k)
            RO.blend_defined(xs, dist, vecs, 0.5)
            port_ms = (time.perf_counter() - t0) * 1e3
            results.append(dict(
                workload=wl, ntotal=ntotal, nlist=nlist, d=d, rows=args.rows, k=args.k, nprobe=1, ms_per_call=round(ms, 3),
                kernels=table,
                coarse=dict(tflops_fp32_algorithmic=round(coarse_tf, 1), tflops_bf16_executed=round(3 * coarse_tf, 1),
                            peak_bf16=peaks["tf_sust"], frac_of_peak=round(3 * coarse_tf / peaks["tf_sust"], 3),
                            peak_source=f"{peaks['src']} (MEASURED_PEAKS.json sustained bf16, else the H100 SXM data sheet)"),
                scan=dict(gbs_booked=round(sc["bytes"] / (sc["ms"] * 1e-3) / 1e9, 1), ms=round(sc["ms"] / args.iters, 3)),
                port=dict(kind="port", rows=args.port_rows, cpu_ms=round(port_ms, 1))))
            del dev, ix, x, cen
            torch.cuda.empty_cache()
    print(json.dumps(dict(metric="feature_retrieval", gpu=name, power_limit_w=power, results=results)))


if __name__ == "__main__":
    main()
