#!/usr/bin/env python
"""Building IVF-Flat retrieval indexes on the device (retrieval_train.py, csrc/kmeans_api.cu) at the sizes
svc_train_retrieval.py meets for a speaker with a few hours of audio, on synthetic clustered features made on the device:

    whisper      200,000 x 1280 -> nlist 5,128, 10 iterations, then the add
    hubert       200,000 x 256  -> nlist 5,128, 10 iterations, then the add
    compressed   540,000 x 1280 -> 10,000 centres (25 Lloyd iterations), then nlist 256 over those

Prints one JSON line: the card and its power limit (read in the same run), the wall time of each stage (host clock
around work that ends in a device synchronise; one warm-up run of the whole workload first), the per-kernel split
(svcb_timing_report, a separate pass), and the assignment GEMM's TFLOP/s (algorithmic fp32 FLOPs 2 n k d; the bf16x3 GEMM
executes 3x that on the tensor cores) against the peak bench.py uses.  The CPU arm (`kind: "port"`) is the numpy oracle's
k-means step (oracle/kmeans_oracle.py, the restatement, not faiss) on a subsample, scaled to the workload's rows.

    python scripts/bench_retrieval_train.py [--port-rows 4000]"""
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

WORKLOADS = [("whisper", 200_000, 1280, None), ("hubert", 200_000, 256, None), ("compressed", 540_000, 1280, 10_000)]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True, check=True).stdout.strip()
    name, pl, clk = [s.strip() for s in q.splitlines()[0].split(",")]
    return name, float(pl), float(clk)


def features(n, d, seed):
    """n rows around n / 40 random centres, spread 0.5, made with torch on the device."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    cen = torch.randn(max(1, n // 40), d, device="cuda", generator=g)
    return (cen[torch.randint(0, cen.shape[0], (n,), device="cuda", generator=g)] +
            0.5 * torch.randn(n, d, device="cuda", generator=g)).contiguous()


def run(x, n_clusters):
    """-> {stage: seconds}; every stage ends in a device synchronise."""
    from whisper_vits_svc_b200 import retrieval_train as RT
    t = {}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if n_clusters:
        x = torch.from_numpy(RT.compress_features(x, n_clusters)).cuda()
        torch.cuda.synchronize()
        t["compress_s"] = time.perf_counter() - t0
        t0 = time.perf_counter()
    ix = RT.train_ivf_flat(x)
    torch.cuda.synchronize()
    t["train_add_s"] = time.perf_counter() - t0
    return t, ix


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--port-rows", type=int, default=4000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_retrieval_train needs a CUDA device (an H100)")
    import bench
    from oracle import kmeans_oracle as KO
    from whisper_vits_svc_b200 import _lib
    from whisper_vits_svc_b200 import retrieval_train as RT
    lib = _lib.load()
    name, power, clk = gpu_info()
    peaks = bench.load_peaks()
    results = []
    for wl, n, d, n_clusters in WORKLOADS:
        x = features(n, d, seed=n + d)
        run(x, n_clusters)   # warm-up: module loads, workspace sizes
        times, ix = run(x, n_clusters)
        lib.svcb_timing_enable(1)
        run(x, n_clusters)
        torch.cuda.synchronize()
        rep = lib.svcb_timing_report().decode()
        lib.svcb_timing_enable(0)
        rows, table, _ = bench.kernel_families(rep, 1)
        by = {r["name"]: r for r in rows}
        co = by["ivf_coarse_tc"]
        tf = co["flops"] / (co["ms"] * 1e-3) / 1e12
        # CPU arm: one oracle k-means step over port-rows rows against the final centroids, scaled to n rows
        k = ix.nlist
        xs = x[:args.port_rows].cpu().numpy()
        t0 = time.perf_counter()
        KO.kmeans_step(xs, ix.centroids)
        port_s = (time.perf_counter() - t0) * (n if not n_clusters else n_clusters) / args.port_rows
        results.append(dict(
            workload=wl, rows=n, d=d, n_clusters=n_clusters, nlist=k, niter=10,
            **{key: round(v, 3) for key, v in times.items()},
            kernels=table,
            assign_gemm=dict(ms_total=round(co["ms"], 2), tflops_fp32_algorithmic=round(tf, 1),
                             tflops_bf16_executed=round(3 * tf, 1), peak_bf16=peaks["tf_sust"],
                             frac_of_peak=round(3 * tf / peaks["tf_sust"], 3),
                             peak_source=f"{peaks['src']} (MEASURED_PEAKS.json sustained bf16, else the H100 SXM data sheet)"),
            port=dict(kind="port", rows=args.port_rows, step_s_scaled=round(port_s, 2),
                      note="numpy oracle, one k-means step at the final nlist, scaled linearly to the training rows")))
        del x, ix
        torch.cuda.empty_cache()
    print(json.dumps(dict(metric="retrieval_index_build", gpu=name, power_limit_w=power, max_sm_clock_mhz=clk,
                          results=results)))


if __name__ == "__main__":
    main()
