#!/usr/bin/env python
"""The batch converter's engine (hostio.BatchEngine, svc_inference_batch.py) with equal-length batches against ragged
batches (svcb_infer_ragged), on a seeded synthetic checkpoint at precision 3 with the features in memory.  Workloads:
  mixed  512 utterances of 200-2800 frames (2-28 s), the length mix of the preprocessing benchmarks;
  equal  256 utterances of exactly 1000 frames (bench_config5.py's mix), where both modes make the same batches.
Each mode runs --repeats times per workload, the modes alternating, after one warm-up run of each.  Per mode: device
seconds (CUDA events around the model calls), wall seconds of the engine loop (NSF sources, staging, copies, slicing),
device calls, mean chunks per call, the share of padded frames in the calls, and audio seconds converted per wall
second (median over the repeats; min and max beside).  Then, with the draws silenced (eps = 0, zero source noise), both
modes convert every utterance of the workload once more and the waveforms are compared with np.array_equal.  Prints one
JSON line with the card and its power limit, read in the same run.

    python scripts/bench_ragged_infer.py [--repeats 3] [--max-batch 32]"""
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

HOP, SR = 320, 32000


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits",
                        "-i", str(torch.cuda.current_device())], capture_output=True, text=True, check=True).stdout
    name, pl = [s.strip() for s in q.strip().splitlines()[0].split(",")]
    return name, float(pl)


def workload(hp, lengths, seed):
    """(key, spk, pit, ppg, vec) CPU jobs; the feature rows are views into one seeded pool (their values do not
    change the work)."""
    rs = np.random.RandomState(seed)
    pool = max(lengths) + 4096
    ppg = torch.from_numpy(rs.randn(pool, hp.vits.ppg_dim).astype(np.float32))
    vec = torch.from_numpy(rs.randn(pool, hp.vits.vec_dim).astype(np.float32))
    pit = torch.from_numpy(rs.randint(100, 501, size=pool).astype(np.float32))
    pit[::7] = 0
    spk = torch.from_numpy((rs.randn(hp.vits.spk_dim) * 0.05).astype(np.float32))
    jobs = []
    for i, n in enumerate(lengths):
        o = int(rs.randint(0, pool - n))
        jobs.append((f"utt{i:04d}", spk, pit[o:o + n], ppg[o:o + n], vec[o:o + n]))
    return jobs


class Quiet:
    """The model with its random draws silenced, so that both modes are deterministic."""

    def __init__(self, m, C):
        self.m, self.C = m, C

    def pitch2source(self, f0, **kw):
        B, T = f0.shape
        return self.m.pitch2source(f0, rand_ini=torch.zeros(B, 11), noise=torch.zeros(B, T * HOP, 11))

    def inference(self, ppg, vec, pit, spk, ppg_l, source, eps=None):
        return self.m.inference(ppg, vec, pit, spk, ppg_l, source, eps=torch.zeros(ppg.shape[0], self.C, ppg.shape[1]))

    def inference_ragged(self, ppg, vec, pit, spk, n_frames, source, eps=None):
        return self.m.inference_ragged(ppg, vec, pit, spk, n_frames, source,
                                       eps=torch.zeros(ppg.shape[0], self.C, ppg.shape[1]))


def run(model, hp, jobs, ragged, max_batch):
    from whisper_vits_svc_b200 import hostio
    eng = hostio.BatchEngine(model, hp, "cuda", max_batch=max_batch, ragged=ragged)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = dict(eng.run(iter(jobs)))
    torch.cuda.synchronize()
    return eng, time.perf_counter() - t0, out


def padded_share(lengths, max_batch, ragged):
    """Padded frames over all frames of the device calls of the engine's plans (windows of 128 utterances)."""
    from whisper_vits_svc_b200 import hostio
    real = padded = 0
    for w0 in range(0, len(lengths), 128):
        lw = lengths[w0:w0 + 128]
        chunks, batches = (hostio.BatchEngine.plan_ragged if ragged else hostio.BatchEngine.plan)(lw, HOP, max_batch)
        for b in batches:
            n = [chunks[j][2] - chunks[j][1] for j in b]
            real += sum(n)
            padded += len(n) * max(n)
    return (padded - real) / padded


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--max-batch", type=int, default=32)
    args = ap.parse_args()
    from whisper_vits_svc_b200 import hostio, hparams, models, synth
    assert torch.cuda.is_available(), "bench_ragged_infer needs a CUDA device"
    name, power = gpu_info()
    hp = hparams.load_hparams(os.path.join(ROOT, "configs", "base.yaml"))
    model = models.SynthesizerInfer(513, 25, hp, precision=3)
    model.load_state_dict(synth.svc_state_dict(hp, 1234))
    model.to("cuda")
    rs = np.random.RandomState(0)
    loads = {"mixed": [int(v) for v in rs.randint(200, 2801, size=512)], "equal": [1000] * 256}
    res = {"metric": "ragged_conversion_batches", "gpu": name, "power_limit_w": power, "max_batch": args.max_batch,
           "precision": 3, "repeats": args.repeats}
    for wname, lengths in loads.items():
        jobs = workload(hp, lengths, 1 + len(lengths))
        audio_s = sum(n * HOP - 1 for n in lengths) / SR
        for ragged in (False, True):       # warm-up: kernels, allocator, pinned staging
            run(model, hp, jobs[:64], ragged, args.max_batch)
        rec = {"utterances": len(lengths), "frames": sum(lengths), "audio_seconds": round(audio_s, 1)}
        for ragged in (False, True):
            rec["ragged" if ragged else "equal_length"] = {"device_s": [], "wall_s": []}
        for _ in range(args.repeats):
            for ragged in (False, True):
                eng, wall, _ = run(model, hp, jobs, ragged, args.max_batch)
                r = rec["ragged" if ragged else "equal_length"]
                r["device_s"].append(eng.device_seconds)
                r["wall_s"].append(wall)
                r["device_calls"] = eng.batches
        n_chunks = sum(len(hostio.chunk_plan(n, HOP)) for n in lengths)
        for ragged in (False, True):
            r = rec["ragged" if ragged else "equal_length"]
            dev, wall = sorted(r.pop("device_s")), sorted(r.pop("wall_s"))
            r.update(device_s_median=round(float(np.median(dev)), 3), device_s_min=round(dev[0], 3), device_s_max=round(dev[-1], 3),
                     wall_s_median=round(float(np.median(wall)), 3), wall_s_min=round(wall[0], 3), wall_s_max=round(wall[-1], 3),
                     chunks=n_chunks, mean_batch=round(n_chunks / r["device_calls"], 2),
                     padded_frame_share=round(padded_share(lengths, args.max_batch, ragged), 4),
                     audio_s_per_wall_s=round(audio_s / float(np.median(wall)), 1))
        rec["wall_speedup"] = round(rec["equal_length"]["wall_s_median"] / rec["ragged"]["wall_s_median"], 3)
        rec["device_speedup"] = round(rec["equal_length"]["device_s_median"] / rec["ragged"]["device_s_median"], 3)
        q = Quiet(model, hp.vits.inter_channels)
        _, _, a = run(q, hp, jobs, False, args.max_batch)
        _, _, b = run(q, hp, jobs, True, args.max_batch)
        rec["silenced_waveforms_equal"] = bool(a.keys() == b.keys() and all(np.array_equal(a[k], b[k]) for k in a))
        res[wname] = rec
    print(json.dumps(res), flush=True)
    assert all(res[w]["silenced_waveforms_equal"] for w in loads), "the two modes' waveforms differ"


if __name__ == "__main__":
    main()
