#!/usr/bin/env python
"""Benchmark of svc_validate.py's work: scoring K trainer checkpoints by validation/mel_loss on the device.

Checkpoints are seeded and full size, in the trainer's layout (model_g, model_d, optim_g, optim_d, step, epoch,
hp_str): model_g holds the 903 SynthesizerInfer entries plus the SynthesizerTrn-only entries, and the discriminator and
AdamW states have the reference's sizes (constants below, counted once from vits/models.py:SynthesizerTrn and
vits_decoder/discriminator.py:Discriminator at configs/base.yaml), about 640 MB per file.  Two validation sets: the
10-item valid.txt that preprocess_train.py writes and a larger list of --items items, both of 1 to 4 s.

Per set: the time to read and upload it; per checkpoint, phase by phase with a device synchronise between phases: load
and pack on the host, upload, device inference, mel and loss; the end-to-end time of the pipelined CLI path
(Scorer.score_paths, which loads the next checkpoint while the device scores the current one); the CPU oracle's time
for one checkpoint on the small set; the peak device memory; torch.load with and without mmap=True.  The results are
printed as one JSON line at the end, and also written to --out when it is given."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

# float counts of the reference's trainer checkpoint at configs/base.yaml
TRN_ONLY = 9_504_640      # SynthesizerTrn state entries that SynthesizerInfer lacks (enc_q, emb_g, speaker_classifier)
TRN_PARAMS = 29_508_084   # SynthesizerTrn parameters (AdamW keeps exp_avg and exp_avg_sq of each)
DISC_PARAMS = 23_460_708  # Discriminator parameters (its whole state dict)


def trainer_checkpoint(path, hp, seed):
    from whisper_vits_svc_b200 import synth
    g = torch.Generator().manual_seed(seed)
    sd = synth.svc_state_dict(hp, seed)
    sd["enc_q.flat"] = torch.randn(TRN_ONLY, generator=g)
    adam = lambda n: {"state": {0: {"step": torch.tensor(100.0), "exp_avg": torch.randn(n, generator=g),
                                    "exp_avg_sq": torch.rand(n, generator=g)}}, "param_groups": [{"lr": 5e-5}]}
    torch.save({"model_g": sd, "model_d": {"flat": torch.randn(DISC_PARAMS, generator=g)}, "optim_g": adam(TRN_PARAMS),
                "optim_d": adam(DISC_PARAMS), "step": 100 * seed, "epoch": seed, "hp_str": ""}, path)


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"unavailable: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ckpts", type=int, default=4)
    ap.add_argument("--items", type=int, default=200)
    ap.add_argument("--out", default=None, help="also write the results to this JSON file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_validate needs a CUDA device")
    from oracle import validation_oracle as V
    from whisper_vits_svc_b200 import validation

    hp = V.load_hp()
    res = {"gpu": gpu_info(), "ckpts": args.ckpts}
    rng = np.random.default_rng(0)
    with tempfile.TemporaryDirectory() as tmp:
        t = time.perf_counter()
        paths = []
        for k in range(args.ckpts):
            p = os.path.join(tmp, f"sovits5.0_{k:04d}.pt")
            trainer_checkpoint(p, hp, 100 + k)
            paths.append(p)
        res["ckpt_bytes"] = os.path.getsize(paths[0])
        res["write_ckpts_s"] = time.perf_counter() - t
        loads = {}
        for mm in (False, True, False, True):   # torch.load alone, then with model_g read as load_svc_model reads it
            t = time.perf_counter()
            ck = torch.load(paths[1 % len(paths)], map_location="cpu", weights_only=False, mmap=mm)
            loads.setdefault(f"torch_load_mmap_{mm}_s", []).append(time.perf_counter() - t)
            _ = [v.clone() for v in ck["model_g"].values()]
            loads.setdefault(f"torch_load_mmap_{mm}_read_model_g_s", []).append(time.perf_counter() - t)
            del ck, _
        res.update(loads)
        sets = {"valid10": rng.integers(101, 400, 10), f"list{args.items}": rng.integers(101, 400, args.items)}
        scorer = validation.Scorer(hp, "cuda")
        try:
            for name, frames in sets.items():
                files = V.write_dataset(os.path.join(tmp, name), hp, frames=tuple(int(f) for f in frames), seed=1)
                r = {"items": len(frames), "audio_s": float(np.sum(frames)) / 100.0}
                torch.cuda.synchronize()
                t = time.perf_counter()
                vset = validation.load_set(hp, files, 1234, int(hp.train.batch_size), "cuda")
                torch.cuda.synchronize()
                r["load_set_s"] = time.perf_counter() - t
                r["batches"] = len(vset.batches)
                # warm-up: one full checkpoint
                scorer.install(validation.prepare_checkpoint(paths[0], scorer.staging, scorer.defaults))
                scorer.score_installed(vset)
                torch.cuda.reset_peak_memory_stats()
                per = []
                for p in paths:
                    t0 = time.perf_counter()
                    prep = validation.prepare_checkpoint(p, scorer.staging, scorer.defaults)
                    t1 = time.perf_counter()
                    scorer.install(prep)
                    torch.cuda.synchronize()
                    t2 = time.perf_counter()
                    tm = {}
                    loss = scorer.score_installed(vset, timings=tm)
                    t3 = time.perf_counter()
                    per.append({"load_pack_s": t1 - t0, "upload_s": t2 - t1, "infer_s": tm["infer"], "mel_s": tm["mel"],
                                "total_s": t3 - t0, "mel_loss": loss})
                r["serial"] = per
                r["peak_mem_bytes"] = torch.cuda.max_memory_allocated()
                out = []
                torch.cuda.synchronize()
                t = time.perf_counter()
                scorer.score_paths(paths, vset, lambda p, loss, err: out.append(loss))
                torch.cuda.synchronize()
                r["pipelined_s"] = time.perf_counter() - t
                r["pipelined_per_ckpt_s"] = r["pipelined_s"] / len(paths)
                r["pipelined_equals_serial"] = out == [x["mel_loss"] for x in per]
                if name == "valid10":
                    from whisper_vits_svc_b200 import hostio, models
                    m = models.SynthesizerInfer(513, 25, hp)
                    hostio.load_svc_model(paths[0], m)
                    sd = {k: v.clone() for k, v in m.state_dict().items()}
                    t = time.perf_counter()
                    batches, n = V.read_batches(files, hp, 1234, int(hp.train.batch_size))
                    loss, _, _ = V.validate(sd, hp, batches, n, V.cpu_draws(1), V.basis32(hp))
                    r["cpu_oracle_one_ckpt_s"] = time.perf_counter() - t
                    r["cpu_threads"] = torch.get_num_threads()
                res[name] = r
                print(json.dumps({name: r}), flush=True)
        finally:
            scorer.close()
    res["gpu_after"] = gpu_info()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
