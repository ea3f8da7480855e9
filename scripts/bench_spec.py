#!/usr/bin/env python
"""Linear spectrograms of a training set (svcb_linear_spec_ragged, preprocess_spec.py) on 512 seeded clips of 2 to 28 s
at 32 kHz.  Prints one JSON line: the card and its power limit (read in the same run), then
  device   the kernel time of each batch of the CLI's plan (CUDA events around the call only, after a warm-up pass over
           every batch), per batch and in total, with frames / s, audio seconds / s and the algorithmic FLOP rate;
  cli      preprocess_spec.py end to end on a temporary dataset (wall clock), and the same work split into phases run
           one after another in this process: read (load_wav on -t threads), device (spec_batch: copies and kernel,
           synchronised) and save (torch.save);
  cpu      the oracle (torch.stft on the CPU, as the reference computes) per file on -t threads over a subset of the
           files, scaled to the whole set by samples.

    python scripts/bench_spec.py [-t 8] [--batch 64] [--cpu-files 48]"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

SR, N_CLIPS, SPEAKERS = 32000, 512, 4


def clips(seed=0):
    """512 int16 clips of 2 to 28 s: a few partials with vibrato over a little noise."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(N_CLIPS):
        n = int(rng.uniform(2, 28) * SR)
        t = np.arange(n, dtype=np.float64) / SR
        f0 = rng.uniform(90, 400)
        ph = 2 * np.pi * f0 * (t + 0.02 * np.sin(2 * np.pi * 5.0 * t))
        x = sum(0.25 / k * np.sin(k * ph) for k in (1, 2, 3, 5)) + 0.02 * rng.standard_normal(n)
        out.append((np.clip(x, -1, 1) * 32767).astype(np.int16))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("-t", "--threads", type=int, default=8)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--cpu-files", type=int, default=48)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_spec needs a CUDA device (an H100)")
    import ctypes
    from scipy.io import wavfile
    from bench_retrieval import gpu_info
    from oracle import spec_oracle as SO
    from whisper_vits_svc_b200 import _lib, dataset, hparams, spectrogram as SP
    import preprocess_spec as CLI
    name, power = gpu_info()
    hp = hparams.load_hparams(os.path.join(ROOT, "configs", "base.yaml"))
    pcm = clips()
    audio = [x.astype(np.float32) / np.float32(32768) for x in pcm]
    total_samples = sum(x.shape[0] for x in audio)
    total_frames = sum(SP.frames(x.shape[0]) for x in audio)
    audio_s = total_samples / SR
    plan = dataset.plan_window([x.shape[0] for x in audio], args.batch, CLI.MAX_PADDED)

    # ---- device: the kernel alone, per batch of the plan
    batches = []
    for g in plan:
        so = np.cumsum([0] + [audio[i].shape[0] for i in g])
        frames = sum(SP.frames(audio[i].shape[0]) for i in g)
        flat = torch.from_numpy(np.concatenate([audio[i] for i in g])).cuda()
        out = torch.empty(SP.BINS * frames, device="cuda")
        batches.append((flat, out, (ctypes.c_int64 * len(so))(*[int(v) for v in so]), len(g), frames))

    def run(b):
        flat, out, offs, n, _ = b
        _lib.call("linear_spec_ragged", flat.data_ptr(), offs, n, out.data_ptr(), None, 0)

    for b in batches:
        run(b)
    torch.cuda.synchronize()
    ms = []
    for b in batches:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run(b)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    dev_s = sum(ms) / 1e3
    flop = 4.0 * SP.N_FFT * SP.BINS * total_frames   # re and im FMAs per (sample, bin), bin 512 included
    device = dict(batches=len(batches), ms_per_batch_mean=round(float(np.mean(ms)), 3), ms_per_batch_max=round(max(ms), 3),
                  ms_total=round(sum(ms), 2), frames_per_s=round(total_frames / dev_s), audio_s_per_s=round(audio_s / dev_s),
                  tflops_fp32_algorithmic=round(flop / dev_s / 1e12, 2))
    del batches
    torch.cuda.empty_cache()

    # ---- cli: end to end, then phase by phase
    with tempfile.TemporaryDirectory() as tmp:
        for i, x in enumerate(pcm):
            d = os.path.join(tmp, "wav", f"spk{i % SPEAKERS}")
            os.makedirs(d, exist_ok=True)
            wavfile.write(os.path.join(d, f"{i:03d}.wav"), SR, x)
        os.makedirs(os.path.join(tmp, "configs"))
        with open(os.path.join(ROOT, "configs", "base.yaml")) as f, open(os.path.join(tmp, "configs", "base.yaml"), "w") as g:
            g.write(f.read())
        t0 = time.perf_counter()
        r = subprocess.run([sys.executable, os.path.join(ROOT, "preprocess_spec.py"), "-w", "wav", "-s", "spe", "-t",
                            str(args.threads), "--batch", str(args.batch)], cwd=tmp, capture_output=True, text=True)
        cli_s = time.perf_counter() - t0
        if r.returncode != 0:
            raise SystemExit(r.stderr[-3000:])
        spe_bytes = sum(os.path.getsize(os.path.join(dp, f)) for dp, _, fs in os.walk(os.path.join(tmp, "spe")) for f in fs)
        shutil.rmtree(os.path.join(tmp, "spe"))
        cwd = os.getcwd()
        os.chdir(tmp)   # the reference's walk takes paths relative to the working directory
        jobs = [(os.path.join(tmp, w), os.path.join(tmp, p)) for w, p in CLI.spec_jobs("wav", "spe")]
        os.chdir(cwd)
        t0 = time.perf_counter()
        with ThreadPoolExecutor(args.threads) as pool:
            loaded = list(pool.map(lambda j: SP.load_wav(j[0], hp), jobs))
        t1 = time.perf_counter()
        specs = [None] * len(jobs)
        for g in dataset.plan_window([x.shape[0] for x in loaded], args.batch, CLI.MAX_PADDED):
            for i, s in zip(g, SP.spec_batch([loaded[i] for i in g], hp)):
                specs[i] = s
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        for (_, p), s in zip(jobs, specs):
            torch.save(s.clone(), p)
        t3 = time.perf_counter()
        cli = dict(end_to_end_s=round(cli_s, 2), files_per_s=round(N_CLIPS / cli_s, 1), audio_s_per_s=round(audio_s / cli_s),
                   output_mb=round(spe_bytes / 1e6), phases_s=dict(read=round(t1 - t0, 2), device=round(t2 - t1, 2),
                                                                    save=round(t3 - t2, 2)))
        del specs

        # ---- cpu: the oracle per file on the same threads, over a subset
        sub = jobs[:: max(1, len(jobs) // args.cpu_files)][:args.cpu_files]
        sub_samples = sum(wavfile.read(w)[1].shape[0] for w, _ in sub)
        t0 = time.perf_counter()
        with ThreadPoolExecutor(args.threads) as pool:
            list(pool.map(lambda j: SO.compute_spec(j[0]), sub))
        cpu_sub = time.perf_counter() - t0
    cpu = dict(kind=f"oracle (torch.stft on the CPU) per file, {args.threads} threads, torch intra-op threads "
                    f"{torch.get_num_threads()}", files=len(sub), seconds=round(cpu_sub, 2),
               scaled_to_all_s=round(cpu_sub * total_samples / sub_samples, 1))
    print(json.dumps(dict(metric="linear_spectrogram", gpu=name, power_limit_w=power, clips=N_CLIPS,
                          audio_s=round(audio_s, 1), frames=total_frames, device=device, cli=cli, cpu=cpu)))


if __name__ == "__main__":
    main()
