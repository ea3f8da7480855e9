#!/usr/bin/env python
"""Measures converting bare recordings (no `.pit.csv`) with svc_inference_batch.py: seeded synthetic weights (SVC and
CREPE-full) and N synthetic voiced clips of 2 to 28 s at 16 kHz, with `.ppg.npy` / `.vec.npy` given in --feat so that
Whisper large-v2 and HuBERT-Soft are not needed.

1. The batch CLI's F0 pass (`svc_inference_batch.extract_pitch`: ragged device batches of whole files, host loader
   threads) against one `crepe_infer.pred_pit` call per file (what the reference's per-file `pitch/inference.py` does,
   here without its model reload), with one CREPE model and the same per-file random draws.  Both write the same CSVs,
   and the script checks that they are byte-equal.  Wall time after a warm-up pass, the two arms alternated.
2. The whole `svc_inference_batch.py` command line on the bare folder, and on the same folder with the F0 pass's CSVs
   given in --feat: wall time of the process, so model loads and the CUDA start-up are included in both.

The card's name, power limit and maximum SM clock are read in the same run.  Everything is written under a temporary
directory that is removed at the end.  Nothing here changes a device setting."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
from scipy.io import wavfile  # noqa: E402


def voiced(rng, n):
    """A gliding harmonic tone with vibrato and a little noise, int16 at 16 kHz."""
    t = np.arange(n) / 16000
    f0 = rng.uniform(110, 330) * (1 + 0.15 * np.sin(2 * np.pi * 0.3 * t)) + 4 * np.sin(2 * np.pi * 5.5 * t)
    ph = 2 * np.pi * np.cumsum(f0) / 16000
    v = sum((0.5 / k) * np.sin(k * ph + rng.uniform(0, 2 * np.pi)) for k in range(1, 9))
    v += 0.01 * rng.standard_normal(n)
    return np.round(0.5 * v / np.abs(v).max() * 32767).astype(np.int16)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=128)
    ap.add_argument("--repeats", type=int, default=2, help="timed passes of each F0 arm, alternated")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_bare_batch.py measures the device path; there is no CPU path"
    import svc_inference_batch as B
    from whisper_vits_svc_b200 import crepe_infer as C, hparams, synth

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(f"card: {card}", flush=True)
    base = tempfile.mkdtemp(prefix="svcb_bare_")
    try:
        hp = hparams.load_hparams(os.path.join(ROOT, "configs", "base.yaml"))
        crepe_sd = synth.crepe_checkpoint(1234, "full")
        os.makedirs(os.path.join(base, "crepe", "assets"))
        torch.save(crepe_sd, os.path.join(base, "crepe", "assets", "full.pth"))
        torch.save({"model_g": synth.svc_state_dict(hp, 1234)}, os.path.join(base, "g.pth"))
        rng = np.random.default_rng(0)
        np.save(os.path.join(base, "spk.npy"), (rng.standard_normal(hp.vits.spk_dim) * 0.05).astype(np.float32))
        wave_dir, feat = os.path.join(base, "waves"), os.path.join(base, "feat")
        os.makedirs(wave_dir)
        os.makedirs(feat)
        lengths = (rng.uniform(2.0, 28.0, args.clips) * 16000).astype(np.int64)
        names = [f"clip{k:04d}" for k in range(args.clips)]
        for name, n in zip(names, lengths):   # 20 ms feature rows, as pred_ppg / pred_vec write them
            wavfile.write(os.path.join(wave_dir, name + ".wav"), 16000, voiced(rng, int(n)))
            np.save(os.path.join(feat, name + ".ppg.npy"), rng.standard_normal((n // 320, hp.vits.ppg_dim), np.float32))
            np.save(os.path.join(feat, name + ".vec.npy"), rng.standard_normal((n // 320, hp.vits.vec_dim), np.float32))
        audio_s = float(lengths.sum() / 16000)
        out = {"card": card, "clips": args.clips, "audio_s": audio_s}

        # 1. the F0 pass, ragged against one pred_pit per file
        wavs = [os.path.join(wave_dir, name + ".wav") for name in names]
        g = torch.Generator().manual_seed(5)
        noises = [torch.randn(int(n), generator=g) for n in lengths]
        dithers = [(torch.rand(C.frames_of(int(n), 320), generator=g) - 0.5) * 40 for n in lengths]
        ragged_csv = [os.path.join(base, "ragged", name + ".pit.csv") for name in names]
        alone_csv = [os.path.join(base, "alone", name + ".pit.csv") for name in names]
        os.makedirs(os.path.join(base, "ragged"))
        os.makedirs(os.path.join(base, "alone"))
        model = C.CrepeB200(crepe_sd, "cuda", "full")

        def ragged():
            assert B.extract_pitch(model, wavs, ragged_csv, noises, dithers) == []

        def alone():
            for k, wav in enumerate(wavs):
                C.pred_pit(model, wav, alone_csv[k], noises[k], dithers[k])

        times = {"ragged": [], "per_file": []}
        ragged()      # warm-up: module loads, the allocator's pool, the page cache of the wavs
        alone()
        for _ in range(args.repeats):
            for arm, fn in (("ragged", ragged), ("per_file", alone)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                times[arm].append(time.perf_counter() - t0)
        same = all(open(a, "rb").read() == open(b, "rb").read() for a, b in zip(ragged_csv, alone_csv))
        assert same, "the ragged F0 pass and pred_pit per file wrote different CSVs"
        best = {arm: min(ts) for arm, ts in times.items()}
        out["f0_pass"] = {"ragged_s": times["ragged"], "per_file_s": times["per_file"],
                          "ragged_audio_s_per_s": audio_s / best["ragged"], "per_file_audio_s_per_s": audio_s / best["per_file"],
                          "speedup": best["per_file"] / best["ragged"], "csvs_byte_equal": same}
        print(f"F0 pass, {args.clips} clips, {audio_s:.0f} s of audio: ragged {best['ragged']:.2f} s, one pred_pit per file "
              f"{best['per_file']:.2f} s ({out['f0_pass']['speedup']:.2f}x); CSVs byte-equal", flush=True)
        del model

        # 2. the command line end to end, bare and with the F0 given
        cmd = [sys.executable, os.path.join(ROOT, "svc_inference_batch.py"), "--config", os.path.join(ROOT, "configs", "base.yaml"),
               "--model", "g.pth", "--wave", "waves", "--spk", "spk.npy", "--feat", "feat"]

        def cli():
            t0 = time.perf_counter()
            r = subprocess.run(cmd, cwd=base, capture_output=True, text=True)
            wall = time.perf_counter() - t0
            assert r.returncode == 0 and f"{args.clips}/{args.clips} files converted" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
            return wall

        bare = cli()
        extracted = sum(os.path.isfile(os.path.join(base, "_svc_out", name + ".wav.pit.csv")) for name in names)
        assert extracted == args.clips, extracted
        for name in names:
            shutil.copy(os.path.join(base, "_svc_out", name + ".wav.pit.csv"), os.path.join(feat, name + ".pit.csv"))
        given = cli()
        out["cli"] = {"bare_s": bare, "pit_given_s": given, "bare_audio_s_per_s": audio_s / bare,
                      "what_is_timed": "the whole process: interpreter and CUDA start-up, model loads, feature reads, "
                                       "the F0 pass (bare only), the conversion and the WAV writes"}
        print(f"svc_inference_batch.py end to end: bare wavs {bare:.1f} s, F0 given {given:.1f} s", flush=True)
        print(json.dumps(out), flush=True)
    finally:
        shutil.rmtree(base, ignore_errors=True)


if __name__ == "__main__":
    main()
