#!/usr/bin/env python
"""Drop-in for the reference's svc_inference_batch.py (same flags; outputs ./_svc_out/<name>.wav).

The reference loads Whisper once, writes a .ppg.npy per file and then starts one
`python svc_inference.py` subprocess per file (svc_inference_batch.py:34-43), re-loading the SVC
checkpoint and re-spawning the HuBERT / pitch extractors every time.  Here the model is loaded
once per GPU, files are sharded across the ranks of a `torchrun` launch (one process per GPU, one
NCCL broadcast of the packed weights, no collective on the data path), and per rank the chunks of ALL its
files are sorted by length and run as full ragged device batches (hostio.BatchEngine) while host threads read
features and write WAVs.  Missing `<name>.ppg.npy` / `<name>.vec.npy` are extracted in-process by the H100 Whisper /
HuBERT-Soft encoders (one model load per rank).  CREPE is outside the H100 hot path (SURVEY.md §8f-4):
`<name>.pit.csv` must sit next to `<name>.wav` (or in --feat); a file without it is reported and skipped — the
reference would silently produce nothing for it either (subprocess exit codes are ignored there).

    python svc_inference_batch.py --config configs/base.yaml --model sovits5.0.pth --wave waves/ --spk singer.npy
    python -m torch.distributed.run --nproc-per-node 8 svc_inference_batch.py ...   # 8 GPUs
"""
import argparse
import os
import sys

sys.path.append(os.path.dirname(os.path.abspath(__file__)))
import numpy as np
import torch
from scipy.io.wavfile import write

from whisper_vits_svc_b200 import hostio, hparams, models, shard

out_path = "./_svc_out"


def main():
    parser = argparse.ArgumentParser()
    parser.add_argument('--config', type=str, required=True, help="yaml file for config.")
    parser.add_argument('--model', type=str, required=True, help="path of model for evaluation")
    parser.add_argument('--wave', type=str, required=True, help="Path of raw audio.")
    parser.add_argument('--spk', type=str, required=True, help="Path of speaker.")
    parser.add_argument('--shift', type=int, default=0, help="Pitch shift key.")
    parser.add_argument('--feat', type=str, default=None, help="dir holding <name>.{ppg,vec}.npy / .pit.csv")
    parser.add_argument('--whisper', type=str, default=os.path.join("whisper_pretrain", "large-v2.pt"))
    parser.add_argument('--hubert', type=str, default=os.path.join("hubert_pretrain", "hubert-soft-0d54a1f4.pt"))
    parser.add_argument('--max-batch', type=int, default=32, help="chunks per device call (chunks of all files, longest first)")
    args = parser.parse_args()
    wave_path = args.wave
    assert os.path.isdir(wave_path), f"{wave_path} is not folder"
    os.makedirs(out_path, exist_ok=True)
    waves = sorted(f for f in os.listdir(wave_path) if f.endswith(".wav"))
    if not torch.cuda.is_available():
        raise SystemExit("this build has no CPU path: a CUDA (sm_90a) device is required")
    rank, local, world = shard.init()
    device = torch.device("cuda", local)
    torch.cuda.set_device(device)
    hp = hparams.load_hparams(args.config)
    model = models.SynthesizerInfer(hp.data.filter_length // 2 + 1, hp.data.segment_size // hp.data.hop_length, hp,
                                    precision=3)
    blob = table = None
    if rank == 0:
        hostio.load_svc_model(args.model, model)
        model.to(device)
        blob, table = model.packed_blob()
    else:
        model.to(device)
    if world > 1:
        blob, table = shard.broadcast_blob(blob, table, device)
        if rank != 0:
            model.install_blob(blob, table)
    sizes = [os.path.getsize(os.path.join(wave_path, f)) for f in waves]
    mine = shard.assign(sizes, world)[rank]
    feat = args.feat or wave_path
    spk = torch.FloatTensor(np.load(args.spk))
    whisper = None
    done, failed = 0, []

    def load(i):
        """Features of one utterance (host threads: file reads overlap the device batches)."""
        name = waves[i]
        stem = os.path.join(feat, name[:-4])
        ppg_p, vec_p, pit_p = stem + ".ppg.npy", stem + ".vec.npy", stem + ".pit.csv"
        if not os.path.isfile(pit_p):
            raise FileNotFoundError(f"{pit_p} missing (the CREPE pitch extractor is out of scope)")
        if not os.path.isfile(ppg_p):
            ppg_p = os.path.join(out_path, name + ".ppg.npy")     # written by the extractor pass below
        if not os.path.isfile(vec_p):
            vec_p = os.path.join(out_path, name + ".vec.npy")
        ppg, vec, pit = hostio.prepare_features(ppg_p, vec_p, pit_p, args.shift)
        return name, spk, pit, ppg, vec

    # PPG pass for files that have none yet (one Whisper load per rank; chunks of a file run as one batch)
    for i in mine:
        name = waves[i]
        if not os.path.isfile(os.path.join(feat, name[:-4] + ".ppg.npy")):
            try:
                from whisper_vits_svc_b200 import whisper_infer
                if whisper is None:
                    whisper = whisper_infer.load_model(args.whisper, device)
                whisper_infer.pred_ppg(whisper, os.path.join(wave_path, name), os.path.join(out_path, name + ".ppg.npy"), device)
            except Exception as e:
                print(f"[rank {rank}] {name}: PPG extraction FAILED {e}")
    del whisper
    hubert = None
    for i in mine:   # the same for the HuBERT-Soft units (svc_inference.py:144-148 of the reference)
        name = waves[i]
        if not os.path.isfile(os.path.join(feat, name[:-4] + ".vec.npy")):
            try:
                from whisper_vits_svc_b200 import hubert_infer
                if hubert is None:
                    hubert = hubert_infer.load_model(args.hubert, device)
                hubert_infer.pred_vec(hubert, os.path.join(wave_path, name), os.path.join(out_path, name + ".vec.npy"))
            except Exception as e:
                print(f"[rank {rank}] {name}: HuBERT extraction FAILED {e}")
    del hubert

    from concurrent.futures import ThreadPoolExecutor
    engine = hostio.BatchEngine(model, hp, device, max_batch=args.max_batch, ragged=True)
    loaders, writers = ThreadPoolExecutor(max_workers=4), ThreadPoolExecutor(max_workers=4)

    def jobs():
        futs = [loaders.submit(load, i) for i in mine]
        for i, f in zip(mine, futs):
            try:
                yield f.result()
            except Exception as e:  # a failed utterance must not stop the shard
                failed.append((waves[i], repr(e)))
                print(f"[rank {rank}] {waves[i]}: FAILED {e}")

    pending = []
    for name, audio in engine.run(jobs()):
        pending.append(writers.submit(write, os.path.join(out_path, name), hp.data.sampling_rate, audio))
        done += 1
    for f in pending:
        f.result()
    loaders.shutdown(); writers.shutdown()
    total = shard.sum_over_ranks(float(done), device)
    if rank == 0:
        print(f"svc_inference_batch: {int(total)}/{len(waves)} files converted on {world} GPU(s)")
    if world > 1:
        shard.barrier()
        torch.distributed.destroy_process_group()
    return 0 if not failed else 1


if __name__ == '__main__':
    sys.exit(main())
