#!/usr/bin/env python
"""Drop-in for the reference's svc_inference_batch.py (same flags; outputs ./_svc_out/<name>.wav).

The reference loads Whisper once, writes a .ppg.npy per file and then starts one
`python svc_inference.py` subprocess per file (svc_inference_batch.py:34-43), re-loading the SVC
checkpoint and re-spawning the HuBERT / pitch extractors every time.  Here the model is loaded
once per GPU, files are sharded across the ranks of a `torchrun` launch (one process per GPU, one
NCCL broadcast of the packed weights, no collective on the data path), and per rank the chunks of ALL its
files are sorted by length and run as full ragged device batches (hostio.BatchEngine) while host threads read
features and write WAVs.

Features are read from --feat (default: the wav folder) as `<stem>.ppg.npy`, `<stem>.vec.npy` and `<stem>.pit.csv`.
Those that are missing are extracted in-process into ./_svc_out/<name>.{ppg.npy,vec.npy,pit.csv}, one model load per
rank and only if some file needs it: first the F0 by CREPE-full (crepe/assets/full.pth, as pitch_inference.py writes it)
in ragged device batches of whole files, then the PPG by Whisper and the units by HuBERT-Soft, file by file.  A
`.pit.csv` in --feat, such as a hand-edited F0, is used as it is and never overwritten.  A file whose features cannot
be made or read is reported and counted as failed, the other files are still converted, and the exit code is 1; the
reference ignores its subprocesses' exit codes and silently produces nothing for such a file.

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

from pitch_inference import MODEL as CREPE_MODEL
from preprocess_crepe import MAX_PADDED
from whisper_vits_svc_b200 import dataset, hostio, hparams, models, shard

out_path = "./_svc_out"


def feature_path(feat: str, name: str, ext: str) -> str:
    """Where the features of wav `name` are read: `<feat>/<stem><ext>` if that file exists, else
    `./_svc_out/<name><ext>`, where the extraction passes write them."""
    given = os.path.join(feat, name[:-4] + ext)
    return given if os.path.isfile(given) else os.path.join(out_path, name + ext)


def missing_pitch(waves, mine, feat: str):
    """The files of `mine` (indices into `waves`) whose F0 must be extracted: those without `<feat>/<stem>.pit.csv`."""
    return [i for i in mine if not os.path.isfile(os.path.join(feat, waves[i][:-4] + ".pit.csv"))]


def extract_pitch(model, wavs, csvs, noises=None, dithers=None, threads: int = 4, batch: int = 32):
    """`crepe_infer.pred_pit(model, wavs[k], csvs[k])` for every k, in ragged device batches of whole files
    (`dataset.run_batched`, as preprocess_crepe.py runs them).  `noises[k]` / `dithers[k]` are file k's random draws
    (drawn per file when left out).  Returns the indices k that failed, each reported on stderr."""
    from whisper_vits_svc_b200 import crepe_infer, hubert_infer
    index = {w: k for k, w in enumerate(wavs)}
    saved = set()

    def run(items):
        ks = [k for k, _ in items]
        return crepe_infer.compute_f0_sing_batch(model, [a for _, a in items],
                                                 None if noises is None else [noises[k] for k in ks],
                                                 None if dithers is None else [dithers[k] for k in ks])

    def save(wav, f0):
        hostio.save_csv_pitch(f0, csvs[index[wav]])
        saved.add(index[wav])

    dataset.run_batched(list(wavs), lambda w: (index[w], hubert_infer.load_audio(w, crepe_infer.SAMPLE_RATE)), run, save,
                        threads, batch, size=lambda item: item[1].shape[0], max_padded=MAX_PADDED)
    return [k for k in range(len(wavs)) if k not in saved]


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
    no_pitch = set()

    def load(i):
        """Features of one utterance (host threads: file reads overlap the device batches)."""
        name = waves[i]
        if i in no_pitch:
            raise RuntimeError("F0 extraction failed")
        ppg, vec, pit = hostio.prepare_features(*(feature_path(feat, name, e) for e in (".ppg.npy", ".vec.npy", ".pit.csv")),
                                                args.shift)
        return name, spk, pit, ppg, vec

    # F0 pass for files that have no pitch file (one CREPE load per rank; whole files in ragged device batches)
    bare = missing_pitch(waves, mine, feat)
    if bare:
        from whisper_vits_svc_b200 import crepe_infer
        try:
            crepe = crepe_infer.load_model(CREPE_MODEL, device)
        except Exception as e:
            print(f"[rank {rank}] F0 extraction FAILED ({len(bare)} files): {e}")
            no_pitch.update(bare)
        else:
            lost = extract_pitch(crepe, [os.path.join(wave_path, waves[i]) for i in bare],
                                 [os.path.join(out_path, waves[i] + ".pit.csv") for i in bare])
            no_pitch.update(bare[k] for k in lost)
            del crepe                   # (its device weights are freed before Whisper large-v2 loads)

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
