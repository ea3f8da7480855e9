#!/usr/bin/env python
"""Drop-in for the reference's prepare/preprocess_hubert.py (same flags, same walk, same files): the HuBERT-Soft units
of every `<wav>/<speaker>/<file>.wav`, saved as `<vec>/<speaker>/<file>.vec.npy` (float32 [frames, 256], squeezed as
the reference does, so a one-frame file is saved as [256]) with hubert_pretrain/hubert-soft-0d54a1f4.pt.  Existing
outputs are overwritten, as in the reference.

Each whole file is one item (no 20 s chunking).  Files run on the H100 in ragged batches of up to --batch items,
planned over a sorted look-ahead window so that padding stays small; -t sets the host threads that read the wavs.  A
file that fails (unreadable, or too short for one frame) is reported and skipped; if a batch fails on the device, its
files are retried one by one."""
import argparse
import os
import sys

sys.path.append(os.path.dirname(os.path.abspath(__file__)))
import numpy as np

from whisper_vits_svc_b200 import dataset

MAX_PADDED = 32 * 20 * 16000   # padded samples per device batch: 32 items of 20 s, about 9 GB of workspace


def vec_jobs(wav_dir, vec_dir):
    """(wav path, output path without .npy) of every file: prepare/preprocess_hubert.py:51-58; under torchrun, this
    rank's share of them (dataset.rank_share)."""
    return dataset.rank_share(dataset.speaker_wavs(wav_dir, vec_dir, ".vec"))


def extract_vecs(jobs, hubert, threads, batch, max_padded=MAX_PADDED):
    from whisper_vits_svc_b200 import dataset, hubert_infer

    out = dict(jobs)

    def load(wav):
        audio = hubert_infer.load_audio(wav, hubert_infer.SAMPLE_RATE)
        if hubert.frames(audio.shape[0]) < 1:
            raise ValueError(f"{audio.shape[0]} samples: too short for one HuBERT frame")
        return audio

    def save(wav, units):
        np.save(out[wav], units.squeeze(), allow_pickle=False)

    return dataset.run_batched(list(out), load, lambda a: hubert_infer.units_batch(hubert, a), save, threads, batch,
                               size=lambda a: a.shape[0], max_padded=max_padded)


@dataset.rank_main
def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument("-w", "--wav", help="wav", dest="wav", required=True)
    parser.add_argument("-v", "--vec", help="vec", dest="vec", required=True)
    parser.add_argument("-t", "--threads", type=int, default=2, help="host threads reading the wavs (0: all cores)")
    parser.add_argument("--batch", type=int, default=32, help="maximum files per device batch")
    args = parser.parse_args(argv)
    print(args.wav)
    print(args.vec)
    from whisper_vits_svc_b200 import hubert_infer

    jobs = vec_jobs(args.wav, args.vec)
    hubert = hubert_infer.load_model(os.path.join("hubert_pretrain", "hubert-soft-0d54a1f4.pt"), "cuda")
    st = extract_vecs(jobs, hubert, os.cpu_count() if args.threads == 0 else args.threads, args.batch)
    print(f"padding overhead: {st['padded'] / max(st['samples'], 1):.3f} (padded samples / samples)")
    dataset.report_failed(st["failed"], len(jobs))
    return 0


if __name__ == "__main__":
    sys.exit(main())
