#!/usr/bin/env python
"""Drop-in for the reference's prepare/preprocess_ppg.py (same flags, same walk, same files): the Whisper PPG of every
`<wav>/<speaker>/<file>.wav`, saved as `<ppg>/<speaker>/<file>.ppg.npy` (float32 [rows, 1280]) with
whisper_pretrain/large-v2.pt.  Files whose output already exists are skipped, as in the reference.

Each file is read at 16 kHz, pad_or_trim-ed (trimmed to 30 s, zero-padded to at least 15 s), turned into its log-mel
with no noise and encoded; its first min(samples // 320, positions) rows are kept.  Files run on the H100 in ragged
batches of up to --batch items, planned over a sorted look-ahead window so that padding stays small; -t sets the host
threads that read the wavs.  A file that fails (unreadable, or shorter than 320 samples) is reported and skipped; if a
batch fails on the device, its files are retried one by one."""
import argparse
import os
import sys

sys.path.append(os.path.dirname(os.path.abspath(__file__)))
import numpy as np

from whisper_vits_svc_b200 import dataset

MAX_PADDED = 32 * 30 * 16000   # padded samples per device batch: 32 items of 30 s, about 1.4 GB of large-v2 workspace


def ppg_jobs(wav_dir, ppg_dir):
    """(wav path, output path without .npy) of every file still to do: prepare/preprocess_ppg.py:57-69.  Under
    torchrun the full walk is shared before the done files are dropped, so that other ranks' new outputs cannot
    change this rank's share."""
    return [(w, p) for w, p in dataset.rank_share(dataset.speaker_wavs(wav_dir, ppg_dir, ".ppg"))
            if not os.path.isfile(f"{p}.npy")]


def extract_ppgs(jobs, whisper, threads, batch, max_padded=MAX_PADDED):
    from whisper_vits_svc_b200 import dataset, whisper_infer

    out = dict(jobs)

    def load(wav):
        audio = whisper_infer.load_audio(wav)
        if audio.shape[0] < 320:
            raise ValueError(f"{audio.shape[0]} samples: shorter than one PPG row (320)")
        return audio

    def save(wav, ppg):
        np.save(out[wav], ppg, allow_pickle=False)

    return dataset.run_batched(list(out), load, lambda a: whisper_infer.ppg_batch(whisper, a), save, threads, batch,
                               size=lambda a: min(max(a.shape[0], whisper_infer.N_SAMPLES // 2), whisper_infer.N_SAMPLES),
                               max_padded=max_padded)


@dataset.rank_main
def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument("-w", "--wav", help="wav", dest="wav", required=True)
    parser.add_argument("-p", "--ppg", help="ppg", dest="ppg", required=True)
    parser.add_argument("-t", "--threads", type=int, default=2, help="host threads reading the wavs (0: all cores)")
    parser.add_argument("--batch", type=int, default=32, help="maximum files per device batch")
    args = parser.parse_args(argv)
    print(args.wav)
    print(args.ppg)
    from whisper_vits_svc_b200 import whisper_infer

    jobs = ppg_jobs(args.wav, args.ppg)
    whisper = whisper_infer.load_model(os.path.join("whisper_pretrain", "large-v2.pt"), "cuda")
    st = extract_ppgs(jobs, whisper, os.cpu_count() if args.threads == 0 else args.threads, args.batch)
    print(f"padding overhead: {st['padded'] / max(st['samples'], 1):.3f} (padded samples / samples)")
    dataset.report_failed(st["failed"], len(jobs))
    return 0


if __name__ == "__main__":
    sys.exit(main())
