#!/usr/bin/env python
"""pYIN F0 of a whole dataset: pyin_f0.compute_f0_pyin (libf0's probabilistic YIN with an HMM voicing model, at a 10
ms hop over 50-1000 Hz; the wrapper and its parameters are this project's choice, no reference command calls pyin) of
every `<wav>/<speaker>/<file>.wav`, saved as `<pit>/<speaker>/<file>.pit.npy` (float64 [n // 160 + 1], 0 where
unvoiced, not rounded).  Existing outputs are overwritten.  The flags, walk and printed lines are those of
preprocess_f0_salience.py.

Files run on the H100 in ragged batches of up to --batch items; the plan sorts a look-ahead window by length to keep
batches even.  -t sets the host threads that read the wavs (0: all cores).  Speakers and files are walked in sorted
order.  Audio is read as preprocess_f0.py reads it (.wav only, resample_poly where the file is not at 16 kHz).  A file
that fails to load, or has no samples, is reported and skipped; if a batch fails on the device, its files are retried
one by one."""
import argparse
import os
import sys

sys.path.append(os.path.dirname(os.path.abspath(__file__)))
import numpy as np

from whisper_vits_svc_b200 import dataset

MAX_PADDED = 64 * 30 * 16000   # padded samples per device batch: 64 items of 30 s, about 2.8 GB of workspace


def pit_jobs(wav_dir, pit_dir):
    """(wav path, output path without .npy) of every file; under torchrun, this rank's share of them
    (dataset.rank_share)."""
    return dataset.rank_share(dataset.speaker_wavs(wav_dir, pit_dir, ".pit"))


def load(wav):
    from whisper_vits_svc_b200 import hubert_infer, pyin_f0
    audio = hubert_infer.load_audio(wav, pyin_f0.SAMPLE_RATE)
    if audio.shape[0] < pyin_f0.MIN_SAMPLES:
        raise ValueError("no samples")
    return audio


def extract_f0(jobs, run, threads, batch, max_padded=MAX_PADDED):
    """Write every job's .pit.npy; run(list of clips) -> list of float64 F0 arrays."""

    out = dict(jobs)
    return dataset.run_batched(list(out), load, run,
                               lambda wav, pit: np.save(out[wav], np.asarray(pit, np.float64), allow_pickle=False),
                               threads, batch, size=lambda a: a.shape[0], max_padded=max_padded)


@dataset.rank_main
def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument("-w", "--wav", help="wav", dest="wav", required=True)
    parser.add_argument("-p", "--pit", help="pit", dest="pit", required=True)
    parser.add_argument("-t", "--thread_count", help="thread count to process, set 0 to use all cpu cores",
                        dest="thread_count", type=int, default=1)
    parser.add_argument("--batch", type=int, default=64, help="maximum files per device batch")
    args = parser.parse_args(argv)
    print(args.wav)
    print(args.pit)
    from whisper_vits_svc_b200 import pyin_f0

    jobs = pit_jobs(args.wav, args.pit)
    ex = pyin_f0.Extractor("cuda")
    try:
        st = extract_f0(jobs, ex.f0_batch, os.cpu_count() if args.thread_count == 0 else args.thread_count, args.batch)
    finally:
        ex.close()
    dataset.report_failed(st["failed"], len(jobs))
    return 0


if __name__ == "__main__":
    sys.exit(main())
