#!/usr/bin/env python
"""Salience-based F0 of a whole dataset: pitch/inference.py's compute_f0_salience (libf0's Melodia-style tracker at a
20 ms hop over 45-1760 Hz, every value twice and a moving average over 3) of every `<wav>/<speaker>/<file>.wav`, saved
as `<pit>/<speaker>/<file>.pit.npy` (float64 [2 (n // 320 + 1)], not rounded).  Existing outputs are overwritten.  The
flags, walk and printed lines are those of preprocess_f0_mouth.py.

Files run on the H100 in ragged batches of up to --batch items; the plan sorts a look-ahead window by length to keep
batches even.  -t sets the host threads that read the wavs (0: all cores).  Speakers and files are walked in sorted
order.  Audio is read as preprocess_f0.py reads it (.wav only, resample_poly where the file is not at 16 kHz).  A file
that fails to load, or has fewer than 320 samples (one hop, where the tracker has no phase advance), is reported and
skipped; if a batch fails on the device, its files are retried one by one."""
import argparse
import os
import sys

sys.path.append(os.path.dirname(os.path.abspath(__file__)))
import numpy as np

from whisper_vits_svc_b200 import dataset

MAX_PADDED = 64 * 30 * 16000   # padded samples per device batch: 64 items of 30 s


def pit_jobs(wav_dir, pit_dir):
    """(wav path, output path without .npy) of every file; under torchrun, this rank's share of them
    (dataset.rank_share)."""
    return dataset.rank_share(dataset.speaker_wavs(wav_dir, pit_dir, ".pit"))


def load(wav):
    from whisper_vits_svc_b200 import hubert_infer, salience_f0
    audio = hubert_infer.load_audio(wav, salience_f0.SAMPLE_RATE)
    if audio.shape[0] < salience_f0.MIN_SAMPLES:
        raise ValueError(f"{audio.shape[0]} samples: fewer than {salience_f0.MIN_SAMPLES}, shorter than one hop")
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
    from whisper_vits_svc_b200 import salience_f0

    jobs = pit_jobs(args.wav, args.pit)
    ex = salience_f0.Extractor("cuda")
    try:
        st = extract_f0(jobs, ex.f0_batch, os.cpu_count() if args.thread_count == 0 else args.thread_count, args.batch)
    finally:
        ex.close()
    dataset.report_failed(st["failed"], len(jobs))
    return 0


if __name__ == "__main__":
    sys.exit(main())
