#!/usr/bin/env python
"""Drop-in for the reference's prepare/preprocess_crepe.py (same flags, same walk, same files): the CREPE-full F0 of
every `<wav>/<speaker>/<file>.wav` at a 10 ms hop, saved as `<pit>/<speaker>/<file>.pit.npy` (float32 [1 + n // 160];
zero where the median-filtered periodicity is below 0.5) with crepe/assets/full.pth.  Existing outputs are overwritten,
as in the reference.

Files run on the H100 in ragged batches of up to --batch items.  Frames of all items form one flat batch, so nothing
is padded; the plan still sorts a look-ahead window by length to keep batches even.  -t sets the host threads that read
the wavs.  A file that fails to load, or has fewer than four frames (the periodicity median's reflect padding needs
them, in the reference too), is reported and skipped; if a batch fails on the device, its files are retried one by
one."""
import argparse
import os
import sys

sys.path.append(os.path.dirname(os.path.abspath(__file__)))
import numpy as np

from pitch_inference import MODEL, require_cuda
from whisper_vits_svc_b200 import dataset

MAX_PADDED = 64 * 30 * 16000   # padded samples per device batch: 64 items of 30 s


def pit_jobs(wav_dir, pit_dir):
    """(wav path, output path without .npy) of every file: prepare/preprocess_crepe.py:62-69; under torchrun, this
    rank's share of them (dataset.rank_share)."""
    return dataset.rank_share(dataset.speaker_wavs(wav_dir, pit_dir, ".pit"))


def extract_pitch(jobs, model, threads, batch, max_padded=MAX_PADDED):
    from whisper_vits_svc_b200 import crepe_infer, dataset, hubert_infer

    out = dict(jobs)

    def load(wav):
        audio = hubert_infer.load_audio(wav, crepe_infer.SAMPLE_RATE)
        if crepe_infer.frames_of(audio.shape[0], 160) < 4:
            raise ValueError(f"{audio.shape[0]} samples: fewer than four frames, too short for the periodicity median")
        return audio

    return dataset.run_batched(list(out), load,
                               lambda a: crepe_infer.compute_f0_batch(model, a),
                               lambda wav, pit: np.save(out[wav], pit, allow_pickle=False), threads, batch,
                               size=lambda a: a.shape[0], max_padded=max_padded)


@dataset.rank_main
def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument("-w", "--wav", help="wav", dest="wav", required=True)
    parser.add_argument("-p", "--pit", help="pit", dest="pit", required=True)
    parser.add_argument("-t", "--threads", type=int, default=2, help="host threads reading the wavs (0: all cores)")
    parser.add_argument("--batch", type=int, default=32, help="maximum files per device batch")
    args = parser.parse_args(argv)
    print(args.wav)
    print(args.pit)
    require_cuda()
    from whisper_vits_svc_b200 import crepe_infer

    jobs = pit_jobs(args.wav, args.pit)
    model = crepe_infer.load_model(MODEL, "cuda")
    st = extract_pitch(jobs, model, os.cpu_count() if args.threads == 0 else args.threads, args.batch)
    dataset.report_failed(st["failed"], len(jobs))
    return 0


if __name__ == "__main__":
    sys.exit(main())
