#!/usr/bin/env python
"""Drop-in for the reference's prepare/preprocess_a.py (same flags, same walk, same files): every
`<wav>/<speaker>/<file>.wav` resampled to -s (16000 or 32000), scaled to a peak of 0.6 x 32767 and written as 16-bit
PCM to `<out>/<speaker>/<file>.wav`; existing outputs are overwritten.

Files run on the H100 in ragged batches of up to --batch items; -t sets the host threads that read the wavs.  Files of
one batch may have different rates: each rate is one device call.  The resampler is scipy's resample_poly filter
(DESIGN.md §8), not librosa's soxr.  A file that is unreadable, has no samples, has non-finite samples or is silent is
reported and skipped, where the reference stops or writes noise; if a batch fails on the device, its files are retried
one by one."""
import argparse
import os
import sys

sys.path.append(os.path.dirname(os.path.abspath(__file__)))
from whisper_vits_svc_b200 import dataset

MAX_PADDED = 64 * 30 * 48000   # padded input samples per device batch: 64 clips of 30 s at 48 kHz, about 0.8 GB


def resample_jobs(wav_dir, out_dir):
    """(wav path, output path) of every file: prepare/preprocess_a.py's walk, in sorted order; under torchrun, this
    rank's share of them (dataset.rank_share)."""
    return dataset.rank_share(dataset.speaker_wavs(wav_dir, out_dir, ".wav"))


def load_clip(path):
    """(samples, rate) of a file the device can take; ValueError for an empty, non-finite or silent one."""
    from whisper_vits_svc_b200 import resample
    x, rate = resample.load(path)
    if not x.any():
        raise ValueError("silent: every sample is 0")
    return x, rate


def resample_files(jobs, sr, threads, batch, max_padded=MAX_PADDED, device="cuda"):
    from scipy.io import wavfile
    from whisper_vits_svc_b200 import dataset, resample

    out = dict(jobs)

    def run(items):
        res = [None] * len(items)
        for rate in sorted({r for _, r in items}):
            idx = [i for i, (_, r) in enumerate(items) if r == rate]
            pcm, peak = resample.pcm16_batch([items[i][0] for i in idx], rate, sr, device)
            for i, p, m in zip(idx, pcm, peak):
                res[i] = (p, m)
        return res

    def save(wav, r):
        pcm, peak = r
        if peak == 0:
            raise ValueError("silent after resampling")
        wavfile.write(out[wav], sr, pcm)

    return dataset.run_batched(list(out), load_clip, run, save, threads, batch, size=lambda p: p[0].shape[0],
                               max_padded=max_padded)


@dataset.rank_main
def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument("-w", "--wav", help="wav", dest="wav", required=True)
    parser.add_argument("-o", "--out", help="out", dest="out", required=True)
    parser.add_argument("-s", "--sr", help="sample rate", dest="sr", type=int, required=True)
    parser.add_argument("-t", "--thread_count", help="thread count to process, set 0 to use all cpu cores",
                        dest="thread_count", type=int, default=1)
    parser.add_argument("--batch", type=int, default=64, help="maximum files per device batch")
    args = parser.parse_args(argv)
    print(args.wav)
    print(args.out)
    print(args.sr)
    os.makedirs(args.out, exist_ok=True)
    if args.sr not in (16000, 32000):
        print(f"-s must be 16000 or 32000, not {args.sr}", file=sys.stderr)
        return 1
    from whisper_vits_svc_b200 import resample

    jobs = resample_jobs(args.wav, args.out)
    threads = os.cpu_count() // 2 + 1 if args.thread_count == 0 else args.thread_count
    try:
        st = resample_files(jobs, args.sr, threads, args.batch)
    finally:
        resample.release_filters()
    dataset.report_failed(st["failed"], len(jobs))
    return 0


if __name__ == "__main__":
    sys.exit(main())
