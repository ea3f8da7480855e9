#!/usr/bin/env python
"""Drop-in for the reference's prepare/preprocess_cdc.py (same flags, same walk, same files): every
`<in>/<speaker>/<file>.wav` with its two lowest STFT bins (1024 / 256 Hann) cut out, written as 16-bit PCM mono at its
own rate to `<out>/<speaker>/<file>.wav`, 256 * (n // 256) samples long; existing outputs are overwritten.

Files run on the H100 in ragged batches of up to --batch items; -t sets the host threads that read the wavs.  The
device computes the round trip in fp64 where the reference uses float32 FFTs, so a sample may differ from the
reference's by 1 LSB (DESIGN.md §8).  A file that fails is reported and skipped, the run goes on, and the count of
failures goes to stderr; the reference stops the run or writes a malformed file.  The failures are a file of 512
samples or fewer (torch.stft's reflect pad fails), more than one channel (the reference writes it transposed), non-finite
samples and an unreadable file.  If a batch fails on the device, its files are retried one by one.  Speakers and files
run in sorted order."""
import argparse
import os
import sys

sys.path.append(os.path.dirname(os.path.abspath(__file__)))
from whisper_vits_svc_b200 import dataset

MAX_PADDED = 64 * 30 * 48000   # padded input samples per device batch: 64 clips of 30 s at 48 kHz, about 0.5 GB


def cdc_jobs(in_dir, out_dir):
    """(wav path, output path) of every file: prepare/preprocess_cdc.py's walk, in sorted order; under torchrun, this
    rank's share of them (dataset.rank_share)."""
    return dataset.rank_share(dataset.speaker_wavs(in_dir, out_dir, ".wav"))


def cut_files(jobs, threads, batch, max_padded=MAX_PADDED, device="cuda"):
    from scipy.io import wavfile
    from whisper_vits_svc_b200 import cdc, dataset

    out = dict(jobs)

    def run(items):
        return list(zip(cdc.cdc_batch([x for x, _ in items], device), [r for _, r in items]))

    def save(wav, r):
        pcm, rate = r
        wavfile.write(out[wav], rate, pcm)

    return dataset.run_batched(list(out), cdc.load, run, save, threads, batch, size=lambda p: p[0].shape[0],
                               max_padded=max_padded)


@dataset.rank_main
def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument("-i", help="input path", dest="inPath", required=True)
    parser.add_argument("-o", help="output path", dest="outPath", required=True)
    parser.add_argument("-t", "--thread_count", help="thread count to process, set 0 to use all cpu cores",
                        dest="thread_count", type=int, default=1)
    parser.add_argument("--batch", type=int, default=64, help="maximum files per device batch")
    args = parser.parse_args(argv)
    print(args.inPath)
    print(args.outPath)
    os.makedirs(args.outPath, exist_ok=True)
    jobs = cdc_jobs(args.inPath, args.outPath)
    threads = os.cpu_count() // 2 + 1 if args.thread_count == 0 else args.thread_count
    st = cut_files(jobs, threads, args.batch)
    dataset.report_failed(st["failed"], len(jobs))
    return 0


if __name__ == "__main__":
    sys.exit(main())
