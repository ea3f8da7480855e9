#!/usr/bin/env python
"""Drop-in for the reference's prepare/preprocess_trim.py (same flags, same walk, same files): every
`<in>/<speaker>/<file>.wav` with its silences cut out by pydub's split_on_silence rules (windows of 200 ms at -45 dBFS,
200 ms kept around each sound), written as 16-bit PCM mono at its own rate to `<out>/<speaker>/<file>.wav`; existing
outputs are overwritten.

Files run on the H100 in ragged batches of up to --batch items; -t sets the host threads that read the wavs.  The
device makes the silence decision of every window; the ranges, slicing and writing are host work.  A file whose windows
are all silent prints the reference's two lines (`list index out of range` and the input path) and writes nothing,
as the reference does.  A file that is not 16-bit PCM mono, or cannot be read, is reported on stderr and skipped, and
the count of such failures goes to stderr.  Speakers and files run in sorted order, and no progress bar is drawn
(DESIGN.md §8)."""
import argparse
import os
import sys

sys.path.append(os.path.dirname(os.path.abspath(__file__)))
from whisper_vits_svc_b200 import dataset

MAX_PADDED = 64 * 30 * 48000   # samples per device batch, as the other preprocess CLIs plan them


def trim_jobs(in_dir, out_dir):
    """(wav path, output path) of every file: prepare/preprocess_trim.py's walk, in sorted order; under torchrun, this
    rank's share of them (dataset.rank_share)."""
    return dataset.rank_share(dataset.speaker_wavs(in_dir, out_dir, ".wav"))


def save_trimmed(wav, out_path, x, rate, flags):
    """trim_silence's host half for one file given its flags: write the kept samples, or print the reference's two
    lines when no chunk is left."""
    from whisper_vits_svc_b200 import trim
    pcm = trim.trim(x, rate, flags)
    if pcm is None:
        print("list index out of range")   # str() of the IndexError audio_chunks[0] raises
        print(f"./{wav}")
        return
    trim.write_wav(out_path, pcm, rate)


def trim_files(jobs, threads, batch, max_padded=MAX_PADDED, device="cuda"):
    from whisper_vits_svc_b200 import dataset, trim

    out = dict(jobs)

    def run(items):
        flags = trim.trim_batch([x for x, _ in items], [r for _, r in items], device)
        return [(x, r, f) for (x, r), f in zip(items, flags)]

    def save(wav, res):
        save_trimmed(wav, out[wav], *res)

    return dataset.run_batched(list(out), trim.load, run, save, threads, batch, size=lambda p: p[0].shape[0],
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
    jobs = trim_jobs(args.inPath, args.outPath)
    threads = os.cpu_count() // 2 + 1 if args.thread_count == 0 else args.thread_count
    st = trim_files(jobs, threads, args.batch)
    dataset.report_failed(st["failed"], len(jobs))
    return 0


if __name__ == "__main__":
    sys.exit(main())
