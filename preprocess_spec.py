#!/usr/bin/env python
"""Drop-in for the reference's prepare/preprocess_spec.py (same flags, same walk, same files): the linear spectrogram
of every `<wav>/<speaker>/<file>.wav` (32 kHz mono), saved with torch.save as `<spe>/<speaker>/<file>.pt`, a float32
[513, samples // 320] tensor.  The config is ./configs/base.yaml, read from the working directory as the reference
does; existing outputs are overwritten.

Files run on the H100 in ragged batches of up to --batch items; -t sets the host threads that read the wavs.  A file
that fails (not at the config's sampling rate, multi-channel, 352 samples or fewer, unreadable) is reported and
skipped, where the reference stops; if a batch fails on the device, its files are retried one by one."""
import argparse
import os
import sys

sys.path.append(os.path.dirname(os.path.abspath(__file__)))
import torch

from whisper_vits_svc_b200 import dataset

MAX_PADDED = 64 * 30 * 32000   # padded samples per device batch: 64 clips of 30 s, about 0.6 GB of audio and spectra


def spec_jobs(wav_dir, spe_dir):
    """(wav path, output path) of every file: prepare/preprocess_spec.py's walk; under torchrun, this rank's share of
    them (dataset.rank_share)."""
    return dataset.rank_share(dataset.speaker_wavs(wav_dir, spe_dir, ".pt"))


def compute_specs(jobs, hp, threads, batch, max_padded=MAX_PADDED, device="cuda"):
    from whisper_vits_svc_b200 import dataset, spectrogram

    spectrogram.check_hparams(hp)
    out = dict(jobs)

    def save(wav, spec):
        torch.save(spec.clone(), out[wav])   # the batch's results share one buffer

    return dataset.run_batched(list(out), lambda w: spectrogram.load_wav(w, hp),
                               lambda a: spectrogram.spec_batch(a, hp, device), save, threads, batch,
                               size=len, max_padded=max_padded)


@dataset.rank_main
def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument("-w", "--wav", help="wav", dest="wav", required=True)
    parser.add_argument("-s", "--spe", help="spe", dest="spe", required=True)
    parser.add_argument("-t", "--thread_count", help="thread count to process, set 0 to use all cpu cores",
                        dest="thread_count", type=int, default=1)
    parser.add_argument("--batch", type=int, default=64, help="maximum files per device batch")
    args = parser.parse_args(argv)
    print(args.wav)
    print(args.spe)
    from whisper_vits_svc_b200 import hparams, spectrogram

    hp = hparams.load_hparams("./configs/base.yaml")
    try:
        spectrogram.check_hparams(hp)
    except ValueError as e:
        print(e, file=sys.stderr)
        return 1
    jobs = spec_jobs(args.wav, args.spe)
    threads = os.cpu_count() // 2 + 1 if args.thread_count == 0 else args.thread_count
    st = compute_specs(jobs, hp, threads, args.batch)
    dataset.report_failed(st["failed"], len(jobs))
    return 0


if __name__ == "__main__":
    sys.exit(main())
