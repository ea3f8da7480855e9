#!/usr/bin/env python
"""Drop-in for the reference's prepare/preprocess_speaker_ave.py (same arguments, same files): the mean of each
speaker's embeddings, `<dataset_speaker>/<speaker>/*.npy`, saved as `<dataset_singer>/<speaker>.spk.npy`, the timbre
file `svc_inference.py --spk` takes.

Speakers and files are taken in os.listdir order, and the sum is the reference's float32 arithmetic,
`0 + e1 + e2 + ...` then `/ count`, so the file is byte-equal to the reference's.  A speaker without any .npy is
skipped.  Entries of `dataset_speaker` that are not directories are skipped (the reference raises on them).  The
reference's `rewrite_timbre_code` branch is hard-coded off and is not restated."""
import argparse
import os
import sys

import numpy as np


def speaker_average(speaker_dir):
    """The mean embedding of the .npy files in `speaker_dir`; None when it has none."""
    subfile_num = 0
    speaker_ave = 0
    for file in os.listdir(speaker_dir):
        if not file.endswith(".npy"):
            continue
        speaker_ave = speaker_ave + np.load(os.path.join(speaker_dir, file)).astype(np.float32)
        subfile_num = subfile_num + 1
    if subfile_num == 0:
        return None
    return speaker_ave / subfile_num


def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument("dataset_speaker", type=str)
    parser.add_argument("dataset_singer", type=str)
    args = parser.parse_args(argv)
    os.makedirs(args.dataset_singer, exist_ok=True)
    for speaker in os.listdir(args.dataset_speaker):
        speaker_dir = os.path.join(args.dataset_speaker, speaker)
        if not os.path.isdir(speaker_dir):
            continue
        speaker_ave = speaker_average(speaker_dir)
        if speaker_ave is not None:
            np.save(os.path.join(args.dataset_singer, f"{speaker}.spk.npy"), speaker_ave, allow_pickle=False)
    return 0


if __name__ == "__main__":
    sys.exit(main())
