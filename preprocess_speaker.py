#!/usr/bin/env python
"""Drop-in for the reference's prepare/preprocess_speaker.py (same arguments, same files): one 256-d speaker
embedding per wav of `dataset_path` (speaker sub-directories and top-level wavs), written under `output_path` as
`<name>.spk.npy`, with speaker_pretrain/best_model.pth.tar and speaker_pretrain/config.json.

Files run on the H100 in ragged batches of up to --batch utterances; -t sets the host threads that read, trim and
normalise the wavs, at most two batches ahead of the device.  A file that fails is reported and skipped; if a
batch fails on the device, its files are retried one by one so only the failing file is lost."""
import argparse
import os
import sys
from argparse import RawTextHelpFormatter

sys.path.append(os.path.dirname(os.path.abspath(__file__)))
import numpy as np

from whisper_vits_svc_b200 import dataset


def get_spk_wavs(dataset_path, output_path):
    """prepare/preprocess_speaker.py:18-29 (creates the output directories as the reference does); under torchrun,
    this rank's share of the files."""
    wav_files = []
    os.makedirs(f"./{output_path}", exist_ok=True)
    for spks in os.listdir(dataset_path):
        if os.path.isdir(f"./{dataset_path}/{spks}"):
            os.makedirs(f"./{output_path}/{spks}", exist_ok=True)
            for file in os.listdir(f"./{dataset_path}/{spks}"):
                if file.endswith(".wav"):
                    wav_files.append(f"./{dataset_path}/{spks}/{file}")
        elif spks.endswith(".wav"):
            wav_files.append(f"./{dataset_path}/{spks}")
    return dataset.rank_share(wav_files, path=lambda w: w)


def embed_path(wav_file, dataset_path, output_path):
    """prepare/preprocess_speaker.py:43-45 (np.save appends .npy)."""
    return wav_file.replace(dataset_path, output_path).replace(".wav", ".spk")


def extract_speaker_embeddings(wav_files, dataset_path, output_path, model, concurrency, batch=32):
    """Embed every file in device batches; returns the number of files that failed (each is reported and skipped).
    The loader threads run at most two batches ahead of the device, so host memory stays bounded."""

    def save(f, e):
        np.save(embed_path(f, dataset_path, output_path), e, allow_pickle=False)

    return dataset.run_batched(wav_files, model.load_wav, lambda wavs: model.embed(wavs).cpu().numpy().astype(np.float32),
                               save, concurrency, batch)["failed"]


@dataset.rank_main
def main(argv=None):
    parser = argparse.ArgumentParser(description="""Compute embedding vectors for each wav file in a dataset.""",
                                     formatter_class=RawTextHelpFormatter)
    parser.add_argument("dataset_path", type=str, help="Path to dataset waves.")
    parser.add_argument("output_path", type=str, help="path for output speaker/speaker_wavs.npy.")
    parser.add_argument("--use_cuda", type=bool, help="flag to set cuda.", default=True)
    parser.add_argument("-t", "--thread_count", help="thread count to process, set 0 to use all cpu cores",
                        dest="thread_count", type=int, default=1)
    parser.add_argument("--batch", type=int, default=32, help="utterances per device batch")
    args = parser.parse_args(argv)
    from whisper_vits_svc_b200 import speaker_infer

    model = speaker_infer.load_model(os.path.join("speaker_pretrain", "best_model.pth.tar"),
                                     os.path.join("speaker_pretrain", "config.json"), "cuda")
    wav_files = get_spk_wavs(args.dataset_path, args.output_path)
    process_num = os.cpu_count() if args.thread_count == 0 else args.thread_count
    n_failed = extract_speaker_embeddings(wav_files, args.dataset_path, args.output_path, model, process_num, args.batch)
    dataset.report_failed(n_failed, len(wav_files))
    return 0


if __name__ == "__main__":
    sys.exit(main())
