#!/usr/bin/env python
"""Drop-in for the reference's svc_train_retrieval.py (same flags, same directory layout, same files): for each
speaker a hubert and then a whisper IVF-Flat index, ./data_svc/indexes/<speaker>/<prefix>{hubert,whisper}.index, built
from the *.npy files under ./data_svc/{hubert,whisper}/<speaker>/.  `svc_inference.py --enable-retrieval` reads them.

The k-means and the list assignment run on the H100 (whisper-vits-svc_b200/retrieval_train.py); faiss and
scikit-learn are not needed.  Differences, by design: feature sets above --compress-features-after rows are compressed
to --n-clusters centres by device Lloyd k-means rather than MiniBatchKMeans, so --n-parallel (which only sized
MiniBatchKMeans' batches) is accepted and ignored; random draws come from numpy with faiss's seed, not faiss's
generator; feature files and speakers are taken in sorted order, so the indexes are reproducible."""
import argparse
import logging
import multiprocessing
import os
import sys
from pathlib import Path

sys.path.append(os.path.dirname(os.path.abspath(__file__)))
import torch

from whisper_vits_svc_b200 import retrieval_train

logger = logging.getLogger(__name__)


def get_speaker_list(base_path: Path):
    speakers_path = base_path / "waves-16k"
    if not speakers_path.exists():
        raise FileNotFoundError(f"path {speakers_path} does not exists")
    return sorted(speaker_dir.name for speaker_dir in speakers_path.iterdir() if speaker_dir.is_dir())


def create_indexes_path(base_path: Path) -> Path:
    indexes_path = base_path / "indexes"
    logger.info("create indexes folder %s", indexes_path)
    indexes_path.mkdir(exist_ok=True)
    return indexes_path


def create_index(feature_name: str, prefix: str, speaker: str, base_path: Path, indexes_path: Path,
                 compress_features_after: int, n_clusters: int) -> None:
    features_path = base_path / feature_name / speaker
    if not features_path.exists():
        raise ValueError(f'features not found by path {features_path}')
    index_path = indexes_path / speaker
    index_path.mkdir(exist_ok=True)
    index_filepath = index_path / f"{prefix}{feature_name}.index"
    logger.debug('index will be save to %s', index_filepath)
    retrieval_train.train_index(features_path, index_filepath, compress_features_after, n_clusters)


def main() -> None:
    arg_parser = argparse.ArgumentParser("crate faiss indexes for feature retrieval")
    arg_parser.add_argument("--debug", action="store_true")
    arg_parser.add_argument("--prefix", default='', help="add prefix to index filename")
    arg_parser.add_argument('--speakers', nargs="+",
                            help="speaker names to create an index. By default all speakers are from data_svc")
    arg_parser.add_argument("--compress-features-after", type=int, default=200_000,
                            help="If the number of features is greater than the value compress "
                                 "feature vectors using k-means on the device.")
    arg_parser.add_argument("--n-clusters", type=int, default=10_000,
                            help="Number of centroids to which features will be compressed")
    arg_parser.add_argument("--n-parallel", type=int, default=multiprocessing.cpu_count() - 1,
                            help="accepted for compatibility and ignored: the compression runs on the GPU")
    args = arg_parser.parse_args()

    logging.basicConfig(level=logging.DEBUG if args.debug else logging.INFO)
    if not torch.cuda.is_available():
        raise SystemExit("this build has no CPU path: a CUDA (sm_90a) device is required")

    base_path = Path(".").absolute() / "data_svc"
    speakers = args.speakers if args.speakers else get_speaker_list(base_path)
    logger.info("got %s speakers: %s", len(speakers), speakers)
    indexes_path = create_indexes_path(base_path)

    for speaker in speakers:
        for feature_name in ("hubert", "whisper"):
            logger.info("create %s index for speaker %s", feature_name, speaker)
            create_index(feature_name, args.prefix, speaker, base_path, indexes_path, args.compress_features_after,
                         args.n_clusters)

    logger.info("done!")


if __name__ == '__main__':
    main()
