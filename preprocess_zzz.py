#!/usr/bin/env python
"""The loader check of the reference's prepare/preprocess_zzz.py, restated without omegaconf: every item of
files/valid.txt goes through the trainer's data path (vits/data_utils.py) as one epoch would take it, so that a
missing, misaligned or wrongly sampled feature file fails here and not in the first training epoch.

- `TextAudioSpeakerSet`: the filter (items with a missing file are dropped; the useful length is
  `len(pitch) - 1`, items under 1 s are dropped and those over 4 s capped), then every item read once: the
  sampling-rate assertion, vec and ppg repeated twice, the `len - 2` trims and the random crop;
- `bucket_batches`: the DistributedBucketSampler's batches for one replica at epoch 0 (batch 4, boundaries
  150, 300, 450), each read and zero-padded by `collate` (TextAudioSpeakerCollate).

The config is ./configs/base.yaml, read from the working directory as the reference does.  Python's `random` and
torch's generator are called as the reference calls them, so under the same seeds the items and batches are equal
to the reference's.  It raises where the reference raises and prints the reference's `----------N----------` line;
it prints no progress bar."""
import argparse
import os
import random
import sys

sys.path.append(os.path.dirname(os.path.abspath(__file__)))
import numpy as np
import torch

BATCH_SIZE = 4
BOUNDARIES = [150, 300, 450]


def load_filepaths(filename, split="|"):
    with open(filename, encoding="utf-8") as f:
        return [line.strip().split(split) for line in f]


class TextAudioSpeakerSet:
    """vits/data_utils.py:TextAudioSpeakerSet: the filtered items of a file list and their useful lengths."""

    def __init__(self, filename, hparams):
        self.items = load_filepaths(filename)
        self.max_wav_value = hparams.max_wav_value
        self.sampling_rate = hparams.sampling_rate
        self.segment_size = hparams.segment_size
        self.hop_length = hparams.hop_length
        self._filter()
        print(f"----------{len(self.items)}----------")

    def _filter(self):
        lengths = []
        items_new = []
        items_min = int(self.segment_size / self.hop_length * 4)   # 1 s
        items_max = int(self.segment_size / self.hop_length * 16)  # 4 s
        for wavpath, spec, pitch, vec, ppg, spk in self.items:
            if not all(os.path.isfile(p) for p in (wavpath, spec, pitch, vec, ppg, spk)):
                continue
            usel = int(np.load(pitch).shape[0] - 1)   # useful length
            if usel < items_min:
                continue
            if usel >= items_max:
                usel = items_max
            items_new.append([wavpath, spec, pitch, vec, ppg, spk, usel])
            lengths.append(usel)
        self.items = items_new
        self.lengths = lengths

    def read_wav(self, filename):
        from scipy.io.wavfile import read
        sampling_rate, data = read(filename)
        assert sampling_rate == self.sampling_rate, f"error: this sample rate of {filename} is {sampling_rate}"
        return (torch.FloatTensor(data.astype(np.float32)) / self.max_wav_value).unsqueeze(0)

    def __len__(self):
        return len(self.items)

    def __getitem__(self, idx):
        """(spe, wav, ppg, vec, pit, spk) of item idx, aligned and, past its useful length, randomly cropped."""
        wav, spe, pit, vec, ppg, spk, use = self.items[idx]
        wav = self.read_wav(wav)
        spe = torch.load(spe)
        pit = torch.FloatTensor(np.load(pit))
        vec = torch.FloatTensor(np.repeat(np.load(vec), 2, 0))   # 320 PPG -> 160 * 2
        ppg = torch.FloatTensor(np.repeat(np.load(ppg), 2, 0))   # 320 PPG -> 160 * 2
        spk = torch.FloatTensor(np.load(spk))

        len_min = min(pit.size()[0], vec.size()[0] - 2, ppg.size()[0] - 2)   # - 2: for safe
        len_wav = len_min * self.hop_length
        pit = pit[:len_min]
        vec = vec[:len_min, :]
        ppg = ppg[:len_min, :]
        spe = spe[:, :len_min]
        wav = wav[:, :len_wav]
        if len_min > use:
            frame_start = random.randint(0, ppg.size(0) - use - 1)
            frame_end = frame_start + use
            pit = pit[frame_start:frame_end]
            vec = vec[frame_start:frame_end, :]
            ppg = ppg[frame_start:frame_end, :]
            spe = spe[:, frame_start:frame_end]
            wav = wav[:, frame_start * self.hop_length:frame_end * self.hop_length]
        return spe, wav, ppg, vec, pit, spk


def bucket_batches(lengths, batch_size=BATCH_SIZE, boundaries=BOUNDARIES, epoch=0):
    """vits/data_utils.py:DistributedBucketSampler's batches (one replica, shuffled): indices grouped by the length
    bucket `boundaries[i] < length <= boundaries[i + 1]` (others are dropped), each bucket padded by repeating itself to
    whole batches, the batches shuffled by a generator seeded with `epoch`."""
    buckets = [[] for _ in range(len(boundaries) - 1)]
    for i, length in enumerate(lengths):
        for b in range(len(boundaries) - 1):
            if boundaries[b] < length <= boundaries[b + 1]:
                buckets[b].append(i)
                break
    for i in range(len(buckets) - 1, 0, -1):   # empty buckets go, except the first
        if len(buckets[i]) == 0:
            buckets.pop(i)
    num_samples_per_bucket = [len(b) + (batch_size - len(b) % batch_size) % batch_size for b in buckets]

    g = torch.Generator()
    g.manual_seed(epoch)
    indices = [torch.randperm(len(bucket), generator=g).tolist() for bucket in buckets]
    batches = []
    for bucket, ids_bucket, num_samples_bucket in zip(buckets, indices, num_samples_per_bucket):
        len_bucket = len(bucket)
        if len_bucket == 0:
            continue
        rem = num_samples_bucket - len_bucket   # extra samples to make it evenly divisible
        ids_bucket = ids_bucket + ids_bucket * (rem // len_bucket) + ids_bucket[:rem % len_bucket]
        for j in range(len(ids_bucket) // batch_size):
            batches.append([bucket[idx] for idx in ids_bucket[j * batch_size:(j + 1) * batch_size]])
    batch_ids = torch.randperm(len(batches), generator=g).tolist()
    batches = [batches[i] for i in batch_ids]
    assert len(batches) * batch_size == sum(num_samples_per_bucket)
    return batches


def collate(batch):
    """vits/data_utils.py:TextAudioSpeakerCollate: the items zero-padded, longest spectrogram first -> (ppg, ppg_lengths,
    vec, pit, spk, spe, spe_lengths, wav, wav_lengths)."""
    _, ids_sorted_decreasing = torch.sort(torch.LongTensor([x[0].size(1) for x in batch]), dim=0, descending=True)
    B = len(batch)
    max_spe_len = max(x[0].size(1) for x in batch)
    max_wav_len = max(x[1].size(1) for x in batch)
    max_ppg_len = max(x[2].size(0) for x in batch)
    spe_lengths = torch.zeros(B, dtype=torch.long)
    wav_lengths = torch.zeros(B, dtype=torch.long)
    ppg_lengths = torch.zeros(B, dtype=torch.float32)
    spe_padded = torch.zeros(B, batch[0][0].size(0), max_spe_len)
    wav_padded = torch.zeros(B, 1, max_wav_len)
    ppg_padded = torch.zeros(B, max_ppg_len, batch[0][2].size(1))
    vec_padded = torch.zeros(B, max_ppg_len, batch[0][3].size(1))
    pit_padded = torch.zeros(B, max_ppg_len)
    spk = torch.zeros(B, batch[0][5].size(0))
    for i in range(len(ids_sorted_decreasing)):
        spe, wav, ppg, vec, pit, s = batch[ids_sorted_decreasing[i]]
        spe_padded[i, :, :spe.size(1)] = spe
        spe_lengths[i] = spe.size(1)
        wav_padded[i, :, :wav.size(1)] = wav
        wav_lengths[i] = wav.size(1)
        ppg_padded[i, :ppg.size(0), :] = ppg
        ppg_lengths[i] = ppg.size(0)
        vec_padded[i, :vec.size(0), :] = vec
        pit_padded[i, :pit.size(0)] = pit
        spk[i] = s
    return ppg_padded, ppg_lengths, vec_padded, pit_padded, spk, spe_padded, spe_lengths, wav_padded, wav_lengths


def main(argv=None):
    argparse.ArgumentParser(description=__doc__.split("\n\n")[0]).parse_args(argv)
    from whisper_vits_svc_b200 import hparams

    hps = hparams.load_hparams("./configs/base.yaml")
    dataset = TextAudioSpeakerSet("files/valid.txt", hps.data)
    for i in range(len(dataset)):
        dataset[i]
    for batch in bucket_batches(dataset.lengths):
        collate([dataset[i] for i in batch])
    return 0


if __name__ == "__main__":
    sys.exit(main())
