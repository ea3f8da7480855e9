"""CPU oracle of the trainer's validation score (TEST INFRASTRUCTURE, not product code).

- `mel_filter_bank`: librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax) with its defaults (Slaney mel scale, Slaney
  area normalisation), restated in fp64 from librosa's definition, apart from whisper_infer.mel_filters;
- `mel_spectrogram`: vits_extend/stft.py:TacotronSTFT.mel_spectrogram as torch computes it on the CPU (reflect pad
  352, torch.stft with center=False, sqrt(re^2 + im^2 + 1e-9), mel_basis @ spec, ln(clamp(x, 1e-5)));
- `validate`: vits_extend/validation.py's loop over padded batches, with SynthesizerTrn.infer (vits/models.py:202-208)
  restated on oracle/svc_oracle.py's stages and every random draw an input, the L1 of each batch summed and divided
  by the number of items.

`python oracle/validation_oracle.py` writes tests/golden/validation_synth.npz: a dataset of ITEM_FRAMES items is
regenerated from DATA_SEED by `write_dataset` (wav, spec, pitch, vec, ppg and speaker files and a valid.txt), read
with Python's `random` seeded with CROP_SEED in batches of BATCH, with CPU draws from `cpu_draws(DRAW_SEED)` and the
full-size weights synth.svc_state_dict(hp, WEIGHT_SEED).  Only the results are stored: the real and fake mels of
every batch, the fake audio of the logged items (item 0 of each batch) and mel_loss."""
from __future__ import annotations

import os
import random
import sys
from typing import Dict, List

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import svc_oracle as S  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "validation_synth.npz")
ITEM_FRAMES = (112, 131, 101)   # useful lengths of 1.12, 1.31 and 1.01 s
BATCH = 2
DATA_SEED, CROP_SEED, DRAW_SEED, WEIGHT_SEED = 11, 1234, 7, 1234
N_FFT, HOP, PAD = 1024, 320, 352


def _hz_to_mel(f):
    """Slaney: linear 3 mel per 200 Hz below 1 kHz, then 27 mel per factor 6.4."""
    f = np.asarray(f, np.float64)
    lin = 3.0 * f / 200.0
    return np.where(f >= 1000.0, 15.0 + 27.0 * np.log(np.maximum(f, 1e-300) / 1000.0) / np.log(6.4), lin)


def _mel_to_hz(m):
    m = np.asarray(m, np.float64)
    return np.where(m >= 15.0, 1000.0 * np.exp((m - 15.0) * np.log(6.4) / 27.0), 200.0 * m / 3.0)


def mel_filter_bank(sr, n_fft, n_mels, fmin=0.0, fmax=None) -> np.ndarray:
    """librosa.filters.mel, float64 [n_mels, n_fft // 2 + 1]: triangles between consecutive points of n_mels + 2
    equally spaced mels from fmin to fmax, each scaled by 2 / (its upper edge - its lower edge) in Hz."""
    fmax = sr / 2.0 if fmax is None else fmax
    edges = _mel_to_hz(np.linspace(_hz_to_mel(fmin), _hz_to_mel(fmax), n_mels + 2))
    freqs = np.arange(n_fft // 2 + 1) * (sr / n_fft)
    w = np.zeros((n_mels, freqs.size))
    for m in range(n_mels):
        a, c, b = edges[m], edges[m + 1], edges[m + 2]
        up = (freqs - a) / (c - a)
        down = (b - freqs) / (b - c)
        w[m] = np.clip(np.minimum(up, down), 0.0, None) * (2.0 / (b - a))
    return w


def basis32(hp) -> torch.Tensor:
    d = hp.data
    return torch.from_numpy(mel_filter_bank(d.sampling_rate, d.filter_length, d.mel_channels, d.mel_fmin,
                                            d.mel_fmax)).float()


def mel_spectrogram(y: torch.Tensor, basis: torch.Tensor) -> torch.Tensor:
    """TacotronSTFT.mel_spectrogram of y [B, L] in [-1, 1] -> [B, n_mels, L // 320]."""
    assert float(y.min()) >= -1 and float(y.max()) <= 1
    y = F.pad(y.unsqueeze(1), (PAD, PAD), mode="reflect").squeeze(1)
    spec = torch.stft(y, N_FFT, hop_length=HOP, win_length=N_FFT, window=torch.hann_window(N_FFT), center=False,
                      normalized=False, onesided=True, return_complex=True)
    spec = torch.view_as_real(spec)
    spec = torch.sqrt(spec.pow(2).sum(-1) + 1e-9)
    return torch.log(torch.clamp(torch.matmul(basis, spec), min=1e-5))


LOG_CLIP = float(np.float32(np.log(np.float64(np.float32(1e-5)))))   # ln(1e-5f), correctly rounded to fp32


# --------------------------------------------------------------------------- dataset and draws
def write_dataset(root: str, hp, frames=ITEM_FRAMES, seed: int = DATA_SEED) -> str:
    """Synthetic items of the trainer's file layout under root; -> the path of root/valid.txt.  Item i has pitch of
    frames[i] + 1 frames (useful length frames[i]), ppg and vec of frames[i] // 2 + 1 rows at 1280 / 256 (so the `len -
    2` trim leaves frames[i] frames), a spectrogram of frames[i] columns, a 256-d speaker and an int16 32 kHz wav of
    (frames[i] + 1) * 320 samples: a harmonic tone following the pitch (0 marks unvoiced) in noise, with a stretch of
    digital silence."""
    from scipy.io import wavfile
    rng = np.random.default_rng(seed)
    os.makedirs(root, exist_ok=True)
    lines = []
    for i, n in enumerate(frames):
        p = os.path.join(root, f"item{i}")
        f0 = rng.uniform(110, 330) * (1 + 0.05 * np.sin(np.arange(n + 1) / 9.0))
        f0[n // 3:n // 3 + 8] = 0.0
        t = np.arange((n + 1) * HOP) / 32000.0
        ph = 2 * np.pi * np.cumsum(np.repeat(f0, HOP)) / 32000.0
        x = sum(0.3 / k * np.sin(k * ph) for k in (1, 2, 3)) * (np.repeat(f0, HOP) > 0) + 0.02 * rng.standard_normal(t.size)
        x[HOP * (n // 2):HOP * (n // 2) + 3 * N_FFT] = 0.0
        wavfile.write(p + ".wav", 32000, np.round(np.clip(x, -1, 1) * 32000).astype(np.int16))
        torch.save(torch.zeros(513, n), p + ".spec.pt")
        np.save(p + ".pit.npy", f0.astype(np.float64))
        rows = n // 2 + 1
        np.save(p + ".vec.npy", rng.standard_normal((rows, hp.vits.vec_dim)).astype(np.float32))
        np.save(p + ".ppg.npy", rng.standard_normal((rows, hp.vits.ppg_dim)).astype(np.float32))
        np.save(p + ".spk.npy", (0.05 * rng.standard_normal(hp.vits.spk_dim)).astype(np.float32))
        lines.append("|".join(p + s for s in (".wav", ".spec.pt", ".pit.npy", ".vec.npy", ".ppg.npy", ".spk.npy")))
    path = os.path.join(root, "valid.txt")
    with open(path, "w", encoding="utf-8") as f:
        f.write("\n".join(lines) + "\n")
    return path


def cpu_draws(seed: int = DRAW_SEED):
    """A draw function for whisper_vits_svc_b200.validation.load_set: a CPU generator seeded with `seed`, drawn batch
    by batch in the reference's order, so that the oracle and the device can share the draws."""
    g = torch.Generator().manual_seed(int(seed))

    def draw(bi, shapes):
        return {k: (torch.randn if kind == "randn" else torch.rand)(shape, generator=g) for k, (shape, kind) in shapes.items()}
    return draw


def read_batches(files: str, hp, seed: int, batch: int) -> List[tuple]:
    """create_dataloader_eval's batches, read with preprocess_zzz (the reference's TextAudioSpeakerSet and
    TextAudioSpeakerCollate, restated) after random.seed(seed): a list of collated tuples."""
    import preprocess_zzz
    random.seed(int(seed))
    ds = preprocess_zzz.TextAudioSpeakerSet(files, hp.data)
    return [preprocess_zzz.collate([ds[i] for i in range(i0, min(i0 + batch, len(ds)))])
            for i0 in range(0, len(ds), batch)], len(ds)


# --------------------------------------------------------------------------- the loop
def infer_trn(sd, hp, ppg, vec, pit, spk, ppg_l, d: Dict[str, torch.Tensor]) -> torch.Tensor:
    """SynthesizerTrn.infer (vits/models.py:202-208) with its draws as inputs: ppg + ppg_noise * 1e-4, the prior with
    eps, the reverse flow, then Generator.forward = x + z_noise, NSF source (rand_ini, noise) and Generator.inference
    over all T frames."""
    with torch.no_grad():
        ppg = ppg + d["ppg_noise"] * 0.0001
        z_p, mask = S.prior_encoder(sd, ppg, ppg_l, vec, pit, d["eps"])
        z = S.flow_reverse(sd, z_p, mask, spk)
        x = z * mask + d["z_noise"]
        source = S.pitch2source(sd, hp, pit, d["rand_ini"], d["noise"])
        return S.generator(sd, hp, spk, x, source)


def draw_shapes(B, T, hp):
    C = hp.vits.inter_channels
    return {"ppg_noise": ((B, T, hp.vits.ppg_dim), "randn"), "eps": ((B, C, T), "randn"),
            "z_noise": ((B, C, T), "randn"), "rand_ini": ((B, 11), "rand"), "noise": ((B, T * HOP, 11), "randn")}


def validate(sd, hp, batches, n_items, draw, basis):
    """vits_extend/validation.py: -> (mel_loss, [(mel_real, mel_fake)], {idx: (real, fake) of item 0}) for batches
    idx < hp.log.num_audio."""
    total, mels, logged = 0.0, [], {}
    for idx, (ppg, ppg_l, vec, pit, spk, _, _, audio, _) in enumerate(batches):
        B, T = pit.shape
        d = draw(idx, draw_shapes(B, T, hp))
        fake = infer_trn(sd, hp, ppg, vec, pit, spk, ppg_l, d)[:, :, :audio.size(2)]
        mel_fake = mel_spectrogram(fake.squeeze(1), basis)
        mel_real = mel_spectrogram(audio.squeeze(1), basis)
        total += F.l1_loss(mel_fake, mel_real).item()
        mels.append((mel_real, mel_fake))
        if idx < hp.log.num_audio:
            logged[idx] = (audio[0][0].numpy(), fake[0][0].numpy())
    return total / n_items, mels, logged


def load_hp():
    from whisper_vits_svc_b200 import hparams
    return hparams.load_hparams(os.path.join(ROOT, "configs", "base.yaml"))


def fixture_run(tmp: str):
    """The fixture's run in tmp: -> (hp, valid.txt path, weights, mel_loss, mels, logged)."""
    from whisper_vits_svc_b200 import synth
    hp = load_hp()
    files = write_dataset(tmp, hp)
    sd = synth.svc_state_dict(hp, WEIGHT_SEED)
    batches, n = read_batches(files, hp, CROP_SEED, BATCH)
    loss, mels, logged = validate(sd, hp, batches, n, cpu_draws(DRAW_SEED), basis32(hp))
    return hp, files, sd, loss, mels, logged


def load_golden() -> dict:
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def main():
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        hp, _, _, loss, mels, logged = fixture_run(tmp)
    out = {"mel_loss": np.float64(loss)}
    for i, (r, f) in enumerate(mels):
        out[f"mel_real_{i}"] = r.numpy()
        out[f"mel_fake_{i}"] = f.numpy()
    for i, (_, f) in logged.items():
        out[f"fake_audio_{i}"] = f
    np.savez_compressed(GOLDEN, **out)
    print(f"{GOLDEN}: mel_loss {loss!r}, {os.path.getsize(GOLDEN)} bytes")


if __name__ == "__main__":
    main()
