"""CREPE pitch extractor on the H100 path -- host-side mirror of the reference's `crepe.predict` as `pitch/inference.py`
(`compute_f0_sing`) and `prepare/preprocess_crepe.py` (`compute_f0`) call it, behind the C ABI (`svcb_crepe_*`,
csrc/crepe_api.cu).  No CPU fallback: a CUDA (sm_90a) device is required.

Inputs are 16 kHz waveforms.  The two random draws of the reference are arguments: `noise` (the `randn_like(audio)` that
is scaled by 0.001 and added to the audio) and `dither` (cents per frame, `scipy.stats.triang` over +-20).  Left out,
both are drawn on the host the way the reference draws them.  The Viterbi path restarts every 512 frames, as the
reference's `batch_size=512` makes it.  The host keeps the two `crepe.filter` passes over the [frames] vectors.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib, hostio, hubert_infer, pack

SAMPLE_RATE = 16000
WINDOW = 1024
PITCH_BINS = 360
SEGMENT = 512                      # batch_size of both reference callers: frames per Viterbi segment
BN_EPS = 0.0010000000474974513     # crepe/model.py:38
BIN_LO, BIN_HI = 39, 299           # frequency_to_bins(50), frequency_to_bins(1000, ceil): crepe/core.py:597-603
CHANNELS = {"full": [1, 1024, 128, 128, 128, 256, 512], "tiny": [1, 128, 16, 16, 16, 32, 64]}
TAPS = [512, 64, 64, 64, 64, 64]
# csrc/crepe_api.cu: input channels per bulk-copied chunk of conv2 .. conv6, frames per image group, image rows
CONV_CK = [64, 64, 64, 32, 16]
IMAGE_G = [1, 1, 2, 4, 8]
IMAGE_ROWS = [192, 128, 192, 320, 568]


def shapes(capacity: str) -> Dict[str, Tuple[int, ...]]:
    """The state dict of crepe/assets/{full,tiny}.pth (crepe/model.py:14-92)."""
    C = CHANNELS[capacity]
    d: Dict[str, Tuple[int, ...]] = {}
    for i in range(6):
        d[f"conv{i + 1}.weight"] = (C[i + 1], C[i], TAPS[i], 1)
        d[f"conv{i + 1}.bias"] = (C[i + 1],)
        for n in ("weight", "bias", "running_mean", "running_var"):
            d[f"conv{i + 1}_BN.{n}"] = (C[i + 1],)
    d["classifier.weight"] = (PITCH_BINS, 4 * C[6])
    d["classifier.bias"] = (PITCH_BINS,)
    return d


def check_model(sd: Dict[str, torch.Tensor], capacity: str) -> Dict[str, torch.Tensor]:
    if capacity not in CHANNELS:
        raise ValueError(f"capacity {capacity!r} is not 'full' or 'tiny'")
    for k, shape in shapes(capacity).items():
        if k not in sd:
            raise ValueError(f"not a CREPE '{capacity}' state dict: {k} is missing")
        if tuple(sd[k].shape) != shape:
            raise ValueError(f"not a CREPE '{capacity}' state dict: {k} has shape {tuple(sd[k].shape)}, need {shape}")
    return {k: sd[k].detach().float().contiguous() for k in shapes(capacity)}


def conv1_image(w: torch.Tensor) -> torch.Tensor:
    """[1024, 512] -> bf16 [8 column tiles][64 K octets][128][8]: a tile is one K-major wgmma B operand."""
    return w.bfloat16().view(8, 128, 64, 8).permute(0, 2, 1, 3).contiguous()


def conv_image(w: torch.Tensor, ck: int) -> torch.Tensor:
    """[Cout, Cin, 64] -> bf16 [Cout / 128][Cin / ck][64 / tg][tg taps][ck / 8][128][8], tg = 128 / ck: 32 KB stages in
    the order the kernel's K loop takes them (channel chunk, then tap group)."""
    cout, cin, taps = w.shape
    tg = 128 // ck
    v = w.bfloat16().view(cout // 128, 128, cin // ck, ck // 8, 8, taps // tg, tg)
    return v.permute(0, 2, 5, 6, 3, 1, 4).contiguous()


def conv_image_unpack(img: torch.Tensor, cout: int, cin: int, ck: int) -> torch.Tensor:
    """Inverse of conv_image (the weights as the kernel sees them, rounded to bf16)."""
    tg = 128 // ck
    v = img.view(cout // 128, cin // ck, 64 // tg, tg, ck // 8, 128, 8).permute(0, 5, 1, 4, 6, 2, 3)
    return v.reshape(cout, cin, 64).float()


def pack_crepe(sd: Dict[str, torch.Tensor], capacity: str) -> List[Tuple[str, torch.Tensor]]:
    """-> [(name, fp32-typed tensor)], the names csrc/crepe_api.cu reads.  BatchNorm becomes an eval scale and shift that
    stay apart from the weights (they follow the ReLU); `full` conv weights become bf16 operand images."""
    items = []
    for i in range(6):
        p = f"conv{i + 1}"
        w = sd[p + ".weight"].squeeze(-1)
        bn = {n: sd[f"{p}_BN.{n}"].double() for n in ("weight", "bias", "running_mean", "running_var")}
        scale = bn["weight"] / torch.sqrt(bn["running_var"] + BN_EPS)
        if capacity == "full":
            img = conv1_image(w.reshape(1024, 512)) if i == 0 else conv_image(w, CONV_CK[i - 1])
            items.append((f"crepe.{p}.wimg", img.view(torch.float32).reshape(-1)))
        else:
            items.append((f"crepe.{p}.w", w))
        items += [(f"crepe.{p}.bias", sd[p + ".bias"]), (f"crepe.{p}.scale", scale.float()),
                  (f"crepe.{p}.shift", (bn["bias"] - bn["running_mean"] * scale).float())]
    items += [("crepe.cls.wt", sd["classifier.weight"].t()), ("crepe.cls.bias", sd["classifier.bias"])]
    return [(n, t.contiguous()) for n, t in items]


def frames_of(n_samples: int, hop: int) -> int:
    """crepe/core.py:663: 1 + n // hop frames (the audio is zero-padded by 512 on both sides)."""
    return 1 + int(n_samples) // int(hop)


def draw_noise(n: int) -> torch.Tensor:
    """pitch/inference.py:78: the randn_like(audio) that is added at 0.001."""
    return torch.randn(int(n))


def draw_dither(frames: int) -> torch.Tensor:
    """crepe/convert.py:51-57: triangular over +-20 cents, one draw per frame."""
    import scipy.stats
    return torch.from_numpy(scipy.stats.triang.rvs(c=0.5, loc=-20, scale=40, size=int(frames)).astype(np.float32))


# ------------------------------------------------------------------------------------------------ device calls
def frame_device(wavs: Sequence, hop: int, noises: Optional[Sequence] = None, device="cuda"):
    """Ragged batch -> (normalised frames [sum F_b, 1024] on the device, frame offsets)."""
    device = _lib.cuda_device(device)
    flat, so = _lib.ragged(wavs, device)
    B = len(so) - 1
    nz = _lib.ragged(noises, device)[0] if noises is not None else None
    if nz is not None and nz.numel() != flat.numel():
        raise ValueError("noise must have the length of its audio")
    fo = _lib.offsets(frames_of(so[b + 1] - so[b], hop) for b in range(B))
    out = torch.empty(fo[-1], WINDOW, device=device, dtype=torch.float32)
    _lib.call("crepe_frame", flat.data_ptr(), so, B, int(hop), nz.data_ptr() if nz is not None else None, out.data_ptr(),
              device=device)
    return out, fo


def decode_device(probs: torch.Tensor, frame_offsets, dither: Optional[torch.Tensor] = None, segment: int = SEGMENT):
    """Masked sigmoid outputs [sum F_b, 360] on the device -> (bins int32, pitch Hz, periodicity), each [sum F_b]."""
    device = _lib.cuda_device(probs.device)
    probs = probs.float().contiguous()
    n = probs.shape[0]
    bins = torch.empty(n, device=device, dtype=torch.int32)
    pitch = torch.empty(n, device=device, dtype=torch.float32)
    period = torch.empty(n, device=device, dtype=torch.float32)
    d = dither.to(device=device, dtype=torch.float32).contiguous() if dither is not None else None
    if d is not None and d.numel() != n:
        raise ValueError("dither must have one value per frame")
    ws = torch.empty(_lib.load().svcb_crepe_decode_workspace_bytes(n), device=device, dtype=torch.uint8)
    _lib.call("crepe_decode", probs.data_ptr(), frame_offsets, len(frame_offsets) - 1, int(segment),
              d.data_ptr() if d is not None else None, bins.data_ptr(), pitch.data_ptr(), period.data_ptr(), ws.data_ptr(),
              ws.numel(), device=device)
    return bins, pitch, period


class CrepeB200:
    """CREPE 'full' or 'tiny', for inference on ragged batches of 16 kHz recordings."""

    def __init__(self, sd: Dict[str, torch.Tensor], device, capacity: str = "full"):
        self.device = _lib.cuda_device(device)
        self.capacity = capacity
        blob_cpu, table = pack.build_blob(pack_crepe(check_model(sd, capacity), capacity))
        self._handle = _lib.Handle("crepe", table, blob_cpu.to(self.device), 0 if capacity == "full" else 1)

    @torch.no_grad()
    def probs_device(self, wavs: Sequence, hop: int, noises: Optional[Sequence] = None):
        """Ragged batch -> (masked sigmoid outputs [sum F_b, 360] on the device, frame offsets)."""
        flat, so = _lib.ragged(wavs, self.device)
        B = len(so) - 1
        nz = _lib.ragged(noises, self.device)[0] if noises is not None else None
        if nz is not None and nz.numel() != flat.numel():
            raise ValueError("noise must have the length of its audio")
        fo = _lib.offsets(frames_of(so[b + 1] - so[b], hop) for b in range(B))
        probs = torch.empty(fo[-1], PITCH_BINS, device=self.device, dtype=torch.float32)
        ws = self._handle.workspace(_lib.load().svcb_crepe_workspace_bytes(self._handle, fo[-1]))
        self._handle.call("crepe_probs", flat.data_ptr(), so, B, int(hop), nz.data_ptr() if nz is not None else None,
                          probs.data_ptr(), ws.data_ptr(), ws.numel())
        return probs, fo


def load_model(path: str, device="cuda", capacity: str = "full") -> CrepeB200:
    """crepe/load.py in effect: crepe/assets/{full,tiny}.pth -> the device model."""
    return CrepeB200(torch.load(path, map_location="cpu", weights_only=True), device, capacity)


# ------------------------------------------------------------------------------------------------ crepe.predict
@torch.no_grad()
def predict_batch(model: CrepeB200, audios: Sequence, hop: int, noises: Optional[Sequence] = None,
                  dithers: Optional[Sequence] = None, return_periodicity: bool = False):
    """crepe.predict(audio + 0.001 noise, 16000, hop, 50, 1000, batch_size=512, viterbi) for each clip of a ragged batch ->
    a list of pitch tensors [F_b] (CPU, fp32), or of (pitch, periodicity) pairs."""
    audios = [torch.as_tensor(np.asarray(a, np.float32)) if not torch.is_tensor(a) else a for a in audios]
    if noises is None:
        noises = [draw_noise(a.numel()) for a in audios]
    probs, fo = model.probs_device(audios, hop, noises)
    if dithers is None:
        dithers = [draw_dither(fo[b + 1] - fo[b]) for b in range(len(audios))]
    dither = torch.cat([torch.as_tensor(d, dtype=torch.float32).reshape(-1) for d in dithers])
    _, pitch, period = decode_device(probs, fo, dither)
    pitch, period = _lib.split(pitch.cpu(), fo), _lib.split(period.cpu(), fo)
    return list(zip(pitch, period)) if return_periodicity else pitch


def predict(model: CrepeB200, audio, hop: int, noise=None, dither=None, return_periodicity: bool = False):
    return predict_batch(model, [audio], hop, None if noise is None else [noise], None if dither is None else [dither],
                         return_periodicity)[0]


# ------------------------------------------------------------------------------------------------ crepe.filter (host)
def mean(signal: torch.Tensor, win_length: int) -> torch.Tensor:
    """crepe/filter.py:10-56 on one [T] vector: the zero-padded sum over the count of values that are not NaN; a result
    of exactly zero becomes NaN."""
    x = signal.float().reshape(1, 1, -1)
    mask = ~torch.isnan(x)
    ones = torch.ones(1, 1, win_length)
    total = F.conv1d(torch.where(mask, x, torch.zeros_like(x)), ones, padding=win_length // 2)
    count = F.conv1d(mask.float(), ones, padding=win_length // 2).clamp(min=1)
    out = total / count
    out[out == 0] = float("nan")
    return out.reshape(-1)


def median(signal: torch.Tensor, win_length: int) -> torch.Tensor:
    """crepe/filter.py:59-106 on one [T] vector: reflect-padded values, zero-padded validity, the lower median of the
    valid values of each window."""
    x = signal.float().reshape(1, 1, -1)
    pad = win_length // 2
    mask = ~torch.isnan(x)
    xp = F.pad(torch.where(mask, x, torch.zeros_like(x)), (pad, pad), mode="reflect").unfold(2, win_length, 1)
    mp = F.pad(mask.float(), (pad, pad)).unfold(2, win_length, 1)
    s, _ = torch.sort(torch.where(mp.bool(), xp, torch.full_like(xp, float("inf"))), dim=-1)
    idx = ((mp.sum(-1) - 1) // 2).clamp(min=0).long()
    out = s.gather(-1, idx.unsqueeze(-1)).squeeze(-1)
    out[torch.isinf(out)] = float("nan")
    return out.reshape(-1)


# ------------------------------------------------------------------------------------------------ the two callers
def compute_f0_sing_batch(model: CrepeB200, audios: Sequence, noises=None, dithers=None) -> List[torch.Tensor]:
    """pitch/inference.py:74-99 per clip: hop 320, every value twice, mean over 5 -> [2 (1 + n // 320)], one per 10 ms."""
    return [mean(p.repeat_interleave(2), 5) for p in predict_batch(model, audios, 320, noises, dithers)]


def compute_f0_sing(model: CrepeB200, audio, noise=None, dither=None) -> torch.Tensor:
    return compute_f0_sing_batch(model, [audio], None if noise is None else [noise], None if dither is None else [dither])[0]


def pred_pit(model: CrepeB200, wavPath: str, pitPath: str, noise=None, dither=None):
    """pitch/inference.py:120-130 (its __main__): the wav read at 16 kHz by `hubert_infer.load_audio`, `compute_f0_sing`,
    and the `.pit.csv` written by `hostio.save_csv_pitch`."""
    audio = hubert_infer.load_audio(wavPath, SAMPLE_RATE)
    hostio.save_csv_pitch(compute_f0_sing(model, audio, noise, dither), pitPath)


def finish_f0(pitch: torch.Tensor, periodicity: torch.Tensor) -> np.ndarray:
    """prepare/preprocess_crepe.py:40-43: median(periodicity, 7), mean(pitch, 5), zero where the periodicity is below 0.5."""
    periodicity = median(periodicity, 7)
    pitch = mean(pitch, 5)
    pitch[periodicity < 0.5] = 0
    return pitch.numpy().astype(np.float32)


def compute_f0_batch(model: CrepeB200, audios: Sequence, noises=None, dithers=None) -> List[np.ndarray]:
    """prepare/preprocess_crepe.py:11-44 per clip: hop 160 -> float32 [1 + n // 160], the contents of `.pit.npy`."""
    return [finish_f0(p, q) for p, q in predict_batch(model, audios, 160, noises, dithers, return_periodicity=True)]


def compute_f0(model: CrepeB200, audio, noise=None, dither=None) -> np.ndarray:
    return compute_f0_batch(model, [audio], None if noise is None else [noise], None if dither is None else [dither])[0]
