"""The trainer's validation score, `validation/mel_loss` (vits_extend/validation.py, called from
vits_extend/train.py:160), for saved checkpoints on the H100 path.

The validation set is read once per run, as `create_dataloader_eval` reads it: `preprocess_zzz.TextAudioSpeakerSet`
over hp.data.validation_files (the reference's filter, trims and random crop) in file order, `batch` items per batch,
no shuffle, no drop_last, each batch through `preprocess_zzz.collate`.  Every batch is uploaded once, its real mels are
computed once, and its five random draws are made once:

- `ppg_noise`: SynthesizerTrn.infer's perturbation `ppg + randn_like(ppg) * 1e-4` (vits/models.py:203), applied here;
- `eps`: the prior's sample (vits/models.py:51);
- `z_noise`: Generator.forward's perturbation `x + randn_like(x)` (vits_decoder/generator.py:116), of the masked z;
- `rand_ini` and `noise`: the NSF source's draws (vits_decoder/nsf.py:232, 311).

So every checkpoint sees the same crops and the same draws, and score differences come from the weights alone.  Per
checkpoint, the padded batch runs unmasked over all T frames as the reference runs it (pitch2source, prior, reverse
flow, the generator on z * mask + z_noise), the fake and real mels are compared by `F.l1_loss` (mean over B x 100 x T,
padding included) and the batch losses are summed and divided by the number of items, not batches, as the reference
does.

Deviations from the reference (DESIGN.md §8): the crops come from Python's `random` seeded with `seed` and the draws
from a device generator seeded with `seed` (the reference's come from unseeded loader workers and the trainer's running
RNG); weight norm is folded at pack time (the reference validates with it attached; the same function up to
rounding); there is no TensorBoard, and `on_audio` receives the audio the reference would log instead.

No CPU fallback: the model and the mel run on a CUDA (sm_90a) device."""
from __future__ import annotations

import random
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib, hostio, models, pack, spectrogram, whisper_infer

HOP = spectrogram.HOP
MAX_MELS = 128   # csrc/mel_api.cu MEL_MAX_MELS
DRAWS = ("ppg_noise", "eps", "z_noise", "rand_ini", "noise")


def mel_basis(hp) -> torch.Tensor:
    """librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax) of vits_extend/stft.py:46-47 at hp.data's values, float32."""
    d = hp.data
    return whisper_infer.mel_filters(int(d.mel_channels), int(d.sampling_rate), int(d.filter_length),
                                     fmin=float(d.mel_fmin), fmax=None if d.mel_fmax is None else float(d.mel_fmax))


@torch.no_grad()
def tacotron_mel(audio: torch.Tensor, basis: torch.Tensor) -> torch.Tensor:
    """TacotronSTFT.mel_spectrogram (vits_extend/stft.py:71-104) of a padded batch: audio [B, L] on a CUDA device,
    basis [n_mels, 513] -> [B, n_mels, L // 320] float32 (svcb_tacotron_mel).  Raises ValueError when the audio leaves
    [-1, 1], where the reference asserts."""
    dev = _lib.cuda_device(audio.device)
    x = audio.to(torch.float32).contiguous()
    if x.dim() != 2:
        raise ValueError(f"audio must be [B, L], not {tuple(x.shape)}")
    lo, hi = torch.aminmax(x)
    if float(lo) < -1.0 or float(hi) > 1.0:
        raise ValueError(f"audio leaves [-1, 1]: min {float(lo)}, max {float(hi)}")
    fb = basis.to(dev, torch.float32).contiguous()
    B, L = x.shape
    out = torch.empty(B, fb.shape[0], L // HOP, dtype=torch.float32, device=dev)
    _lib.call("tacotron_mel", x.data_ptr(), B, L, fb.data_ptr(), fb.shape[0], out.data_ptr(), device=dev)
    return out


@dataclass
class Batch:
    """One collated batch on the device: the model inputs (ppg with its perturbation applied), the mask, the real audio
    [B, 1, L] and its mels, and the fixed draws."""
    ppg: torch.Tensor
    ppg_l: torch.Tensor
    vec: torch.Tensor
    pit: torch.Tensor
    spk: torch.Tensor
    mask: torch.Tensor
    audio: torch.Tensor
    mel_real: torch.Tensor
    draws: Dict[str, torch.Tensor] = field(default_factory=dict)


@dataclass
class ValidationSet:
    batches: List[Batch]
    n_items: int


def draw_shapes(B: int, T: int, hp) -> Dict[str, tuple]:
    """(shape, 'randn' | 'rand') of each draw of a batch of B items padded to T frames, in the reference's call
    order."""
    C = int(hp.vits.inter_channels)
    nh = pack.config_from_hp(hp, 3)["n_harmonics"]
    return {"ppg_noise": ((B, T, int(hp.vits.ppg_dim)), "randn"), "eps": ((B, C, T), "randn"),
            "z_noise": ((B, C, T), "randn"), "rand_ini": ((B, nh), "rand"), "noise": ((B, T * HOP, nh), "randn")}


def device_draws(seed: int, device) -> Callable[[int, Dict[str, tuple]], Dict[str, torch.Tensor]]:
    """The default draw: one device generator seeded with `seed`, drawn batch by batch in the reference's order."""
    g = torch.Generator(device=device)
    g.manual_seed(int(seed))

    def draw(bi, shapes):
        return {k: (torch.randn if kind == "randn" else torch.rand)(shape, generator=g, device=device)
                for k, (shape, kind) in shapes.items()}
    return draw


@torch.no_grad()
def load_set(hp, files: str, seed: int, batch: int, device="cuda", draw=None) -> ValidationSet:
    """The validation set of `files` (a file list in the reference's format), read and drawn once.  `draw(batch index,
    draw_shapes(...))` supplies the draws (default: device_draws(seed)).  ValueError when no item passes the filter."""
    import preprocess_zzz

    dev = _lib.cuda_device(device)
    spectrogram.check_hparams(hp)
    random.seed(int(seed))
    ds = preprocess_zzz.TextAudioSpeakerSet(files, hp.data)
    if len(ds) == 0:
        raise ValueError(f"the validation set {files} is empty: no item has all its files and at least 1 s")
    draw = draw or device_draws(seed, dev)
    basis = mel_basis(hp).to(dev)
    out = []
    for bi, i0 in enumerate(range(0, len(ds), batch)):
        ppg, ppg_l, vec, pit, spk, _, _, wav, _ = preprocess_zzz.collate([ds[i] for i in range(i0, min(i0 + batch, len(ds)))])
        B, T = pit.shape
        if wav.shape[2] != T * HOP:
            raise ValueError(f"batch {bi}: {wav.shape[2]} samples for {T} frames")
        d = {k: v.to(dev) for k, v in draw(bi, draw_shapes(B, T, hp)).items()}
        ppg = ppg.to(dev) + d.pop("ppg_noise") * 0.0001
        ppg_l = ppg_l.to(dev)
        mask = (torch.arange(T, device=dev)[None, :] < ppg_l[:, None]).to(torch.float32).unsqueeze(1)
        audio = wav.to(dev)
        out.append(Batch(ppg, ppg_l.to(torch.int64), vec.to(dev), pit.to(dev), spk.to(dev), mask, audio,
                         tacotron_mel(audio.squeeze(1), basis), d))
    return ValidationSet(out, len(ds))


def prepare_checkpoint(path: str, staging: models.SynthesizerInfer, defaults: Dict[str, torch.Tensor]):
    """Host work of one checkpoint: hostio.load_svc_model into the CPU model `staging` (reset to `defaults` first, so
    a missing key keeps its default and not the previous checkpoint's value), then the packed blob.  -> (state dict,
    blob, table).  Safe on a worker thread while the device scores the previous checkpoint."""
    staging.load_state_dict(defaults)
    hostio.load_svc_model(path, staging)
    sd = {k: v.clone() for k, v in staging.state_dict().items()}
    blob, table = pack.build_blob(pack.pack_svc_state_dict(sd, staging._cfg))
    return sd, blob, table


class Scorer:
    """One reused device SynthesizerInfer (precision 3) and the mel basis; `score(path, vset)` loads, repacks and
    scores one checkpoint.  Device memory does not grow with the number of checkpoints: each new blob replaces the
    last, and every batch's buffers have the sizes of the first checkpoint's."""

    def __init__(self, hp, device="cuda"):
        spectrogram.check_hparams(hp)
        self.hp, self.device = hp, _lib.cuda_device(device)
        if int(hp.data.mel_channels) > MAX_MELS:
            raise ValueError(f"mel_channels {hp.data.mel_channels}: the device mel supports at most {MAX_MELS}")
        mk = lambda: models.SynthesizerInfer(int(hp.data.filter_length) // 2 + 1,
                                             int(hp.data.segment_size) // int(hp.data.hop_length), hp, precision=3)
        self.staging = mk()   # CPU: checkpoints are read into it on the loader thread
        self.defaults = {k: v.clone() for k, v in self.staging.state_dict().items()}
        self.model = mk().eval().to(self.device)
        self.basis = mel_basis(hp).to(self.device)
        self._pool = ThreadPoolExecutor(max_workers=1)

    def close(self):
        self._pool.shutdown(wait=True)

    def prefetch(self, path: str):
        """A future of prepare_checkpoint(path): one checkpoint ahead at most, since the staging model is shared."""
        return self._pool.submit(prepare_checkpoint, path, self.staging, self.defaults)

    def install(self, prepared):
        """Upload a prepared checkpoint into the device model.  The previous blob and workspace are freed first, so
        they are never held together with the upload's staging copies."""
        sd, blob, table = prepared
        self.model.release()
        self.model.load_state_dict(sd)
        self.model.install_blob(blob.to(self.device), table)

    @torch.no_grad()
    def fake_audio(self, b: Batch) -> torch.Tensor:
        """generator.infer(ppg, vec, pit, spk, ppg_l) of vits/models.py:202-208 with the batch's fixed draws ->
        [B, 1, T * 320]."""
        m = self.model
        source = m.pitch2source(b.pit, rand_ini=b.draws["rand_ini"], noise=b.draws["noise"])
        z_p = m.prior(b.ppg, b.vec, b.pit, b.ppg_l, b.draws["eps"])
        z = m.flow_reverse(z_p, b.ppg_l, b.spk)
        return m.generator(b.spk, z * b.mask + b.draws["z_noise"], source)

    @torch.no_grad()
    def score_installed(self, vset: ValidationSet, on_audio=None, timings: Optional[dict] = None) -> float:
        """validation/mel_loss of the installed weights.  on_audio(idx, real, fake), for batches idx <
        hp.log.num_audio: item 0's real and fake audio (float32 numpy), which the reference logs.  timings, when given,
        gains the seconds spent in the model ('infer') and the mel and loss ('mel'), with a device synchronise
        between the two."""
        import time
        total = 0.0
        n_audio = int(self.hp.log.num_audio)
        for idx, b in enumerate(vset.batches):
            t0 = time.perf_counter()
            fake = self.fake_audio(b)[:, :, :b.audio.size(2)]
            if timings is not None:
                torch.cuda.synchronize(self.device)
                t1 = time.perf_counter()
                timings["infer"] = timings.get("infer", 0.0) + t1 - t0
            mel_fake = tacotron_mel(fake.squeeze(1), self.basis)
            total += F.l1_loss(mel_fake, b.mel_real).item()
            if timings is not None:
                timings["mel"] = timings.get("mel", 0.0) + time.perf_counter() - t1
            if on_audio is not None and idx < n_audio:
                on_audio(idx, b.audio[0][0].cpu().numpy(), fake[0][0].cpu().numpy())
        return total / vset.n_items

    def score_paths(self, paths: Sequence[str], vset: ValidationSet, on_result, on_audio=None):
        """Score every checkpoint of `paths`, reading the next one on the loader thread while the device scores the
        current one.  on_result(path, loss, error): loss is None and error the exception when a checkpoint fails to
        load; the others are still scored.  on_audio(path, idx, real, fake) as in score_installed."""
        paths = list(paths)
        fut = self.prefetch(paths[0]) if paths else None
        for i, path in enumerate(paths):
            try:
                self.install(fut.result())
                err = None
            except Exception as e:   # noqa: BLE001 - reported, and the other checkpoints are scored
                err = e
            # the staging model is free again once install() has copied it
            fut = self.prefetch(paths[i + 1]) if i + 1 < len(paths) else None
            if err is not None:
                on_result(path, None, err)
                continue
            cb = None if on_audio is None else (lambda idx, r, f, p=path: on_audio(p, idx, r, f))
            on_result(path, self.score_installed(vset, cb), None)
