"""HuBERT-Soft content encoder on the H100 path — host-side mirror of the reference's `hubert/inference.py`
(`load_model`, `pred_vec`) and `hubert/hubert_model.py` (`hubert_soft`, `HubertSoft.units`) behind the C ABI
(`svcb_hubert_*`, csrc/hubert_api.cu).  SURVEY.md §8f-2.  No CPU fallback: a CUDA (sm_90a) device is required."""
from __future__ import annotations

import ctypes
from typing import Dict, List, Tuple

import numpy as np
import torch

from . import _lib, pack
from .whisper_infer import _bf16_as_f32, load_audio

SAMPLE_RATE = 16000
CHUNK = 20 * SAMPLE_RATE            # hubert/inference.py:30-33
POS_GROUPS, POS_HALF = 16, 24


def n_layers(sd: Dict[str, torch.Tensor]) -> int:
    return 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("encoder.layers."))


def pack_hubert(sd: Dict[str, torch.Tensor]) -> Tuple[List[Tuple[str, torch.Tensor]], int]:
    """-> ([(name, fp32-typed tensor)], n_layer).  Names consumed by csrc/hubert_api.cu.  State-dict keys:
    hubert/hubert_model.py:11-30 (`module.` prefixes already stripped, :219)."""
    items: List[Tuple[str, torch.Tensor]] = []

    def put(n, t):
        items.append((n, t.detach().float().contiguous()))

    fe = "feature_extractor."
    put("fe.conv0.w", pack.pack_conv(sd[fe + "conv0.weight"].float()))
    put("fe.gn.g", sd[fe + "norm0.weight"]); put("fe.gn.b", sd[fe + "norm0.bias"])
    for i in range(1, 7):
        wi = sd[fe + f"conv{i}.weight"].float()                                 # [512, 512, k]
        put(f"fe.conv{i}.w", pack.pack_conv(wi))                                # fp32 stem (flags bit 0)
        # tensor-core stem: W[co][j * 512 + ci] as a bf16 tile image (csrc/whisper_gemm.cu)
        items.append((f"fe.conv{i}.wimg", _bf16_as_f32(wi.permute(0, 2, 1).reshape(wi.shape[0], -1))))
    put("fp.ln.g", sd["feature_projection.norm.weight"]); put("fp.ln.b", sd["feature_projection.norm.bias"])
    items.append(("fp.w", _bf16_as_f32(sd["feature_projection.projection.weight"])))
    put("fp.b", sd["feature_projection.projection.bias"])
    # positional conv: weight_norm(dim=2) folded (hubert_model.py:122), one fp32 conv per (group, half of its outputs)
    pc = "positional_embedding.conv."
    w = torch._weight_norm(sd[pc + "weight_v"].float(), sd[pc + "weight_g"].float(), 2)      # [768, 48, 128]
    per_g = w.shape[0] // POS_GROUPS
    for g in range(POS_GROUPS):
        for h in range(per_g // POS_HALF):
            rows = slice(g * per_g + h * POS_HALF, g * per_g + (h + 1) * POS_HALF)
            put(f"pos.{g}.{h}.w", pack.pack_conv(w[rows]))
    for g in range(POS_GROUPS):   # tensor-core form: W_g[co][j * 48 + ci], output channels padded from 48 to 256
        wg = w[g * per_g:(g + 1) * per_g]                                       # [48, 48, 128]
        wp = torch.zeros(256, wg.shape[1] * wg.shape[2])
        wp[:per_g] = wg.permute(0, 2, 1).reshape(per_g, -1)
        items.append((f"pos.{g}.wimg", _bf16_as_f32(wp)))
        bp = torch.zeros(256)
        bp[:per_g] = sd[pc + "bias"].float()[g * per_g:(g + 1) * per_g]
        put(f"pos.{g}.bimg", bp)
    put("pos.b", sd[pc + "bias"])
    put("norm.g", sd["norm.weight"]); put("norm.b", sd["norm.bias"])
    L = n_layers(sd)
    for i in range(L):
        b, p = f"encoder.layers.{i}.", f"L{i}"
        items.append((p + ".wqkv", _bf16_as_f32(sd[b + "self_attn.in_proj_weight"])))
        put(p + ".bqkv", sd[b + "self_attn.in_proj_bias"])
        items.append((p + ".wo", _bf16_as_f32(sd[b + "self_attn.out_proj.weight"])))
        put(p + ".bo", sd[b + "self_attn.out_proj.bias"])
        items.append((p + ".w1", _bf16_as_f32(sd[b + "linear1.weight"])))
        put(p + ".b1", sd[b + "linear1.bias"])
        items.append((p + ".w2", _bf16_as_f32(sd[b + "linear2.weight"])))
        put(p + ".b2", sd[b + "linear2.bias"])
        put(p + ".ln1.g", sd[b + "norm1.weight"]); put(p + ".ln1.b", sd[b + "norm1.bias"])
        put(p + ".ln2.g", sd[b + "norm2.weight"]); put(p + ".ln2.b", sd[b + "norm2.bias"])
    items.append(("proj.w", _bf16_as_f32(sd["proj.weight"])))
    put("proj.b", sd["proj.bias"])
    return items, L


TAP_NAMES = ("features", "projected", "embedded", "layer0", "encoded")
TAP_WIDTH = (512, 768, 768, 768, 768)


class HubertSoftB200:
    """`HubertSoft` of the reference for inference: `units(wav)` with wav [B, 1, N] or [B, N] -> [B, T, 256] fp32."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device):
        self.device = _lib.cuda_device(device)
        items, self.n_layer = pack_hubert(state_dict)
        blob_cpu, table = pack.build_blob(items)
        self._handle = _lib.Handle("hubert", table, blob_cpu.to(self.device), self.n_layer)

    def _workspace(self, B: int, N: int) -> torch.Tensor:
        return self._handle.workspace(_lib.load().svcb_hubert_workspace_bytes(self._handle, B, N))

    def eval(self):
        return self

    @staticmethod
    def frames(n_samples: int) -> int:
        return int(_lib.load().svcb_hubert_frames(int(n_samples)))

    @torch.no_grad()
    def units(self, wav: torch.Tensor, taps: dict | None = None, fp32_stem: bool = False) -> torch.Tensor:
        """fp32_stem: the stride-2 convs and the positional conv in fp32 on the CUDA cores (flags 3; parity work)."""
        if wav.dim() == 3:
            wav = wav[:, 0]
        wav = wav.to(self.device, torch.float32).contiguous()
        B, N = wav.shape
        T = self.frames(N)
        if T < 1:
            raise _lib.SvcbError("audio shorter than one HuBERT frame")
        ws = self._workspace(B, N)
        out = torch.empty(B, T, 256, device=self.device, dtype=torch.float32)
        tap_arr = None
        if taps is not None:
            bufs = [torch.empty(B, T, w, device=self.device, dtype=torch.float32) for w in TAP_WIDTH]
            tap_arr = (ctypes.c_void_p * len(bufs))(*[b.data_ptr() for b in bufs])
        self._handle.call("hubert_units", wav.data_ptr(), out.data_ptr(), B, N, ws.data_ptr(), ws.numel(), tap_arr,
                          3 if fp32_stem else 0)
        if taps is not None:
            for n, b in zip(TAP_NAMES, bufs):
                taps[n] = b
        return out

    @torch.no_grad()
    def units_ragged(self, wav: torch.Tensor, n_samples: List[int]) -> torch.Tensor:
        """`units` for a ragged batch: item b is wav[b, :n_samples[b]] (at least one frame each) -> [B, frames(N), 256];
        item b's first frames(n_samples[b]) rows equal a lone `units` of it bit for bit, its later rows are zero."""
        wav = wav.to(self.device, torch.float32).contiguous()
        B, N = wav.shape
        assert len(n_samples) == B
        ws = self._workspace(B, N)
        out = torch.empty(B, self.frames(N), 256, device=self.device, dtype=torch.float32)
        lens = (ctypes.c_int32 * B)(*n_samples)
        self._handle.call("hubert_units_ragged", wav.data_ptr(), lens, out.data_ptr(), B, N, ws.data_ptr(), ws.numel())
        return out


def hubert_soft(path: str, device="cuda") -> HubertSoftB200:
    """hubert/hubert_model.py:212-222."""
    checkpoint = torch.load(path, map_location="cpu")
    checkpoint = {(k[len("module."):] if k.startswith("module.") else k): v for k, v in checkpoint.items()}
    return HubertSoftB200(checkpoint, device)


def load_model(path, device) -> HubertSoftB200:
    """hubert/inference.py:17-23 (the reference's `.half()` on CUDA corresponds to the bf16 tensor-core GEMMs here)."""
    return hubert_soft(path, device)


def chunk_plan(audln: int, chunk: int = CHUNK):
    """hubert/inference.py:29-48 as data: [(start, end)] — 20 s chunks, the remainder as a last shorter one."""
    out, idx = [], 0
    while idx + chunk < audln:
        out.append((idx, idx + chunk))
        idx += chunk
    if idx < audln:
        out.append((idx, audln))
    return out


def pred_vec(model: HubertSoftB200, wavPath: str, vecPath: str, device=None):
    """hubert/inference.py:25-50: 16 kHz mono audio -> [length, 256] (hop 320) saved with np.save.  The full 20 s chunks of
    a file run as ONE batch (the reference runs them one by one); a remainder too short for one frame is dropped, where
    the reference would raise inside conv1d."""
    audio = load_audio(wavPath, SAMPLE_RATE)
    plan = chunk_plan(audio.shape[0])
    vec_a = []
    full = [(s, e) for s, e in plan if e - s == CHUNK]
    if full:
        batch = torch.from_numpy(np.stack([audio[s:e] for s, e in full]))
        vec_a.extend(model.units(batch).reshape(-1, 256).cpu().numpy())
    for s, e in plan:
        if e - s != CHUNK and model.frames(e - s) >= 1:
            vec_a.extend(model.units(torch.from_numpy(audio[s:e])[None]).reshape(-1, 256).cpu().numpy())
    np.save(vecPath, np.asarray(vec_a, dtype=np.float32), allow_pickle=False)


@torch.no_grad()
def units_batch(model: HubertSoftB200, audios: List[np.ndarray]) -> List[np.ndarray]:
    """prepare/preprocess_hubert.py:pred_vec for several files in one ragged device batch: `units` of each WHOLE file
    (no 20 s chunking) -> float32 [frames(len), 256] per item, each equal to a lone run of it."""
    lens = [int(a.shape[0]) for a in audios]
    wav = np.zeros((len(audios), max(lens)), np.float32)
    for b, a in enumerate(audios):
        wav[b, :lens[b]] = a
    out = model.units_ragged(torch.from_numpy(wav), lens).cpu()
    return [out[b, :model.frames(n)].numpy() for b, n in enumerate(lens)]
