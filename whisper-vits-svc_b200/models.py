"""Host-side mirror of the reference's acoustic-model surface (vits/models.py:211-256).

`SynthesizerInfer(spec_channels, segment_size, hp)` keeps the constructor, the 903-key
state-dict (so `load_svc_model`, svc_inference.py:61-74, works unchanged) and the three methods
callers use -- `inference`, `pitch2source`, `source2wav` -- but every arithmetic step runs in
libsvc_b200.so through the C ABI (include/svcb.h).  PyTorch is only the owner of device memory
and streams here.  There is no CPU path: calling a compute method without a CUDA device, or
without the built library, raises.

`precision` selects how the dense convolutions are computed (DESIGN.md §3): 3 (default) =
bf16x3-split wgmma MMAs + fused fp32 narrow stages (meets the 1e-3 waveform gate, ~1e-5 measured),
1 = plain bf16 MMAs (faster, ~4e-3), 0 = all-fp32 CUDA-core kernels (device-side reference).

The reference draws three random tensors internally (vits/models.py:51,
vits_decoder/nsf.py:232-236,311); they are explicit keyword arguments here (`eps`, `rand_ini`,
`noise`) defaulting to fresh torch draws on the model's device, which is how parity tests inject
the reference's own draws.
"""
from __future__ import annotations

import ctypes
from typing import Dict, Optional

import numpy as np
import torch

from . import _lib, pack, synth


class SynthesizerInfer(torch.nn.Module):
    def __init__(self, spec_channels, segment_size, hp, precision: int = 3):
        super().__init__()
        self.segment_size = segment_size  # unused at inference, kept for signature parity
        self.hp = hp
        self._cfg = pack.config_from_hp(hp, precision)
        self.hop = int(np.prod(self._cfg["up_rates"]))
        # reference-format parameters, default-initialised like a seeded synthetic checkpoint
        proto = synth.svc_state_dict(hp, seed=int(getattr(getattr(hp, "train", {}), "seed", 1234) or 1234))
        self._keys = list(proto.keys())
        for k, v in proto.items():
            self.register_buffer(self._mangle(k), v, persistent=True)
        self._handle = None
        self._blob = None
        self._ws = None
        self._packed_device = None

    # ---- state-dict surface (reference key names) -----------------------------------------
    @staticmethod
    def _mangle(k: str) -> str:
        return "p__" + k.replace(".", "__")

    def state_dict(self, *a, **kw):  # noqa: D401 - reference key names, not mangled buffers
        return {k: getattr(self, self._mangle(k)) for k in self._keys}

    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        missing = [k for k in self._keys if k not in sd]
        if strict and missing:
            raise KeyError(f"missing keys in state_dict: {missing[:5]}{'...' if len(missing) > 5 else ''}")
        for k in self._keys:
            if k in sd:
                cur = getattr(self, self._mangle(k))
                if tuple(sd[k].shape) != tuple(cur.shape):
                    raise ValueError(f"shape mismatch for {k}: {tuple(sd[k].shape)} vs {tuple(cur.shape)}")
                cur.copy_(sd[k].to(cur.device, torch.float32))
        self._release()
        return self

    def remove_weight_norm(self):
        """The reference's SynthesizerInfer.remove_weight_norm raises AttributeError
        (vits/models.py:96-98 reads an undefined self.n_flows); weight-norm is always folded at
        pack time here, so this is a no-op."""
        return None

    def forward(self, ppg, vec, pit, spk, ppg_l, source, **kw):
        return self.inference(ppg, vec, pit, spk, ppg_l, source, **kw)

    # ---- device plumbing -------------------------------------------------------------------
    def _release(self):
        if self._handle is not None:
            _lib.load().svcb_model_destroy(self._handle)
        self._handle = None
        self._blob = None

    def __del__(self):
        try:
            self._release()
        except Exception:
            pass

    def _device(self) -> torch.device:
        return getattr(self, self._mangle(self._keys[0])).device

    def _ensure(self):
        dev = self._device()
        if dev.type != "cuda":
            raise _lib.SvcbError("SynthesizerInfer computes only on a CUDA device (sm_90a); "
                                 "call .to('cuda') first. There is no CPU fallback.")
        if self._handle is not None and self._packed_device == dev:
            return
        self._release()
        lib = _lib.load()
        sd_cpu = {k: v.detach().cpu() for k, v in self.state_dict().items()}
        items = pack.pack_svc_state_dict(sd_cpu, self._cfg)
        blob_cpu, table = pack.build_blob(items)
        self.install_blob(blob_cpu.to(dev), table)

    def install_blob(self, blob_dev: torch.Tensor, table):
        """Create the device handle from an already packed blob (used by the multi-GPU path after
        the NCCL broadcast of rank 0's blob)."""
        lib = _lib.load()
        self._release()
        entries = (_lib.TensorEntry * len(table))()
        for e, (name, off, numel) in zip(entries, table):
            e.name = name.encode()
            e.offset_bytes = off
            e.numel = numel
        cfg = _lib.Config.from_dict(self._cfg)
        handle = ctypes.c_void_p()
        with torch.cuda.device(blob_dev.device):
            st = lib.svcb_model_create(blob_dev.data_ptr(), blob_dev.numel() * 4, entries, len(table),
                                       ctypes.byref(cfg), ctypes.byref(handle))
        _lib.check(st, "svcb_model_create")
        self._blob = blob_dev
        self._table = table
        self._handle = handle
        self._packed_device = blob_dev.device

    def packed_blob(self):
        self._ensure()
        return self._blob, self._table

    def _workspace(self, B: int, T: int) -> torch.Tensor:
        need = int(_lib.load().svcb_workspace_bytes(self._handle, B, T))
        if self._ws is None or self._ws.numel() < need or self._ws.device != self._packed_device:
            self._ws = torch.empty(need, dtype=torch.uint8, device=self._packed_device)
        return self._ws

    @staticmethod
    def _stream():
        return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def _f32(self, t: torch.Tensor) -> torch.Tensor:
        return t.to(self._packed_device, torch.float32).contiguous()

    def _taps(self, taps: Optional[Dict[str, torch.Tensor]]):
        if not taps:
            return None
        st = _lib.Taps()
        for name, t in taps.items():
            assert t.is_cuda and t.is_contiguous() and t.dtype == torch.float32, f"tap {name} must be a contiguous fp32 CUDA tensor"
            st.ptr[_lib.TAPS[name]] = t.data_ptr()
        return ctypes.byref(st)

    # ---- reference surface -----------------------------------------------------------------
    @torch.no_grad()
    def pitch2source(self, f0, rand_ini=None, noise=None):
        """Generator.pitch2source (vits_decoder/generator.py:160-165): f0 [B,T] -> [B,1,T*hop]."""
        self._ensure()
        f0 = self._f32(f0)
        B, T = f0.shape
        L = T * self.hop
        nh = self._cfg["n_harmonics"]
        dev = self._packed_device
        if rand_ini is None:
            rand_ini = torch.rand(B, nh, device=dev)
        if noise is None:
            noise = torch.randn(B, L, nh, device=dev)
        rand_ini, noise = self._f32(rand_ini), self._f32(noise)
        assert rand_ini.shape == (B, nh) and noise.shape == (B, L, nh)
        out = torch.empty(B, 1, L, device=dev, dtype=torch.float32)
        # the source scan needs O(B*T) bytes, not the pipeline's peak: the host loop calls this on the
        # whole utterance before chunking (svc_inference.py:89-91)
        ws = torch.empty(int(_lib.load().svcb_source_workspace_bytes(self._handle, B, T)), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            st = _lib.load().svcb_source(self._handle, f0.data_ptr(), rand_ini.data_ptr(), noise.data_ptr(),
                                         out.data_ptr(), B, T, ws.data_ptr(), ws.numel(), self._stream())
        _lib.check(st, "svcb_source")
        return out

    @torch.no_grad()
    def source2wav(self, source):
        """Generator.source2wav (generator.py:167-173) -> int16 numpy array on the host."""
        self._ensure()
        src = self._f32(source).reshape(-1)
        out = torch.empty(src.numel(), dtype=torch.int16, device=src.device)
        with torch.cuda.device(src.device):
            st = _lib.load().svcb_source2wav(src.data_ptr(), out.data_ptr(), src.numel(), self._stream())
        _lib.check(st, "svcb_source2wav")
        return out.cpu().numpy()

    @torch.no_grad()
    def inference(self, ppg, vec, pit, spk, ppg_l, source, eps=None, taps=None):
        """SynthesizerInfer.inference (vits/models.py:251-256).
        ppg [B,T,ppg_dim], vec [B,T,vec_dim], pit [B,T], spk [B,spk_dim], ppg_l [B] int64,
        source [B,1,T*hop] -> wave [B,1,T*hop]."""
        self._ensure()
        dev = self._packed_device
        ppg, vec, pit, spk, source = map(self._f32, (ppg, vec, pit, spk, source))
        B, T, _ = ppg.shape
        C = self._cfg["inter_channels"]
        lengths = ppg_l.to(dev, torch.int64).contiguous()
        if eps is None:
            eps = torch.randn(B, C, T, device=dev)
        eps = self._f32(eps)
        assert vec.shape[:2] == (B, T) and pit.shape == (B, T) and spk.shape[0] == B
        assert source.shape == (B, 1, T * self.hop) and eps.shape == (B, C, T)
        wave = torch.empty(B, 1, T * self.hop, device=dev, dtype=torch.float32)
        ws = self._workspace(B, T)
        with torch.cuda.device(dev):
            st = _lib.load().svcb_infer(self._handle, ppg.data_ptr(), vec.data_ptr(), pit.data_ptr(),
                                        spk.data_ptr(), lengths.data_ptr(), source.data_ptr(), eps.data_ptr(),
                                        wave.data_ptr(), B, T, ws.data_ptr(), ws.numel(), self._taps(taps),
                                        self._stream())
        _lib.check(st, "svcb_infer")
        return wave

    # ---- stage entry points (parity tests, profiling) ---------------------------------------
    @torch.no_grad()
    def prior(self, ppg, vec, pit, ppg_l, eps, taps=None):
        self._ensure()
        dev = self._packed_device
        ppg, vec, pit, eps = map(self._f32, (ppg, vec, pit, eps))
        B, T, _ = ppg.shape
        lengths = ppg_l.to(dev, torch.int64).contiguous()
        z_p = torch.empty(B, self._cfg["inter_channels"], T, device=dev)
        ws = self._workspace(B, T)
        with torch.cuda.device(dev):
            st = _lib.load().svcb_prior(self._handle, ppg.data_ptr(), vec.data_ptr(), pit.data_ptr(),
                                        lengths.data_ptr(), eps.data_ptr(), z_p.data_ptr(), B, T,
                                        ws.data_ptr(), ws.numel(), self._taps(taps), self._stream())
        _lib.check(st, "svcb_prior")
        return z_p

    @torch.no_grad()
    def flow_reverse(self, z_p, ppg_l, spk, taps=None):
        self._ensure()
        dev = self._packed_device
        z_p, spk = self._f32(z_p), self._f32(spk)
        B, C, T = z_p.shape
        lengths = ppg_l.to(dev, torch.int64).contiguous()
        z = torch.empty_like(z_p)
        ws = self._workspace(B, T)
        with torch.cuda.device(dev):
            st = _lib.load().svcb_flow(self._handle, z_p.data_ptr(), lengths.data_ptr(), spk.data_ptr(),
                                       z.data_ptr(), B, T, ws.data_ptr(), ws.numel(), self._taps(taps),
                                       self._stream())
        _lib.check(st, "svcb_flow")
        return z

    @torch.no_grad()
    def generator(self, spk, z, source, taps=None):
        """Generator.inference(spk, x, har_source) (vits_decoder/generator.py:175-200)."""
        self._ensure()
        dev = self._packed_device
        spk, z, source = map(self._f32, (spk, z, source))
        B, U, T = z.shape
        assert U == self._cfg["gen_input"] and source.shape == (B, 1, T * self.hop)
        wave = torch.empty(B, 1, T * self.hop, device=dev)
        ws = self._workspace(B, T)
        with torch.cuda.device(dev):
            st = _lib.load().svcb_generator(self._handle, spk.data_ptr(), z.data_ptr(), source.data_ptr(),
                                            wave.data_ptr(), B, T, ws.data_ptr(), ws.numel(),
                                            self._taps(taps), self._stream())
        _lib.check(st, "svcb_generator")
        return wave
