"""ctypes binding of libsvc_b200.so (the C ABI in include/svcb.h).

There is no fallback: if the library is missing or a call fails, a SvcbError is raised.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char, c_char_p, c_float, c_int, c_int16, c_int32, c_int64, c_size_t, c_uint64, c_void_p

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsvc_b200.so")

SVCB_MAX_UPS = 8
SVCB_MAX_RES = 4
SVCB_TAP_COUNT = 24

TAPS = {
    "enc_front": 0, **{f"enc_layer{i}": 1 + i for i in range(6)}, "z_p": 7,
    **{f"flow{i}": 8 + i for i in range(4)}, "gen_pre": 12,
    **{f"gen_up{i}": 13 + i for i in range(5)}, **{f"gen_stage{i}": 18 + i for i in range(5)},
}


class SvcbError(RuntimeError):
    pass


class Config(ctypes.Structure):
    _fields_ = [
        ("ppg_dim", c_int32), ("vec_dim", c_int32), ("spk_dim", c_int32), ("inter_channels", c_int32),
        ("hidden_channels", c_int32), ("filter_channels", c_int32),
        ("enc_layers", c_int32), ("enc_heads", c_int32), ("enc_kernel", c_int32), ("enc_window", c_int32),
        ("n_flows", c_int32), ("wn_layers", c_int32), ("wn_kernel", c_int32),
        ("gen_input", c_int32), ("gen_initial_channel", c_int32),
        ("n_ups", c_int32), ("up_rates", c_int32 * SVCB_MAX_UPS), ("up_kernels", c_int32 * SVCB_MAX_UPS),
        ("n_res", c_int32), ("res_kernels", c_int32 * SVCB_MAX_RES),
        ("res_dilations", (c_int32 * 3) * SVCB_MAX_RES),
        ("sampling_rate", c_int32), ("n_harmonics", c_int32), ("precision", c_int32),
    ]

    @classmethod
    def from_dict(cls, d: dict) -> "Config":
        c = cls()
        for k, v in d.items():
            if k in ("up_rates", "up_kernels", "res_kernels"):
                arr = getattr(c, k)
                for i, x in enumerate(v):
                    arr[i] = int(x)
            elif k == "res_dilations":
                for i, row in enumerate(v):
                    for j, x in enumerate(row):
                        c.res_dilations[i][j] = int(x)
            else:
                setattr(c, k, int(v))
        return c


class WhisperConfig(ctypes.Structure):
    _fields_ = [("n_mels", c_int32), ("n_ctx", c_int32), ("n_state", c_int32), ("n_head", c_int32),
                ("n_layer", c_int32)]


class IvfConfig(ctypes.Structure):
    _fields_ = [("d", c_int32), ("nlist", c_int32), ("nprobe", c_int32), ("pad_", c_int32), ("ntotal", c_int64)]


class TensorEntry(ctypes.Structure):
    _fields_ = [("name", c_char * 96), ("offset_bytes", c_uint64), ("numel", c_uint64)]


class Taps(ctypes.Structure):
    _fields_ = [("ptr", c_void_p * SVCB_TAP_COUNT)]


# name -> (restype, argtypes); mirrors include/svcb.h one to one
SIGNATURES = {
    "svcb_last_error": (c_char_p, []),
    "svcb_version": (c_int, []),
    "svcb_sizeof": (c_size_t, [c_int32]),
    "svcb_last_launch_count": (c_int64, []),
    "svcb_whisper_create": (c_int, [c_void_p, c_size_t, POINTER(TensorEntry), c_int32, POINTER(WhisperConfig), POINTER(c_void_p)]),
    "svcb_whisper_destroy": (None, [c_void_p]),
    "svcb_whisper_workspace_bytes": (c_size_t, [c_void_p, c_int32, c_int32]),
    "svcb_whisper_encode": (c_int, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_size_t, c_void_p]),
    "svcb_whisper_encode_ragged": (c_int, [c_void_p, c_void_p, POINTER(c_int32), c_void_p, c_int32, c_int32, c_void_p, c_size_t, c_void_p]),
    "svcb_hubert_create": (c_int, [c_void_p, c_size_t, POINTER(TensorEntry), c_int32, c_int32, POINTER(c_void_p)]),
    "svcb_hubert_destroy": (None, [c_void_p]),
    "svcb_hubert_frames": (c_int32, [c_int32]),
    "svcb_hubert_workspace_bytes": (c_size_t, [c_void_p, c_int32, c_int32]),
    "svcb_hubert_units": (c_int, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_size_t, c_void_p, c_int32, c_void_p]),
    "svcb_hubert_units_ragged": (c_int, [c_void_p, c_void_p, POINTER(c_int32), c_void_p, c_int32, c_int32, c_void_p, c_size_t, c_void_p]),
    "svcb_whisper_log_mel": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_void_p]),
    "svcb_whisper_log_mel_ragged": (c_int, [c_void_p, POINTER(c_int32), c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_void_p]),
    "svcb_linear_spec_ragged": (c_int, [c_void_p, POINTER(c_int64), c_int32, c_void_p, c_void_p, c_size_t, c_void_p]),
    "svcb_tacotron_mel": (c_int, [c_void_p, c_int32, c_int64, c_void_p, c_int32, c_void_p, c_void_p]),
    "svcb_resample_ragged": (c_int, [c_void_p, POINTER(c_int64), c_int32, c_int32, c_int32, c_void_p, c_int64, c_int64, c_void_p, c_void_p]),
    "svcb_pcm16_normalise_ragged": (c_int, [c_void_p, POINTER(c_int64), c_int32, c_void_p, c_void_p, c_void_p]),
    "svcb_cdc_ragged": (c_int, [c_void_p, POINTER(c_int64), c_int32, c_void_p, c_void_p]),
    "svcb_trim_silence_ragged": (c_int, [c_void_p, POINTER(c_int64), POINTER(c_int32), c_int32, c_void_p, c_void_p]),
    "svcb_world_f0_workspace_bytes": (c_size_t, [c_int64, c_int32]),
    "svcb_world_f0_ragged": (c_int, [c_void_p, POINTER(c_int64), c_int32, c_void_p, c_void_p, c_size_t, c_void_p]),
    "svcb_praat_f0_workspace_bytes": (c_size_t, [c_int64, c_int32]),
    "svcb_praat_f0_ragged": (c_int, [c_void_p, POINTER(c_int64), c_int32, c_void_p, c_void_p, c_size_t, c_void_p]),
    "svcb_salience_f0_workspace_bytes": (c_size_t, [c_int64, c_int32]),
    "svcb_salience_f0_ragged": (c_int, [c_void_p, POINTER(c_int64), c_int32] + [c_void_p] * 5 + [c_size_t, c_void_p]),
    "svcb_salience_dp_workspace_bytes": (c_size_t, [c_int64]),
    "svcb_salience_dp_ragged": (c_int, [c_void_p, POINTER(c_int64), c_int32, c_void_p, c_void_p, c_size_t, c_void_p]),
    "svcb_pyin_f0_workspace_bytes": (c_size_t, [c_int64, c_int32]),
    "svcb_pyin_f0_ragged": (c_int, [c_void_p, POINTER(c_int64), c_int32] + [c_void_p] * 7 + [c_size_t, c_void_p]),
    "svcb_pyin_dp_workspace_bytes": (c_size_t, [c_int64]),
    "svcb_pyin_dp_ragged": (c_int, [c_void_p, POINTER(c_int64), c_int32] + [c_void_p] * 3 + [c_size_t, c_void_p]),
    "svcb_ivf_create": (c_int, [c_void_p, c_size_t, POINTER(TensorEntry), c_int32, POINTER(IvfConfig), POINTER(c_void_p)]),
    "svcb_ivf_destroy": (None, [c_void_p]),
    "svcb_ivf_workspace_bytes": (c_size_t, [c_void_p, c_int32, c_int32]),
    "svcb_ivf_retrieve": (c_int, [c_void_p] * 5 + [c_int32, c_int32, c_float, c_void_p, c_size_t, c_void_p]),
    "svcb_kmeans_workspace_bytes": (c_size_t, [c_int32] * 4),
    "svcb_kmeans_pack": (c_int, [c_void_p] * 3 + [c_int32] * 2 + [c_void_p]),
    "svcb_kmeans_assign": (c_int, [c_void_p] * 6 + [c_int32] * 4 + [c_void_p, c_size_t, c_void_p]),
    "svcb_kmeans_update": (c_int, [c_void_p] * 6 + [c_int32] * 3 + [c_void_p, c_size_t, c_void_p]),
    "svcb_kmeans_split": (c_int, [c_void_p, c_void_p, c_int32, c_int32, c_void_p]),
    "svcb_speaker_create": (c_int, [c_void_p, c_size_t, POINTER(TensorEntry), c_int32, POINTER(c_void_p)]),
    "svcb_speaker_destroy": (None, [c_void_p]),
    "svcb_speaker_frames": (c_int32, [c_int64]),
    "svcb_speaker_workspace_bytes": (c_size_t, [c_void_p, c_int32, c_int64]),
    "svcb_speaker_mel": (c_int, [c_void_p, c_void_p, POINTER(c_int64), c_int32, c_void_p, c_void_p, c_size_t, c_void_p]),
    "svcb_speaker_embed": (c_int, [c_void_p, c_void_p, POINTER(c_int64), c_int32, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "svcb_vad_create": (c_int, [c_void_p, c_size_t, POINTER(TensorEntry), c_int32, POINTER(c_void_p)]),
    "svcb_vad_destroy": (None, [c_void_p]),
    "svcb_vad_windows": (c_int64, [c_int64]),
    "svcb_vad_workspace_bytes": (c_size_t, [c_void_p, c_int32, c_int64]),
    "svcb_vad_probs": (c_int, [c_void_p, c_void_p, POINTER(c_int64), c_int32, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "svcb_crepe_create": (c_int, [c_void_p, c_size_t, POINTER(TensorEntry), c_int32, c_int32, POINTER(c_void_p)]),
    "svcb_crepe_destroy": (None, [c_void_p]),
    "svcb_crepe_frames": (c_int64, [c_int64, c_int32]),
    "svcb_crepe_workspace_bytes": (c_size_t, [c_void_p, c_int64]),
    "svcb_crepe_frame": (c_int, [c_void_p, POINTER(c_int64), c_int32, c_int32, c_void_p, c_void_p, c_void_p]),
    "svcb_crepe_probs": (c_int, [c_void_p, c_void_p, POINTER(c_int64), c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "svcb_crepe_decode_workspace_bytes": (c_size_t, [c_int64]),
    "svcb_crepe_decode": (c_int, [c_void_p, POINTER(c_int64), c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "svcb_op_gemm_bf16_scratch_bytes": (c_size_t, [c_int32] * 3),
    "svcb_op_gemm_bf16": (c_int, [c_void_p] * 5 + [c_int32] * 6 + [POINTER(c_int32), c_void_p, c_size_t, c_void_p]),
    "svcb_op_attention_tc_bf16_scratch_bytes": (c_size_t, [c_int32] * 3),
    "svcb_op_attention_tc_bf16": (c_int, [c_void_p, c_void_p] + [c_int32] * 5 + [POINTER(c_int32), c_void_p, c_size_t, c_void_p]),
    "svcb_op_ln_rows": (c_int, [c_void_p] * 5 + [c_int32] * 3 + [c_void_p]),
    "svcb_op_im2col_s1_image": (c_int, [c_void_p, c_void_p] + [c_int32] * 3 + [c_void_p]),
    "svcb_op_im2col_rows_image": (c_int, [c_void_p, c_void_p, POINTER(c_int32)] + [c_int32] * 7 + [c_void_p, c_size_t, c_void_p]),
    "svcb_timing_enable": (None, [c_int32]),
    "svcb_timing_report": (c_char_p, []),
    "svcb_model_create": (c_int, [c_void_p, c_size_t, POINTER(TensorEntry), c_int32, POINTER(Config), POINTER(c_void_p)]),
    "svcb_model_destroy": (None, [c_void_p]),
    "svcb_workspace_bytes": (c_size_t, [c_void_p, c_int32, c_int32]),
    "svcb_source_workspace_bytes": (c_size_t, [c_void_p, c_int32, c_int32]),
    "svcb_source": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_size_t, c_void_p]),
    "svcb_source2wav": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p]),
    "svcb_prior": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_size_t, POINTER(Taps), c_void_p]),
    "svcb_flow": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_size_t, POINTER(Taps), c_void_p]),
    "svcb_generator": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_size_t, POINTER(Taps), c_void_p]),
    "svcb_infer": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_size_t, POINTER(Taps), c_void_p]),
    "svcb_infer_ragged": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_int32), c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_size_t, c_void_p]),
    "svcb_op_conv1d": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p] + [c_int32] * 9 + [c_void_p]),
    "svcb_op_snake_alias": (c_int, [c_void_p] * 6 + [c_int32] * 3 + [c_void_p]),
    "svcb_op_layernorm_c": (c_int, [c_void_p] * 5 + [c_int32] * 4 + [c_float, c_void_p]),
    "svcb_op_rel_attention": (c_int, [c_void_p] * 5 + [c_int32] * 5 + [c_void_p]),
    "svcb_op_rel_attention_tc_scratch_bytes": (c_size_t, [c_int32] * 3),
    "svcb_op_rel_attention_tc": (c_int, [c_void_p] * 5 + [c_int32] * 5 + [c_void_p, c_size_t, c_void_p]),
    "svcb_op_conv_tc": (c_int, [c_void_p] * 6 + [c_int32] * 9 + [c_void_p]),
    "svcb_op_amp_conv_tc_scratch_bytes": (c_size_t, [c_int32] * 3),
    "svcb_op_amp_conv_tc": (c_int, [c_void_p] * 9 + [c_int32] * 7 + [c_float, c_void_p, c_size_t, c_void_p]),
    "svcb_op_amp_s2d_link_scratch_bytes": (c_size_t, [c_int32] * 3),
    "svcb_op_amp_s2d_link": (c_int, [c_void_p] * 12 + [c_int32] * 6 + [c_void_p, c_size_t, c_void_p]),
    "svcb_op_amp_s2d_link_ragged": (c_int, [c_void_p] * 13 + [c_int32] * 6 + [c_void_p, c_size_t, c_void_p]),
    "svcb_op_tc_gemm_selftest": (c_int, [c_void_p, c_void_p, c_void_p] + [c_int32] * 4 + [c_void_p]),
}

_lib = None


def load():
    """Load libsvc_b200.so and bind every symbol of include/svcb.h.  Raises when the library is
    missing -- the product path has no CPU or PyTorch fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise SvcbError(f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                        "(make -C whisper-vits-svc_b200/csrc). There is no fallback path.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    for which, st in enumerate((Config, TensorEntry, Taps, IvfConfig)):
        if lib.svcb_sizeof(which) != ctypes.sizeof(st):
            raise SvcbError(f"ABI struct {st.__name__} size mismatch: C {lib.svcb_sizeof(which)} vs ctypes {ctypes.sizeof(st)}")
    _lib = lib
    return lib


def check(status: int, what: str):
    if status != 0:
        msg = load().svcb_last_error()
        raise SvcbError(f"{what} failed with status {status}: {msg.decode() if msg else ''}")


def last_launch_count() -> int:
    return int(load().svcb_last_launch_count())


def cuda_device(device) -> torch.device:
    """torch.device(device), or SvcbError when it is not a CUDA device."""
    dev = torch.device(device)
    if dev.type != "cuda":
        raise SvcbError(f"libsvc_b200 computes only on a CUDA (sm_90a) device, not {dev}; there is no CPU fallback")
    return dev


def stream() -> c_void_p:
    """The current device's current torch stream, as an svcb_stream."""
    return c_void_p(torch.cuda.current_stream().cuda_stream)


def call(name: str, *args, device=None) -> None:
    """svcb_<name>(*args, stream) on `device` (default: the current device) and its current stream."""
    with torch.cuda.device(device):
        st = getattr(load(), "svcb_" + name)(*args, stream())
    check(st, "svcb_" + name)


def offsets(lengths):
    """The prefix sums [0, l0, l0 + l1, ...] as a ctypes int64 array: a ragged batch's `*_offsets_host` argument."""
    o = [0]
    for n in lengths:
        o.append(o[-1] + int(n))
    return (c_int64 * len(o))(*o)


def ragged(clips, device):
    """1-D clips (numpy arrays, tensors or lists) -> (their float32 concatenation on `device`, offsets).  Clips already
    on the device are joined by one kernel.  Host clips are copied straight into their slices of the device buffer,
    since joining them on the host first is a few times slower."""
    xs = [(c.float() if torch.is_tensor(c) else torch.as_tensor(np.asarray(c, np.float32))).reshape(-1) for c in clips]
    offs = offsets(x.numel() for x in xs)
    if xs and all(x.is_cuda for x in xs):
        return torch.cat(xs).to(device), offs
    flat = torch.empty(offs[-1], dtype=torch.float32, device=device)
    for b, x in enumerate(xs):
        flat[offs[b]:offs[b + 1]].copy_(x)
    return flat, offs


def split(x, offs):
    """x cut at the offsets: one piece per item."""
    return [x[offs[b]:offs[b + 1]] for b in range(len(offs) - 1)]


class Handle:
    """A device model behind the C ABI: the packed blob (on a CUDA device) and the handle svcb_<kind>_create made from
    it, with one grow-only workspace.  The blob lives as long as the handle; dropping the Handle destroys both.  A
    Handle passes to any svcb_* function as the opaque handle pointer (ctypes reads `_as_parameter_`)."""

    def __init__(self, kind: str, table, blob: torch.Tensor, *create_args):
        self.kind, self._as_parameter_, self._ws = kind, None, None
        self.device = cuda_device(blob.device)
        entries = (TensorEntry * len(table))()
        for e, (name, off, numel) in zip(entries, table):
            e.name, e.offset_bytes, e.numel = name.encode(), off, numel
        args = [ctypes.byref(a) if isinstance(a, ctypes.Structure) else a for a in create_args]
        h = c_void_p()
        with torch.cuda.device(self.device):
            st = getattr(load(), f"svcb_{kind}_create")(blob.data_ptr(), blob.numel() * blob.element_size(), entries,
                                                        len(table), *args, ctypes.byref(h))
        check(st, f"svcb_{kind}_create")
        self.blob, self.table, self._as_parameter_ = blob, table, h

    def __del__(self):
        if self._as_parameter_ is not None:
            try:
                getattr(load(), f"svcb_{self.kind}_destroy")(self)
            except Exception:
                pass

    def workspace(self, nbytes: int) -> torch.Tensor:
        """A uint8 device buffer of at least nbytes.  It only grows; the old buffer is freed before the larger one is
        allocated, so the two are never held at once."""
        if self._ws is None or self._ws.numel() < nbytes:
            self._ws = None
            self._ws = torch.empty(int(nbytes), dtype=torch.uint8, device=self.device)
        return self._ws

    def call(self, name: str, *args) -> None:
        """svcb_<name>(handle, *args, stream) on the handle's device."""
        call(name, self, *args, device=self.device)
