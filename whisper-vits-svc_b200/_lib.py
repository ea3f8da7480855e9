"""ctypes binding of libsvc_b200.so (the C ABI in include/svcb.h).

There is no fallback: if the library is missing or a call fails, a SvcbError is raised.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char, c_char_p, c_float, c_int, c_int16, c_int32, c_int64, c_size_t, c_uint64, c_void_p

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
    "svcb_hubert_create": (c_int, [c_void_p, c_size_t, POINTER(TensorEntry), c_int32, c_int32, POINTER(c_void_p)]),
    "svcb_hubert_destroy": (None, [c_void_p]),
    "svcb_hubert_frames": (c_int32, [c_int32]),
    "svcb_hubert_workspace_bytes": (c_size_t, [c_void_p, c_int32, c_int32]),
    "svcb_hubert_units": (c_int, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_size_t, c_void_p, c_int32, c_void_p]),
    "svcb_whisper_log_mel": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_void_p]),
    "svcb_ivf_create": (c_int, [c_void_p, c_size_t, POINTER(TensorEntry), c_int32, POINTER(IvfConfig), POINTER(c_void_p)]),
    "svcb_ivf_destroy": (None, [c_void_p]),
    "svcb_ivf_workspace_bytes": (c_size_t, [c_void_p, c_int32, c_int32]),
    "svcb_ivf_retrieve": (c_int, [c_void_p] * 5 + [c_int32, c_int32, c_float, c_void_p, c_size_t, c_void_p]),
    "svcb_speaker_create": (c_int, [c_void_p, c_size_t, POINTER(TensorEntry), c_int32, POINTER(c_void_p)]),
    "svcb_speaker_destroy": (None, [c_void_p]),
    "svcb_speaker_frames": (c_int32, [c_int64]),
    "svcb_speaker_workspace_bytes": (c_size_t, [c_void_p, c_int32, c_int64]),
    "svcb_speaker_mel": (c_int, [c_void_p, c_void_p, POINTER(c_int64), c_int32, c_void_p, c_void_p, c_size_t, c_void_p]),
    "svcb_speaker_embed": (c_int, [c_void_p, c_void_p, POINTER(c_int64), c_int32, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "svcb_op_gemm_bf16_scratch_bytes": (c_size_t, [c_int32] * 3),
    "svcb_op_gemm_bf16": (c_int, [c_void_p] * 5 + [c_int32] * 4 + [c_void_p, c_size_t, c_void_p]),
    "svcb_op_attention_tc_bf16_scratch_bytes": (c_size_t, [c_int32] * 3),
    "svcb_op_attention_tc_bf16": (c_int, [c_void_p, c_void_p] + [c_int32] * 5 + [c_void_p, c_size_t, c_void_p]),
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
    "svcb_op_conv1d": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p] + [c_int32] * 9 + [c_void_p]),
    "svcb_op_snake_alias": (c_int, [c_void_p] * 6 + [c_int32] * 3 + [c_void_p]),
    "svcb_op_layernorm_c": (c_int, [c_void_p] * 5 + [c_int32] * 4 + [c_float, c_void_p]),
    "svcb_op_rel_attention": (c_int, [c_void_p] * 5 + [c_int32] * 5 + [c_void_p]),
    "svcb_op_rel_attention_tc_scratch_bytes": (c_size_t, [c_int32] * 3),
    "svcb_op_rel_attention_tc": (c_int, [c_void_p] * 5 + [c_int32] * 5 + [c_void_p, c_size_t, c_void_p]),
    "svcb_op_conv_tc": (c_int, [c_void_p] * 6 + [c_int32] * 9 + [c_void_p]),
    "svcb_op_amp_conv_tc_scratch_bytes": (c_size_t, [c_int32] * 3),
    "svcb_op_amp_conv_tc": (c_int, [c_void_p] * 9 + [c_int32] * 6 + [c_void_p, c_size_t, c_void_p]),
    "svcb_op_amp_s2d_link_scratch_bytes": (c_size_t, [c_int32] * 3),
    "svcb_op_amp_s2d_link": (c_int, [c_void_p] * 12 + [c_int32] * 5 + [c_void_p, c_size_t, c_void_p]),
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
