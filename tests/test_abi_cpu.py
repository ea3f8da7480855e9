"""The C-ABI library loads and exports every symbol include/svcb.h declares (no compute)."""
import os
import re

import pytest

from tests.util import ROOT
from whisper_vits_svc_b200 import _lib


def _declared():
    src = open(os.path.join(ROOT, "include", "svcb.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(svcb_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_exported_and_bound():
    names = _declared()
    assert "svcb_infer" in names and "svcb_model_create" in names
    lib = _lib.load()
    for n in names:
        assert hasattr(lib, n), f"{n} not exported by libsvc_b200.so"
        assert n in _lib.SIGNATURES, f"{n} has no ctypes signature in _lib.py"
    assert sorted(_lib.SIGNATURES) == names


def test_version_and_error_string():
    lib = _lib.load()
    assert lib.svcb_version() >= 100
    assert isinstance(lib.svcb_last_error(), (bytes, type(None)))


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(_lib.SvcbError):
        _lib.load()


def test_no_cpu_path():
    import torch
    from whisper_vits_svc_b200 import hparams, models
    hp = hparams.load_hparams(os.path.join(ROOT, "configs", "base.yaml"))
    m = models.SynthesizerInfer(513, 25, hp)
    if not torch.cuda.is_available():
        with pytest.raises(_lib.SvcbError):
            m.pitch2source(torch.zeros(1, 4))


def test_config_struct_layout_matches_header():
    import ctypes
    lib = _lib.load()
    assert ctypes.sizeof(_lib.Config) == lib.svcb_sizeof(0) == 4 * 52
    assert ctypes.sizeof(_lib.TensorEntry) == lib.svcb_sizeof(1) == 96 + 16
    assert ctypes.sizeof(_lib.Taps) == lib.svcb_sizeof(2) == 8 * _lib.SVCB_TAP_COUNT


def test_ragged_offsets_rejected_before_any_cuda_call():
    # Every check of the offsets runs on the host before the stream or a device pointer is touched, so no device is
    # needed: the data pointers below are dummies and the stream is null.
    import ctypes
    lib = _lib.load()
    d = 256

    def rejects(st, *parts):
        msg = lib.svcb_last_error().decode()
        assert st == -1, msg   # SVCB_E_BAD_SHAPE
        for p in parts:
            assert p in msg, msg

    o = _lib.offsets
    rejects(lib.svcb_linear_spec_ragged(d, o([1000]), 0, d, None, 0, None), "B = 0; need at least one item")
    rejects(lib.svcb_linear_spec_ragged(d, o([1000, 352]), 2, d, None, 0, None), "item 1 has 352 samples", "353")
    rejects(lib.svcb_resample_ragged(d, o([10, 0]), 2, 1, 2, d, 5, 0, d, None), "item 1 has 0 samples")
    neg = (ctypes.c_int64 * 3)(-1, 5, 10)
    rejects(lib.svcb_resample_ragged(d, neg, 2, 1, 2, d, 5, 0, d, None), "negative first offset")
    dec = (ctypes.c_int64 * 3)(0, 10, 4)
    rejects(lib.svcb_pcm16_normalise_ragged(d, dec, 2, d, d, None), "item 1 has -6 samples", "decrease")
    rejects(lib.svcb_pcm16_normalise_ragged(d, o([]), 0, d, d, None), "at least one item")


def test_ragged_host_packing():
    import ctypes
    import numpy as np
    import torch
    clips = [np.arange(3, dtype=np.float64), torch.ones(2, dtype=torch.float16), [], [5.0]]
    flat, offs = _lib.ragged(clips, "cpu")
    assert flat.dtype == torch.float32 and flat.tolist() == [0, 1, 2, 1, 1, 5]
    assert list(offs) == [0, 3, 5, 5, 6] and isinstance(offs, ctypes.c_int64 * 5)
    assert [p.tolist() for p in _lib.split(flat, offs)] == [[0, 1, 2], [1, 1], [], [5]]
    empty, eo = _lib.ragged([], "cpu")
    assert empty.shape == (0,) and list(eo) == [0]
