"""H100-native SVC inference hot path behind the reference's Python surface.

Sub-modules are imported lazily by name so that host-only helpers (hparams, synth, hostio)
work without the CUDA library; anything that computes goes through `_lib` and fails loudly
when `libsvc_b200.so` is missing."""
__version__ = "0.1.0"
