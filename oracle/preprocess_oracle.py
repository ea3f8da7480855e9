"""CPU oracle for dataset PPG preparation (TEST INFRASTRUCTURE): prepare/preprocess_ppg.py:29-39 feeds the encoder
`log_mel_spectrogram(pad_or_trim(audio))` and keeps `ppg[:len(audio) // 320]`.  whisper_oracle restates the log-mel
and the encoder; this module restates `pad_or_trim` (whisper/audio.py:29-50) and imports the live one where the
reference tree exists, behind the librosa stub ref_import already uses."""
from __future__ import annotations

import numpy as np

N_SAMPLES = 30 * 16000   # whisper/audio.py:19


def pad_or_trim(array: np.ndarray, length_max: int = N_SAMPLES, length_min: int = N_SAMPLES // 2) -> np.ndarray:
    """whisper/audio.py:29-50 on numpy arrays along the last axis: keep the first length_max samples, then zero-pad at
    the end to length_min."""
    array = array[..., :length_max]
    short = length_min - array.shape[-1]
    if short > 0:
        array = np.concatenate([array, np.zeros(array.shape[:-1] + (short,), array.dtype)], axis=-1)
    return array


def reference_pad_or_trim():
    """The unmodified whisper/audio.py:pad_or_trim (raises where the reference tree is absent)."""
    from oracle import ref_import
    ref_import.import_whisper_model()     # stubs librosa, then imports whisper.model -> whisper.audio
    import whisper.audio as wa  # noqa
    return wa.pad_or_trim
