"""Speaker encoder oracle (TEST INFRASTRUCTURE): what the reference's speaker/infer.py computes, restated where its
dependencies (librosa, pyworld, soundfile, fsspec) are absent.

* `stft_magnitude`, `trim`, `load_wav`: float64 numpy restatements of librosa 0.10.1's `stft` (center, reflect,
  periodic Hann), `effects.trim` (float32 RMS as librosa computes it) and `load` for 16 kHz PCM wavs.  They are pinned
  independently in the tests: the STFT against torch.stft, the mel basis (whisper_oracle.slaney_mel_filterbank) against
  transformers' mel_filter_bank, trim against signals with known boundaries.
* `melspectrogram`: AudioProcessor.melspectrogram in float64 like the reference (lfilter returns float64).
* `compute_embedding`: LSTMSpeakerEncoder.compute_embedding as a functional torch-CPU fp32 restatement.
* `import_reference`: the UNMODIFIED speaker/models/lstm.py and speaker/utils/audio.py behind stub librosa / pyworld /
  soundfile / fsspec modules whose librosa answers filters.mel, stft, effects.trim and load from this module.
* `python -m oracle.speaker_oracle` writes tests/golden/speaker_*.npz from the reference's own load_wav ->
  melspectrogram -> compute_embedding (needs the reference tree).
"""
from __future__ import annotations

import importlib
import importlib.machinery
import os
import re
import json
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
SR, N_FFT, HOP, N_MELS = 16000, 1024, 256, 80
AUDIO = dict(preemphasis=0.98, ref_level_db=20.0, min_level_db=-100.0, max_norm=4.0)


# ------------------------------------------------------------------------------------------------ front end
def stft_magnitude(y: np.ndarray, n_fft: int = N_FFT, hop: int = HOP) -> np.ndarray:
    """|librosa.stft(y, n_fft, hop, win_length=n_fft, window="hann", center=True, pad_mode="reflect")| -> [1 + n_fft/2, T]."""
    y = np.asarray(y, np.float64)
    yp = np.pad(y, (n_fft // 2, n_fft // 2), mode="reflect")
    T = 1 + (yp.shape[0] - n_fft) // hop
    frames = np.lib.stride_tricks.sliding_window_view(yp, n_fft)[::hop][:T]
    win = 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(n_fft) / n_fft)   # periodic Hann (scipy get_window fftbins=True)
    return np.abs(np.fft.rfft(frames * win, axis=-1)).T


def mel_basis(n_mels: int = N_MELS, sr: int = SR, n_fft: int = N_FFT) -> np.ndarray:
    """librosa.filters.mel(sr, n_fft, n_mels, fmin=0, fmax=sr/2): Slaney scale and area norm, [n_mels, 1 + n_fft/2]."""
    from oracle import whisper_oracle
    return whisper_oracle.slaney_mel_filterbank(n_mels, sr, n_fft)


def melspectrogram(y: np.ndarray, audio: dict = AUDIO) -> np.ndarray:
    """AudioProcessor.melspectrogram (audio.py:561-571) with signal_norm, symmetric_norm and clip_norm: -> [80, T] f32."""
    from scipy.signal import lfilter
    y = np.asarray(y)
    if audio["preemphasis"] != 0:
        y = lfilter([1, -audio["preemphasis"]], [1], y)
    S = 20.0 * np.log10(np.maximum(1e-5, mel_basis() @ stft_magnitude(y)))
    S = S - audio["ref_level_db"]
    S = (S - audio["min_level_db"]) / (-audio["min_level_db"])
    S = 2 * audio["max_norm"] * S - audio["max_norm"]
    return np.clip(S, -audio["max_norm"], audio["max_norm"]).astype(np.float32)


def trim(y: np.ndarray, top_db: float = 60, frame_length: int = N_FFT, hop_length: int = HOP):
    """librosa.effects.trim -> (y[start:end], [start, end])."""
    y = np.asarray(y)
    yp = np.pad(y, (frame_length // 2, frame_length // 2), mode="constant")
    T = 1 + (yp.shape[0] - frame_length) // hop_length
    x = np.lib.stride_tricks.sliding_window_view(yp, frame_length)[::hop_length][:T].astype(np.float32)
    rms = np.sqrt(np.mean(x * x, axis=-1, dtype=np.float32))
    db = 10.0 * np.log10(np.maximum(np.float32(1e-10), rms * rms)) - 10.0 * np.log10(np.maximum(np.float32(1e-10), rms.max() ** 2))
    nz = np.flatnonzero(db > -top_db)
    start, end = (int(nz[0]) * hop_length, min(y.shape[-1], (int(nz[-1]) + 1) * hop_length)) if nz.size else (0, 0)
    return y[start:end], np.asarray([start, end])


def load_wav(path: str, sr: int = SR):
    """librosa.load(path, sr=16000) for a 16 kHz PCM wav: mono float32 in [-1, 1)."""
    from scipy.io import wavfile
    rate, x = wavfile.read(path)
    assert rate == sr, "the fixtures are 16 kHz"
    x = x.astype(np.float32) / np.float32(np.iinfo(x.dtype).max + 1) if x.dtype.kind == "i" else x.astype(np.float32)
    return (x.mean(axis=1) if x.ndim > 1 else x), sr


def prepare(x: np.ndarray, top_db: float = 60) -> np.ndarray:
    """AudioProcessor.load_wav after reading: 160-sample margin, trim, x / max|x| * 0.95."""
    x = trim(x[160:-160], top_db)[0]
    return x / abs(x).max() * 0.95


# ------------------------------------------------------------------------------------------------ LSTM
def window_offsets(T: int, num_frames: int = 250, num_eval: int = 10):
    L = min(num_frames, T)
    return [int(o) for o in np.linspace(0, T - L, num=num_eval)], L


@torch.no_grad()
def compute_embedding(sd: dict, mel: np.ndarray):
    """mel [T, 80] -> (embedding [256], window embeddings [10, 256]), fp32 on the CPU (lstm.py:8-20,58-101)."""
    x = torch.as_tensor(np.asarray(mel, np.float32))
    offs, L = window_offsets(x.shape[0])
    h_in = torch.stack([x[o:o + L] for o in offs])          # [10, L, 80]
    for l in range(3):
        p = f"layers.{l}."
        wih, whh = sd[p + "lstm.weight_ih_l0"].float(), sd[p + "lstm.weight_hh_l0"].float()
        b = sd[p + "lstm.bias_ih_l0"].float() + sd[p + "lstm.bias_hh_l0"].float()
        H = whh.shape[1]
        gx = h_in @ wih.T + b
        h = torch.zeros(h_in.shape[0], H)
        c = torch.zeros(h_in.shape[0], H)
        outs = []
        for t in range(L):
            i, f, g, o = (gx[:, t] + h @ whh.T).split(H, dim=1)
            c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
            h = torch.sigmoid(o) * torch.tanh(c)
            outs.append(h)
        h_in = torch.stack(outs, 1) @ sd[p + "linear.weight"].float().T
    d = torch.nn.functional.normalize(h_in[:, -1], p=2, dim=1)
    return d.mean(0).numpy(), d.numpy()


# ------------------------------------------------------------------------------------------------ the reference
def _module(name):
    m = types.ModuleType(name)
    m.__spec__ = importlib.machinery.ModuleSpec(name, loader=None)
    return m


def import_reference(monkeypatch=None):
    """-> (speaker.models.lstm, speaker.utils.audio) imported unmodified with stub librosa / pyworld / soundfile / fsspec.
    Pass pytest's monkeypatch so the stubs and the imported modules leave sys.modules after the test."""
    from oracle import ref_import
    ref_import._ensure_path()
    put = monkeypatch.setitem if monkeypatch else (lambda mp, k, v: mp.__setitem__(k, v))
    drop = monkeypatch.delitem if monkeypatch else (lambda mp, k: mp.__delitem__(k))
    lib = _module("librosa")
    lib.filters = _module("librosa.filters")
    lib.effects = _module("librosa.effects")
    lib.filters.mel = lambda sr, n_fft, n_mels, fmin=0.0, fmax=None, **_: (
        mel_basis(n_mels, sr, n_fft) if fmin == 0 and fmax in (None, sr / 2) else None)
    lib.stft = lambda y, n_fft, hop_length, win_length, pad_mode, window, center: (
        stft_magnitude(y, n_fft, hop_length).astype(np.complex128))   # only |D| is read
    lib.effects.trim = lambda y, top_db, frame_length, hop_length: trim(y, top_db, frame_length, hop_length)
    lib.load = lambda path, sr: load_wav(path, sr)
    stubs = {"librosa": lib, "librosa.filters": lib.filters, "librosa.effects": lib.effects,
             "pyworld": _module("pyworld"), "soundfile": _module("soundfile")}
    try:
        import fsspec  # noqa: F401
    except ImportError:
        stubs["fsspec"] = _module("fsspec")
    for k, v in stubs.items():
        put(sys.modules, k, v)
    for name in [n for n in sys.modules if n == "speaker" or n.startswith("speaker.")]:
        drop(sys.modules, name)
    lstm = importlib.import_module("speaker.models.lstm")
    audio = importlib.import_module("speaker.utils.audio")
    for name in [n for n in sys.modules if n == "speaker" or n.startswith("speaker.")]:
        put(sys.modules, name, sys.modules[name])
    return lstm, audio


def reference_config() -> dict:
    from oracle import ref_import
    with open(os.path.join(ref_import.REF_ROOT, "speaker_pretrain", "config.json"), encoding="utf-8") as f:
        return json.loads(re.sub(r"//.*\n", "\n", f.read()))


def reference_embedding(lstm, audio, sd: dict, wav_path: str, windows: bool = False):
    """speaker/infer.py:80-98 through the unmodified modules: -> (mel [T, 80], embedding [256], window embeddings)."""
    ap = audio.AudioProcessor(**reference_config()["audio"], verbose=False)
    ap.do_sound_norm = True
    ap.do_trim_silence = True
    spec = ap.melspectrogram(ap.load_wav(wav_path, sr=ap.sample_rate))
    enc = lstm.LSTMSpeakerEncoder(80, 256, 768, 3)
    enc.load_state_dict(sd)
    enc.eval()
    x = torch.from_numpy(spec.T).unsqueeze(0)
    with torch.no_grad():
        emb = enc.compute_embedding(x).numpy().squeeze()
        win = enc.compute_embedding(x, return_mean=False).numpy()
    return spec.T.copy(), emb, win


# ------------------------------------------------------------------------------------------------ goldens
SPEAKER_CASES = {   # name: (seed, seconds of voice, seconds of near-silence at each end)
    "speaker_short_trim": (71, 2.5, 0.4),
    "speaker_10s": (72, 160400 / SR, 0.0),
}


def synth_voice(seed: int, seconds: float, quiet: float) -> np.ndarray:
    """A vowel-like int16 clip: a gliding harmonic tone with vibrato and a little noise, near-silent ends (about -94 dBFS)."""
    rng = np.random.default_rng(seed)
    n = int(round(seconds * SR))
    t = np.arange(n) / SR
    f0 = 140 + 40 * np.sin(2 * np.pi * 0.3 * t) + 4 * np.sin(2 * np.pi * 5.5 * t)
    ph = 2 * np.pi * np.cumsum(f0) / SR
    v = sum((0.5 / k) * np.sin(k * ph + rng.uniform(0, 2 * np.pi)) for k in range(1, 16))
    v *= 0.6 + 0.4 * np.sin(2 * np.pi * 1.7 * t) ** 2
    v += 0.01 * rng.standard_normal(n)
    q = int(round(quiet * SR))
    x = np.concatenate([2e-5 * rng.standard_normal(q), 0.5 * v / np.abs(v).max(), 2e-5 * rng.standard_normal(q)])
    return np.round(x * 32767).astype(np.int16)


def speaker_case(name):
    import tempfile
    from scipy.io import wavfile
    from whisper_vits_svc_b200 import synth
    seed, sec, quiet = SPEAKER_CASES[name]
    wav = synth_voice(seed, sec, quiet)
    sd = synth.speaker_checkpoint(seed)["model"]
    lstm, audio = import_reference()
    with tempfile.TemporaryDirectory() as tmp:
        p = os.path.join(tmp, "x.wav")
        wavfile.write(p, SR, wav)
        mel, emb, win = reference_embedding(lstm, audio, sd, p)
    np.savez_compressed(os.path.join(GOLDEN, name + ".npz"), wav=wav, mel=mel.astype(np.float32), windows=win.astype(np.float32),
                        embedding=emb.astype(np.float32), seed=np.int64(seed))
    print(name, "samples", wav.shape[0], "frames", mel.shape[0])


def load_golden(name):
    return dict(np.load(os.path.join(GOLDEN, name + ".npz")))


if __name__ == "__main__":
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    for case in SPEAKER_CASES:
        speaker_case(case)
