"""Silero VAD oracle (TEST INFRASTRUCTURE): a torch-CPU restatement of the 16 kHz branch of vad/assets/silero_vad.jit
from its state-dict tensors, with the reference's stateful loop over 512-sample windows, plus the hooks that compare it
with the live model and with the live `vad.utils.get_speech_timestamps`, and the fixture generator.

    python oracle/vad_oracle.py     # writes tests/golden/vad_*.npz; needs the reference tree (build container only)

Per window (the last one zero-padded to 512): reflect pad 96 -> 704 samples; STFT as conv1d with the [258, 1, 256]
basis at stride 64 (8 frames, rows 0..128 real, 129..257 imaginary); magnitude; s = log1p(mag 2^20), norm = s - the
frame mean of the 7-tap filtered, reflect-padded (3) bin mean; first_layer and the encoder (BatchNorm eval) on
cat([mag, norm]) down to one 64-d vector; one step of the 2-layer LSTM (state carried across windows, zero at the start
of each file); ReLU, conv 64 -> 1, sigmoid.
"""
from __future__ import annotations

import os
import sys
from typing import Dict, List

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")
WINDOW = 512
MODEL_NPZ = "vad_model"
FIXTURES = ("vad_test10s", "vad_synth")


# ------------------------------------------------------------------------------------------------ the restatement
def _block(sd, p, x, proj: bool):
    y = F.relu(F.conv1d(x, sd[f"{p}.dw_conv.0.weight"], sd[f"{p}.dw_conv.0.bias"], padding=2, groups=x.shape[1]))
    y = F.conv1d(y, sd[f"{p}.pw_conv.0.weight"], sd[f"{p}.pw_conv.0.bias"])
    r = F.conv1d(x, sd[f"{p}.proj.weight"], sd[f"{p}.proj.bias"]) if proj else x
    return F.relu(y + r)


def _conv_bn(sd, i, x, stride):
    y = F.conv1d(x, sd[f"encoder.{i}.weight"], sd[f"encoder.{i}.bias"], stride=stride)
    b = f"encoder.{i + 1}."
    y = F.batch_norm(y, sd[b + "running_mean"], sd[b + "running_var"], sd[b + "weight"], sd[b + "bias"], False, 0.0, 1e-5)
    return F.relu(y)


def front(sd: Dict[str, torch.Tensor], chunks: torch.Tensor) -> torch.Tensor:
    """[N, 512] windows (independent of each other) -> the encoder's [N, 64]."""
    x = F.pad(chunks[:, None, :], (96, 96), mode="reflect")
    ft = F.conv1d(x, sd["feature_extractor.forward_basis_buffer"], stride=64)
    re, im = ft[:, :129], ft[:, 129:]
    mag = torch.sqrt(re ** 2 + im ** 2)
    s = torch.log1p(mag * 1048576)
    m = s.mean(1, keepdim=True)
    m = torch.cat([m[..., 1:4].flip(-1), m, m[..., -4:-1].flip(-1)], -1)     # reflect pad by 3
    m = F.conv1d(m, sd["adaptive_normalization.filter_"]).mean(-1, keepdim=True)
    x = torch.cat([mag, s - m], 1)
    x = _block(sd, "first_layer.0", x, True)
    x = _conv_bn(sd, 0, x, 2)
    x = _block(sd, "encoder.3.0", x, True)
    x = _conv_bn(sd, 4, x, 2)
    x = _block(sd, "encoder.7.0", x, False)
    x = _conv_bn(sd, 8, x, 2)
    x = _block(sd, "encoder.11.0", x, True)
    x = _conv_bn(sd, 12, x, 1)
    return x[:, :, 0]


def lstm_step(sd, x, h, c):
    """One step of the 2-layer LSTM (gates i, f, g, o) and the decoder: x [N, 64], h, c [2, N, 64] -> prob [N], h, c."""
    hs, cs = [], []
    for l in range(2):
        g = (x @ sd[f"decoder.rnn.weight_ih_l{l}"].T + sd[f"decoder.rnn.bias_ih_l{l}"]
             + h[l] @ sd[f"decoder.rnn.weight_hh_l{l}"].T + sd[f"decoder.rnn.bias_hh_l{l}"])
        i, f, gg, o = g.chunk(4, 1)
        cn = torch.sigmoid(f) * c[l] + torch.sigmoid(i) * torch.tanh(gg)
        x = torch.sigmoid(o) * torch.tanh(cn)
        hs.append(x); cs.append(cn)
    y = F.conv1d(F.relu(x)[:, :, None], sd["decoder.decoder.1.weight"], sd["decoder.decoder.1.bias"])
    return torch.sigmoid(y)[:, 0, 0], torch.stack(hs), torch.stack(cs)


def chunks_of(wav) -> torch.Tensor:
    w = torch.as_tensor(np.asarray(wav, np.float32)).reshape(-1)
    n = -(-w.numel() // WINDOW)
    return F.pad(w, (0, n * WINDOW - w.numel())).reshape(n, WINDOW)


@torch.no_grad()
def speech_probs(sd: Dict[str, torch.Tensor], wav, per_window: bool = False):
    """One file -> (probs [W], encoder outputs [W, 64]).  per_window runs the whole model one window at a time, as
    the reference's loop calls it; otherwise the (independent) front ends run as one batch and only the LSTM loops."""
    ch = chunks_of(wav)
    h = c = torch.zeros(2, 1, 64)
    probs, encs = [], []
    enc_all = None if per_window else front(sd, ch)
    for i in range(ch.shape[0]):
        e = front(sd, ch[i:i + 1]) if per_window else enc_all[i:i + 1]
        p, h, c = lstm_step(sd, e, h, c)
        probs.append(p)
        encs.append(e)
    if not probs:
        return np.zeros(0, np.float32), np.zeros((0, 64), np.float32)
    return torch.cat(probs).numpy(), torch.cat(encs).numpy()


# ------------------------------------------------------------------------------------------------ model files
def write_jit(path: str, sd: Dict[str, torch.Tensor], filter_length=256, hop_length=64, to_pad=3):
    """A TorchScript container with silero_vad.jit's `_model.*` tensor names and STFT / normalisation attributes (no
    model code): what `vad_infer.read_model` reads."""
    root = _Container()
    inner = torch.nn.Module()
    root.add_module("_model", inner)
    for key, t in sd.items():
        mod = inner
        *path_, name = key.split(".")
        for p in path_:
            if not hasattr(mod, p):
                mod.add_module(p, torch.nn.Module())
            mod = getattr(mod, p)
        mod.register_buffer(name, torch.as_tensor(t).clone())
    for attr, mod_name, v in (("filter_length", "feature_extractor", filter_length), ("hop_length", "feature_extractor", hop_length),
                              ("to_pad", "adaptive_normalization", to_pad)):
        if hasattr(inner, mod_name):
            setattr(getattr(inner, mod_name), attr, v)
    torch.jit.script(root).save(path)


class _Container(torch.nn.Module):
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return x


def load_tensors() -> Dict[str, torch.Tensor]:
    z = np.load(os.path.join(GOLDEN, MODEL_NPZ + ".npz"))
    return {k: torch.from_numpy(z[k]) for k in z.files}


def load_golden(name: str) -> dict:
    return dict(np.load(os.path.join(GOLDEN, name + ".npz")))


def clips(g: dict) -> List[str]:
    """The clip names of a fixture: keys `<clip>.wav`."""
    return sorted(k[:-4] for k in g if k.endswith(".wav"))


# ------------------------------------------------------------------------------------------------ live reference
def ref_model_path() -> str:
    from oracle import ref_import
    return os.path.join(ref_import.REF_ROOT, "vad", "assets", "silero_vad.jit")


def live_model():
    return torch.jit.load(ref_model_path(), map_location="cpu").eval()


@torch.no_grad()
def live_probs(model, wav):
    """The reference's loop (vad/utils.py:253-268) on the live model -> (probs [W], encoder outputs [W, 64])."""
    model.reset_states()
    ch = chunks_of(wav)
    probs = [model(ch[i], 16000).item() for i in range(ch.shape[0])]
    mm = model._model
    if ch.shape[0] == 0:
        return np.zeros(0, np.float32), np.zeros((0, 64), np.float32)
    mag = mm.feature_extractor(ch)
    enc = mm.encoder(mm.first_layer(torch.cat([mag, mm.adaptive_normalization(mag)], 1)))
    return np.array(probs, np.float32), enc[:, :, 0].numpy()


def import_vad_utils():
    from oracle import ref_import
    ref_import._ensure_path()
    import vad.utils as U
    return U


class ScriptedProbs:
    """Stands in for the model in get_speech_timestamps: returns the given probabilities in order."""

    def __init__(self, probs):
        self.probs = [float(p) for p in probs]

    def reset_states(self):
        self.i = 0

    def __call__(self, chunk, sr):
        p = self.probs[self.i]
        self.i += 1
        return torch.tensor([[p]])


def reference_timestamps(probs, n_samples: int, **kw) -> List[dict]:
    """The live vad.utils.get_speech_timestamps driven by scripted probabilities (one per 512-sample window)."""
    U = import_vad_utils()
    assert len(probs) == -(-n_samples // WINDOW)
    return U.get_speech_timestamps(torch.zeros(n_samples), ScriptedProbs(probs), sampling_rate=16000, **kw)


# ------------------------------------------------------------------------------------------------ fixtures
THRESHOLDS = (0.2, 0.05)    # the CLI's threshold and its release point threshold - 0.15


def margin(probs) -> float:
    p = np.asarray(probs, np.float64)
    return float(min(np.abs(p - t).min() for t in THRESHOLDS)) if p.size else float("inf")


def synth_clips(seed: int = 5) -> Dict[str, np.ndarray]:
    """Tone and noise bursts separated by silences of several lengths, silence, and lengths around one window."""
    rng = np.random.default_rng(seed)
    t = lambda n: np.arange(n) / 16000.0   # noqa: E731
    parts = []
    for burst, gap in ((0.6, 0.05), (0.3, 0.15), (1.2, 0.4), (0.2, 0.08), (0.8, 1.0)):
        n = int(burst * 16000)
        parts.append((0.3 * np.sin(2 * np.pi * 220 * t(n)) * (1 + 0.5 * np.sin(2 * np.pi * 4 * t(n)))
                      + 0.05 * rng.standard_normal(n)).astype(np.float32))
        parts.append(np.zeros(int(gap * 16000), np.float32))
        n = int(0.5 * burst * 16000)
        parts.append((0.2 * rng.standard_normal(n)).astype(np.float32))
        parts.append((1e-4 * rng.standard_normal(int(gap * 16000))).astype(np.float32))
    out = {"bursts": np.concatenate(parts), "zeros": np.zeros(16000 * 2 + 77, np.float32)}
    for n in (1, 511, 512, 513):
        out[f"len{n}"] = (0.3 * rng.standard_normal(n)).astype(np.float32)
    return out


def test_wav_16k() -> np.ndarray:
    from whisper_vits_svc_b200.whisper_infer import load_audio
    from oracle import ref_import
    return load_audio(os.path.join(ref_import.REF_ROOT, "test.wav"), 16000)


def excerpt(wav: np.ndarray, seconds: float = 10.0) -> np.ndarray:
    """The ~10 s excerpt of test.wav with speech and silence whose live probabilities stay farthest from both
    thresholds (start on a window boundary, candidates every 2 s)."""
    model = live_model()
    n = int(seconds * 16000) // WINDOW * WINDOW + 123
    best = None
    for s in range(0, wav.shape[0] - n, 32 * WINDOW * 2):
        x = wav[s:s + n]
        p, _ = live_probs(model, x)
        if (p > 0.5).mean() < 0.2 or (p < 0.05).mean() < 0.1:
            continue
        if best is None or margin(p) > best[0]:
            best = (margin(p), s)
    return wav[best[1]:best[1] + n]


def vad_case(name: str, wavs: Dict[str, np.ndarray], sd: Dict[str, torch.Tensor], model):
    """tests/golden/<name>.npz: per clip the audio, the live probabilities and encoder outputs, the live
    get_speech_timestamps(threshold=0.2) as [k, 2] and the probabilities' smallest distance to 0.2 and 0.05."""
    out = {}
    for clip, w in wavs.items():
        p, e = live_probs(model, w)
        po, eo = speech_probs(sd, w)
        if p.size:
            print(f"{name}/{clip}: {p.size} windows, oracle max-abs prob {np.abs(po - p).max():.2e} enc {np.abs(eo - e).max():.2e}, "
                  f"margin {margin(p):.2e}")
        ts = reference_timestamps(p, w.shape[0], threshold=0.2) if p.size else []
        out[f"{clip}.wav"] = w.astype(np.float32)
        out[f"{clip}.probs"] = p
        out[f"{clip}.enc"] = e.astype(np.float32)
        out[f"{clip}.ts"] = np.array([[t["start"], t["end"]] for t in ts], np.int64).reshape(-1, 2)
        out[f"{clip}.margin"] = np.float64(margin(p))
    np.savez_compressed(os.path.join(GOLDEN, name + ".npz"), **out)


if __name__ == "__main__":
    torch.set_num_threads(8)
    model = live_model()
    sd = {k[len("_model."):]: v.clone() for k, v in model.state_dict().items()
          if k.startswith("_model.") and not k.endswith("num_batches_tracked")}
    np.savez_compressed(os.path.join(GOLDEN, MODEL_NPZ + ".npz"), **{k: v.numpy() for k, v in sd.items()})
    vad_case("vad_test10s", {"test10s": excerpt(test_wav_16k())}, sd, model)
    vad_case("vad_synth", synth_clips(), sd, model)
