"""fp32 torch-CPU restatement of the reference's CREPE pitch path (TEST INFRASTRUCTURE): `crepe.predict` as
`pitch/inference.py:74-99` and `prepare/preprocess_crepe.py:11-44` call it, with the two random draws (`noise`, `dither`)
as inputs.  librosa is not installed, so `viterbi` restates `librosa.sequence.viterbi` in float64; `import_reference()`
loads the unmodified `crepe` package behind stub `librosa` / `resampy` modules whose `librosa.sequence.viterbi` is that
restatement.  `python -m oracle.crepe_oracle` writes the goldens under tests/golden/ (needs the reference tree).
"""
from __future__ import annotations

import io
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

from . import ref_import

PITCH_BINS, WINDOW, CENTS_PER_BIN, SEGMENT = 360, 1024, 20, 512
BN_EPS = 0.0010000000474974513
GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


# ------------------------------------------------------------------------------------------------ 1-2: input, framing
def frames(audio: torch.Tensor, hop: int, noise: torch.Tensor | None = None) -> torch.Tensor:
    """crepe/core.py:626-702 (pad = True) on audio + 0.001 noise: [1 + n // hop, 1024]."""
    audio = audio.float().reshape(-1)
    if noise is not None:
        audio = audio + noise.float().reshape(-1) * 0.001
    total = 1 + audio.numel() // hop
    x = F.pad(audio, (WINDOW // 2, WINDOW // 2))
    idx = (torch.arange(total) * hop)[:, None] + torch.arange(WINDOW)[None]
    fr = x[idx].clone()
    fr -= fr.mean(dim=1, keepdim=True)
    fr /= torch.max(torch.tensor(1e-10), fr.std(dim=1, keepdim=True))
    return fr


# ------------------------------------------------------------------------------------------------ 3: the network
def network(sd, fr: torch.Tensor, layers: bool = False):
    """crepe/model.py:94-134 -> sigmoid outputs [F, 360] (and the six pooled layer outputs [F, C, P])."""
    x = fr[:, None, :, None]
    outs = []
    for i in range(6):
        p = f"conv{i + 1}"
        x = F.pad(x, (0, 0, 254, 254) if i == 0 else (0, 0, 31, 32))
        x = F.conv2d(x, sd[p + ".weight"], sd[p + ".bias"], stride=(4, 1) if i == 0 else (1, 1))
        x = F.relu(x)
        x = F.batch_norm(x, sd[p + "_BN.running_mean"], sd[p + "_BN.running_var"], sd[p + "_BN.weight"], sd[p + "_BN.bias"],
                         False, 0.0, BN_EPS)
        x = F.max_pool2d(x, (2, 1), (2, 1))
        outs.append(x.squeeze(-1))
    feat = x.permute(0, 2, 1, 3).reshape(fr.shape[0], -1)
    probs = torch.sigmoid(F.linear(feat, sd["classifier.weight"], sd["classifier.bias"]))
    return (probs, outs) if layers else probs


# ------------------------------------------------------------------------------------------------ 4: range mask
def frequency_to_bins(f: float, ceil: bool = False) -> int:
    b = (1200 * torch.log2(torch.tensor(float(f)) / 10.0) - 1997.3794084376191) / CENTS_PER_BIN
    return int((torch.ceil(b) if ceil else torch.floor(b)).int())


def mask(probs: torch.Tensor, fmin: float = 50.0, fmax: float = 1000.0) -> torch.Tensor:
    probs = probs.clone()
    probs[:, :frequency_to_bins(fmin)] = -float("inf")
    probs[:, frequency_to_bins(fmax, True):] = -float("inf")
    return probs


# ------------------------------------------------------------------------------------------------ 5: Viterbi
def transition_matrix(n: int = PITCH_BINS) -> np.ndarray:
    xx, yy = np.meshgrid(range(n), range(n))
    t = np.maximum(12 - abs(xx - yy), 0)
    return t / t.sum(axis=1, keepdims=True)


def viterbi(prob: np.ndarray, transition: np.ndarray, p_init: np.ndarray | None = None) -> np.ndarray:
    """librosa.sequence.viterbi(prob [S, T], transition [S, S]) in float64: uniform start, logs as log(x + tiny) with the
    tiny of prob's dtype, np.argmax's first maximum on ties."""
    S, T = prob.shape
    tiny = float(np.finfo(prob.dtype).tiny) if np.issubdtype(prob.dtype, np.floating) else float(np.finfo(np.float32).tiny)
    log_trans = np.log(transition.astype(np.float64) + tiny)
    log_prob = np.log(prob.T.astype(np.float64) + tiny)
    p_init = np.full(S, 1.0 / S) if p_init is None else p_init
    value = np.zeros((T, S))
    ptr = np.zeros((T, S), dtype=np.int64)
    value[0] = log_prob[0] + np.log(p_init + tiny)
    for t in range(1, T):
        trans_out = value[t - 1][None, :] + log_trans.T     # [to, from]
        ptr[t] = np.argmax(trans_out, axis=1)
        value[t] = log_prob[t] + trans_out[np.arange(S), ptr[t]]
    states = np.zeros(T, dtype=np.int64)
    states[-1] = np.argmax(value[-1])
    for t in range(T - 2, -1, -1):
        states[t] = ptr[t + 1, states[t + 1]]
    return states


def decode(masked: torch.Tensor, dither: torch.Tensor | None = None, segment: int = SEGMENT):
    """crepe/decode.py:55-80 + crepe/convert.py:12-33 + crepe/core.py:710-722 per segment of `segment` frames, as
    crepe.predict's batch loop applies them -> (bins int64, pitch Hz fp32, periodicity fp32), each [F]."""
    trans = transition_matrix()
    bins = []
    for s in range(0, masked.shape[0], segment):
        p = torch.softmax(masked[s:s + segment].T[None], dim=1)[0]
        bins.append(torch.from_numpy(viterbi(p.numpy(), trans)))
    bins = torch.cat(bins)
    cents = CENTS_PER_BIN * bins + 1997.3794084376191
    if dither is not None:
        cents = cents + dither.float().reshape(-1)
    pitch = 10 * 2 ** (cents / 1200)
    return bins, pitch, masked.gather(1, bins[:, None]).reshape(-1)


def predict(sd, audio, hop: int, noise=None, dither=None):
    """-> (masked sigmoid outputs [F, 360], bins, pitch, periodicity)."""
    masked = mask(network(sd, frames(audio, hop, noise)))
    return (masked,) + decode(masked, dither)


# ------------------------------------------------------------------------------------------------ 7-8: filters, callers
def mean(x: np.ndarray, win: int) -> np.ndarray:
    """crepe/filter.py:10-56 on one vector."""
    x = np.asarray(x, np.float32)
    out = np.empty_like(x)
    for i in range(len(x)):
        w = x[max(0, i - win // 2):i + win // 2 + 1]
        ok = ~np.isnan(w)
        out[i] = np.float32(w[ok].sum(dtype=np.float32)) / np.float32(max(int(ok.sum()), 1))
    out[out == 0] = np.nan
    return out


def median(x: np.ndarray, win: int) -> np.ndarray:
    """crepe/filter.py:59-106 on one vector: reflect-padded values, validity zero outside, the lower median."""
    x = np.asarray(x, np.float32)
    pad = win // 2
    ok = np.pad(~np.isnan(x), pad)
    xp = np.pad(np.where(np.isnan(x), np.float32(0), x), pad, mode="reflect")
    out = np.empty_like(x)
    for i in range(len(x)):
        v = np.sort(xp[i:i + win][ok[i:i + win]])
        out[i] = v[(len(v) - 1) // 2] if len(v) else np.nan
    return out


def compute_f0_sing(sd, audio, noise=None, dither=None) -> np.ndarray:
    pitch = predict(sd, audio, 320, noise, dither)[2]
    return mean(np.repeat(pitch.numpy(), 2, -1), 5)


def compute_f0(sd, audio, noise=None, dither=None) -> np.ndarray:
    _, _, pitch, period = predict(sd, audio, 160, noise, dither)
    period, pitch = median(period.numpy(), 7), mean(pitch.numpy(), 5)
    pitch[period < 0.5] = 0
    return pitch.astype(np.float32)


def csv_text(pitch) -> str:
    """pitch/inference.py:102-110."""
    out = io.StringIO()
    for i in range(len(pitch)):
        t = i * 10
        minute = t // 60000
        print(f"{minute}m {(t - minute * 60000) // 1000}s {t % 1000:3d},{int(pitch[i])}", file=out)
    return out.getvalue()


# ------------------------------------------------------------------------------------------------ the reference
def import_reference():
    """The unmodified `crepe` package of the reference tree.  It imports librosa and resampy at module level: stubs
    stand in while it loads, and `librosa.sequence.viterbi` is the restatement above.  The stubs and the path entry
    leave `sys.modules` and `sys.path` again, so that nothing else in the process meets them."""
    if "crepe" not in sys.modules:
        if not reference_available():
            raise RuntimeError(f"reference tree not found at {ref_import.REF_ROOT}")
        added = [n for n in ("librosa", "librosa.sequence", "resampy") if n not in sys.modules]
        for name in added:
            ref_import._stub(name)
        sys.modules["librosa"].sequence = sys.modules["librosa.sequence"]
        sys.modules["librosa.sequence"].viterbi = viterbi
        sys.path.insert(0, ref_import.REF_ROOT)   # for this import only: the order of sys.path is other importers' business
        try:
            import crepe  # noqa
        finally:
            sys.path.remove(ref_import.REF_ROOT)
            for name in added:
                del sys.modules[name]
    return sys.modules["crepe"]


def reference_available() -> bool:
    return os.path.isfile(os.path.join(ref_import.REF_ROOT, "crepe", "model.py"))


def reference_predict(sd, capacity: str, audio, hop: int, noise, dither):
    """crepe.predict of the unmodified reference with `sd` loaded and the two draws replaced by the given ones ->
    (masked sigmoid outputs [F, 360], pitch [F], periodicity [F])."""
    import scipy.stats
    crepe = import_reference()
    model = crepe.Crepe(capacity)
    model.load_state_dict(sd)
    model.eval()
    crepe.core.infer.model, crepe.core.infer.capacity = model, capacity
    seen, pos = [], [0]
    o_rvs = scipy.stats.triang.rvs
    hook = model.register_forward_hook(lambda m, i, o: seen.append(o))

    def rvs(c, loc, scale, size):
        n = int(np.prod(tuple(size)))
        out = dither.numpy()[pos[0]:pos[0] + n].astype(np.float64).reshape(tuple(size))
        pos[0] += n
        return out

    scipy.stats.triang.rvs = rvs
    try:
        a = audio.float().reshape(1, -1) + noise.float().reshape(1, -1) * 0.001
        pitch, period = crepe.predict(a, 16000, hop, 50, 1000, capacity, batch_size=SEGMENT, device="cpu",
                                      return_periodicity=True)
    finally:
        scipy.stats.triang.rvs = o_rvs
        hook.remove()
    return torch.cat(seen), pitch[0], period[0]


# ------------------------------------------------------------------------------------------------ goldens
# the arrays of the reference's crepe/assets/tiny.pth (1.9 MB of fp32, which hardly compresses), by layer, so that each
# fixture file stays under 1 MB
TINY_FILES = {"crepe_tiny_conv123.npz": ("conv1", "conv2", "conv3"),
              "crepe_tiny_conv456_classifier.npz": ("conv4", "conv5", "conv6", "classifier")}


def tiny_weights():
    """The state dict of the reference's pretrained `tiny` model, from tests/golden/."""
    sd = {}
    for name in TINY_FILES:
        with np.load(os.path.join(GOLDEN, name)) as z:
            sd.update({k: torch.from_numpy(z[k]) for k in z.files})
    return sd


def tones(seed: int = 7):
    """Synthetic harmonic tones at 16 kHz with a known F0 track: steady 110, 220, 440, 880 Hz, a glide, a vibrato, a
    silent gap and F0 outside 50-1000 Hz -> (audio, f0 per sample; 0 = silence)."""
    sr, seg = 16000, 8000
    t = np.arange(seg) / sr
    f0 = [np.full(seg, f) for f in (110.0, 220.0, 440.0, 880.0)]
    f0.append(np.linspace(150.0, 600.0, seg))
    f0.append(300.0 * 2 ** (0.5 / 12 * np.sin(2 * np.pi * 5.5 * t)))
    f0.append(np.zeros(seg // 2))
    f0 += [np.full(seg // 2, 30.0), np.full(seg // 2, 1500.0), np.full(seg, 330.0)]
    f0 = np.concatenate(f0)
    phase = 2 * np.pi * np.cumsum(f0) / sr
    audio = sum(np.sin(k * phase) / k for k in range(1, 6)) * (f0 > 0) * 0.2
    return torch.from_numpy(audio.astype(np.float32)), f0.astype(np.float32)


def write_goldens():
    import scipy.stats
    from whisper_vits_svc_b200 import synth
    tiny = torch.load(os.path.join(ref_import.REF_ROOT, "crepe", "assets", "tiny.pth"), map_location="cpu", weights_only=True)
    tiny = {k: v for k, v in tiny.items() if not k.endswith("num_batches_tracked")}
    for name, keep in TINY_FILES.items():
        np.savez_compressed(os.path.join(GOLDEN, name), **{k: v.numpy() for k, v in tiny.items() if k.startswith(keep)})

    audio, f0 = tones()
    g = torch.Generator().manual_seed(11)
    noise = torch.randn(audio.numel(), generator=g)
    d = {"audio": audio.numpy(), "f0": f0, "noise": noise.numpy()}
    for hop in (160, 320):
        n = 1 + audio.numel() // hop
        dither = torch.from_numpy(scipy.stats.triang.rvs(c=0.5, loc=-20, scale=40, size=n, random_state=hop).astype(np.float32))
        probs, pitch, period = reference_predict(tiny, "tiny", audio, hop, noise, dither)
        masked, bins, o_pitch, o_period = predict(tiny, audio, hop, noise, dither)
        probs = mask(probs)   # the reference's own rows: its 512-frame batches round the convolutions differently
        assert torch.allclose(probs[:, 39:299], masked[:, 39:299], atol=1e-6) and torch.equal(pitch, o_pitch)
        assert torch.equal(period, probs.gather(1, bins[:, None]).reshape(-1))
        d.update({f"dither{hop}": dither.numpy(), f"probs{hop}": probs.numpy(), f"bins{hop}": bins.numpy().astype(np.int32),
                  f"pitch{hop}": pitch.numpy(), f"periodicity{hop}": period.numpy()})
    d["csv"] = np.frombuffer(csv_text(compute_f0_sing(tiny, audio, noise, torch.from_numpy(d["dither320"]))).encode(), np.uint8)
    d["pit"] = compute_f0(tiny, audio, noise, torch.from_numpy(d["dither160"]))
    np.savez_compressed(os.path.join(GOLDEN, "crepe_tiny_tones.npz"), **d)

    seed = 4321
    sd = synth.crepe_checkpoint(seed, "full")
    a = audio[6000:6000 + 4 * 320]
    nz = noise[:a.numel()]
    fr = frames(a, 320, nz)
    crepe = import_reference()
    model = crepe.Crepe("full")
    model.load_state_dict(sd)
    model.eval()
    with torch.no_grad():
        ref = model(fr)
        emb = model.embed(fr)
    probs, outs = network(sd, fr, layers=True)
    assert torch.allclose(ref, probs, atol=1e-6) and torch.allclose(emb.squeeze(-1), outs[4], atol=1e-5)
    np.savez_compressed(os.path.join(GOLDEN, "crepe_full_synth.npz"), seed=seed, audio=a.numpy(), noise=nz.numpy(), hop=320,
                        frames=fr.numpy(), probs=probs.numpy(),
                        **{f"layer{i + 2}": outs[i + 1].numpy().astype(np.float16) for i in range(5)})


if __name__ == "__main__":
    write_goldens()
