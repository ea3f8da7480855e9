"""Host-side mirror of whisper/inference.py (`load_model`, `pred_ppg`) over the H100 encoder.

`load_model(path, device)` reads the reference checkpoint format {"dims", "model_state_dict"}
(whisper/inference.py:12-20), applies the loader's surgery (decoder dropped, last quarter of the
encoder blocks dropped, ln_post kept), packs the weights once (linear weights -> bf16, q/k/v
concatenated) and returns an object whose `.encoder(mel)` runs libsvc_b200.so.  The reference runs
fp16 on GPU / fp32 on CPU (whisper/inference.py:22-23); here GEMMs and attention take bf16
operands with fp32 accumulation and an fp32 residual stream.

`pred_ppg(whisper, wavPath, ppgPath, device)` keeps the reference's framing (15 s chunks + remainder,
0.1*randn mel noise, row trim to samples//320, np.save; whisper/inference.py:32-62) but runs all
chunks of a file as ONE batch.  The log-mel front-end (whisper/audio.py:54-100) runs on the device
too (`svcb_whisper_log_mel`, SURVEY.md §8f-1): the audio is uploaded once, STFT / mel / log / noise
happen in three launches and the mel tensor never visits the host.  The Slaney mel filterbank is
restated here (host, once) because librosa is not a dependency; the torch restatement of the whole
front end lives in oracle/whisper_oracle.py and is what the GPU test compares against.
"""
from __future__ import annotations

import ctypes
import math
from typing import Dict, List, Optional

import numpy as np
import torch

from . import _lib, pack

SAMPLE_RATE = 16000
N_FFT = 400
N_MELS = 80
HOP_LENGTH = 160
N_SAMPLES = 30 * SAMPLE_RATE  # whisper/audio.py:19


# ------------------------------------------------------------------------------ packing
def _bf16_as_f32(w: torch.Tensor) -> torch.Tensor:
    """nn.Linear weight [N, K] -> bf16 GEMM tile image [N/256][K/64][8][256][8] (csrc/whisper_gemm.cu:
    one (n-tile, k-tile) block = one contiguous bulk copy in the K-major panel order), returned as a
    float32 view of the bytes."""
    w = w.detach().float().contiguous().bfloat16()
    n, k = w.shape
    assert n % 256 == 0 and k % 64 == 0, (n, k)
    img = w.view(n // 256, 256, k // 64, 8, 8).permute(0, 2, 3, 1, 4).contiguous()  # nt, kt, kc, row, e
    return img.view(torch.float32).reshape(-1)


def sinusoids(length: int, channels: int, max_timescale: float = 10000.0) -> torch.Tensor:
    """whisper/model.py:48-54"""
    inc = np.log(max_timescale) / (channels // 2 - 1)
    inv = torch.exp(-inc * torch.arange(channels // 2))
    t = torch.arange(length)[:, None] * inv[None, :]
    return torch.cat([torch.sin(t), torch.cos(t)], dim=1)


def kept_layers(dims: dict) -> int:
    n = int(dims["n_audio_layer"])
    return n - n // 4  # whisper/inference.py:17-19


def pack_whisper(ckpt: dict):
    """-> ([(name, fp32-typed tensor)], cfg dict).  Names consumed by csrc/whisper_api.cu."""
    dims, sd = ckpt["dims"], ckpt["model_state_dict"]
    D = int(dims["n_audio_state"])
    n_layer = kept_layers(dims)
    items = []

    def put(n, t):
        items.append((n, t.detach().float().contiguous()))

    # conv1 (k=3, stride 1) as a GEMM over an im2col image of the log-mel: W1[co][j*n_mels + ci] = w[co][ci][j],
    # K padded from 3 * n_mels to a multiple of 64
    w1 = sd["encoder.conv1.weight"].float()
    k1 = 3 * w1.shape[1]
    w1p = torch.zeros(D, (k1 + 63) // 64 * 64)
    w1p[:, :k1] = w1.permute(0, 2, 1).reshape(D, k1)
    items.append(("conv1.wimg", _bf16_as_f32(w1p)))
    put("conv1.b", sd["encoder.conv1.bias"])
    # conv2 (k=3, stride 2) runs as a GEMM over an im2col image: W2[co][j*D + ci] = w[co][ci][j]
    items.append(("conv2.wimg", _bf16_as_f32(sd["encoder.conv2.weight"].float().permute(0, 2, 1).reshape(D, 3 * D))))
    put("conv2.b", sd["encoder.conv2.bias"])
    pos = sd.get("encoder.positional_embedding")
    if pos is None:  # a buffer; absent from synthetic checkpoints, recomputed like the constructor does
        pos = sinusoids(int(dims["n_audio_ctx"]), D)
    put("pos", pos)
    for i in range(n_layer):
        b = f"encoder.blocks.{i}"
        p = f"blk.{i}"
        put(p + ".ln1.g", sd[b + ".attn_ln.weight"]); put(p + ".ln1.b", sd[b + ".attn_ln.bias"])
        wqkv = torch.cat([sd[b + ".attn.query.weight"], sd[b + ".attn.key.weight"], sd[b + ".attn.value.weight"]], 0)
        bqkv = torch.cat([sd[b + ".attn.query.bias"].float(), torch.zeros(D), sd[b + ".attn.value.bias"].float()], 0)
        items.append((p + ".wqkv", _bf16_as_f32(wqkv)))
        put(p + ".bqkv", bqkv)
        items.append((p + ".wo", _bf16_as_f32(sd[b + ".attn.out.weight"])))
        put(p + ".bo", sd[b + ".attn.out.bias"])
        put(p + ".ln2.g", sd[b + ".mlp_ln.weight"]); put(p + ".ln2.b", sd[b + ".mlp_ln.bias"])
        items.append((p + ".w1", _bf16_as_f32(sd[b + ".mlp.0.weight"])))
        put(p + ".b1", sd[b + ".mlp.0.bias"])
        items.append((p + ".w2", _bf16_as_f32(sd[b + ".mlp.2.weight"])))
        put(p + ".b2", sd[b + ".mlp.2.bias"])
    put("ln_post.g", sd["encoder.ln_post.weight"]); put("ln_post.b", sd["encoder.ln_post.bias"])
    cfg = dict(n_mels=int(dims["n_mels"]), n_ctx=int(dims["n_audio_ctx"]), n_state=D,
               n_head=int(dims["n_audio_head"]), n_layer=n_layer)
    return items, cfg


class WhisperEncoderB200:
    """`whisper.encoder(mel)` of the reference: mel [B, n_mels, n] -> [B, (n-1)//2+1, n_state] fp32."""

    def __init__(self, ckpt: dict, device):
        self.device = _lib.cuda_device(device)
        self.dims = dict(ckpt["dims"])
        items, self.cfg = pack_whisper(ckpt)
        blob_cpu, table = pack.build_blob(items)
        self._handle = _lib.Handle("whisper", table, blob_cpu.to(self.device), _lib.WhisperConfig(**self.cfg))
        self._filters = mel_filters(self.cfg["n_mels"]).to(self.device).contiguous()
        self._lm_scratch = None

    def _workspace(self, B: int, n: int) -> torch.Tensor:
        return self._handle.workspace(_lib.load().svcb_whisper_workspace_bytes(self._handle, B, n))

    @torch.no_grad()
    def __call__(self, mel: torch.Tensor) -> torch.Tensor:
        mel = mel.to(self.device, torch.float32).contiguous()
        B, nm, n = mel.shape
        assert nm == self.cfg["n_mels"]
        n2 = (n - 1) // 2 + 1
        assert n2 <= self.cfg["n_ctx"], "incorrect audio shape"  # whisper/model.py:155
        ws = self._workspace(B, n)
        out = torch.empty(B, n2, self.cfg["n_state"], device=self.device, dtype=torch.float32)
        self._handle.call("whisper_encode", mel.data_ptr(), out.data_ptr(), B, n, ws.data_ptr(), ws.numel())
        return out

    @torch.no_grad()
    def log_mel(self, audio: torch.Tensor, noise: Optional[torch.Tensor] = None, noise_gain: float = 0.1) -> torch.Tensor:
        """whisper/audio.py:68-100 (+ the extractor's `mel + randn_like(mel) * 0.1`, whisper/inference.py:46,58)
        on the device: audio [B, n_samples] (16 kHz) -> mel [B, n_mels, n_samples // 160] fp32."""
        audio = audio.to(self.device, torch.float32).contiguous()
        if audio.dim() == 1:
            audio = audio.unsqueeze(0)
        B, N = audio.shape
        nm = self.cfg["n_mels"]
        F = N // HOP_LENGTH
        mel = torch.empty(B, nm, F, device=self.device, dtype=torch.float32)
        if noise is not None:
            noise = noise.to(self.device, torch.float32).contiguous()
            assert tuple(noise.shape) == (B, nm, F)
        if self._lm_scratch is None or self._lm_scratch.numel() < B:
            self._lm_scratch = torch.empty(max(B, 64), dtype=torch.int32, device=self.device)
        _lib.call("whisper_log_mel", audio.data_ptr(), self._filters.data_ptr(), noise.data_ptr() if noise is not None else None,
                  float(noise_gain), mel.data_ptr(), self._lm_scratch.data_ptr(), B, N, nm, device=self.device)
        return mel

    @torch.no_grad()
    def log_mel_ragged(self, audio: torch.Tensor, n_samples: List[int]) -> torch.Tensor:
        """`log_mel` without noise for a ragged batch: item b is audio[b, :n_samples[b]] (more than 200 samples).
        -> mel [B, n_mels, N // 160]; item b's first n_samples[b] // 160 frames equal a lone `log_mel` of it bit for
        bit, its later frames are zero (the padding the encoder's first convolution expects)."""
        audio = audio.to(self.device, torch.float32).contiguous()
        B, N = audio.shape
        assert len(n_samples) == B
        nm = self.cfg["n_mels"]
        mel = torch.empty(B, nm, N // HOP_LENGTH, device=self.device, dtype=torch.float32)
        if self._lm_scratch is None or self._lm_scratch.numel() < 2 * B:
            self._lm_scratch = torch.empty(max(2 * B, 64), dtype=torch.int32, device=self.device)
        lens = (ctypes.c_int32 * B)(*n_samples)
        _lib.call("whisper_log_mel_ragged", audio.data_ptr(), lens, self._filters.data_ptr(), mel.data_ptr(),
                  self._lm_scratch.data_ptr(), B, N, nm, device=self.device)
        return mel

    @torch.no_grad()
    def encode_ragged(self, mel: torch.Tensor, n_frames: List[int]) -> torch.Tensor:
        """The encoder for a ragged batch: item b is mel[b, :, :n_frames[b]], whose later columns must be zero (as
        `log_mel_ragged` leaves them).  -> [B, (n-1)//2+1, n_state]; item b's first (n_frames[b]-1)//2+1 rows equal a
        lone run of it bit for bit, its later rows are zero."""
        mel = mel.to(self.device, torch.float32).contiguous()
        B, nm, n = mel.shape
        assert nm == self.cfg["n_mels"] and len(n_frames) == B
        n2 = (n - 1) // 2 + 1
        assert n2 <= self.cfg["n_ctx"], "incorrect audio shape"
        ws = self._workspace(B, n)
        out = torch.empty(B, n2, self.cfg["n_state"], device=self.device, dtype=torch.float32)
        lens = (ctypes.c_int32 * B)(*n_frames)
        self._handle.call("whisper_encode_ragged", mel.data_ptr(), lens, out.data_ptr(), B, n, ws.data_ptr(), ws.numel())
        return out


class WhisperB200:
    """What `load_model` returns: exposes `.encoder` and `.dims` like the reference's Whisper module."""

    def __init__(self, ckpt: dict, device):
        self.dims = dict(ckpt["dims"])
        self.encoder = WhisperEncoderB200(ckpt, device)


def load_model(path, device) -> WhisperB200:
    """whisper/inference.py:11-29"""
    ckpt = torch.load(path, map_location="cpu", weights_only=False)
    return WhisperB200(ckpt, device)


# ------------------------------------------------------------------------------ audio front-end (host)
def _hz_to_mel_slaney(f):
    f = np.asarray(f, dtype=np.float64)
    f_sp = 200.0 / 3
    mels = f / f_sp
    min_log_hz, min_log_mel, logstep = 1000.0, 1000.0 / f_sp, np.log(6.4) / 27.0
    return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-10) / min_log_hz) / logstep, mels)


def _mel_to_hz_slaney(m):
    m = np.asarray(m, dtype=np.float64)
    f_sp = 200.0 / 3
    min_log_hz, min_log_mel, logstep = 1000.0, 1000.0 / f_sp, np.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)


def mel_filters(n_mels: int = N_MELS, sr: int = SAMPLE_RATE, n_fft: int = N_FFT, fmin: float = 0.0,
                fmax: float | None = None) -> torch.Tensor:
    """librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax) (Slaney scale, slaney area norm; fmax None is sr / 2).  The
    defaults are what whisper/audio.py:54-65 asks librosa for; vits_extend/stft.py:46-47 asks for fmin 50, fmax 16000."""
    if fmax is None:
        fmax = sr / 2
    fftfreqs = np.linspace(0, sr / 2, n_fft // 2 + 1)
    mel_pts = _mel_to_hz_slaney(np.linspace(_hz_to_mel_slaney(fmin), _hz_to_mel_slaney(fmax), n_mels + 2))
    fdiff = np.diff(mel_pts)
    ramps = mel_pts[:, None] - fftfreqs[None, :]
    w = np.zeros((n_mels, n_fft // 2 + 1))
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        w[i] = np.maximum(0, np.minimum(lower, upper))
    enorm = 2.0 / (mel_pts[2:n_mels + 2] - mel_pts[:n_mels])
    return torch.from_numpy((w * enorm[:, None]).astype(np.float32))


def load_audio(path: str, sr: int = SAMPLE_RATE) -> np.ndarray:
    """whisper/audio.py:24-26 uses librosa.load(sr=16000) (mono float32, resampled); restated with
    scipy: int PCM -> [-1,1), channel mean, polyphase resampling.  Differences from the reference
    extractor: .wav only (librosa/audioread decode more containers), and `resample_poly` instead of
    librosa's soxr/kaiser resampler, so PPGs of non-16 kHz files differ slightly from the reference's."""
    from scipy.signal import resample_poly
    from .resample import decode_wav
    rate, x = decode_wav(path)
    if rate != sr:
        g = math.gcd(int(rate), sr)
        x = resample_poly(x, sr // g, int(rate) // g).astype(np.float32)
    return x


def chunk_plan(audln: int, chunk: int = 15 * SAMPLE_RATE):
    """whisper/inference.py:37-61 as data: [(start, end, ppg_rows)]."""
    out, idx = [], 0
    while idx + chunk < audln:
        out.append((idx, idx + chunk, chunk // 320))
        idx += chunk
    if idx < audln:
        out.append((idx, audln, (audln - idx) // 320))
    return out


@torch.no_grad()
def pred_ppg(whisper: WhisperB200, wavPath: str, ppgPath: str, device, mel_noise: Optional[List[torch.Tensor]] = None):
    audio = load_audio(wavPath)
    plan = chunk_plan(audio.shape[0])
    enc = whisper.encoder
    nm = enc.cfg["n_mels"]
    # chunks of equal length (all the full 15 s ones) form one batch; the remainder runs alone
    groups: Dict[int, List[int]] = {}
    for i, (s, e, _) in enumerate(plan):
        groups.setdefault(e - s, []).append(i)
    outs: Dict[int, np.ndarray] = {}
    for n, idx in groups.items():
        wav = torch.from_numpy(np.stack([audio[plan[i][0]:plan[i][1]] for i in idx]))
        F = n // HOP_LENGTH
        if mel_noise is not None:
            nz = torch.stack([mel_noise[i] for i in idx])
        else:  # host RNG like the reference's randn_like on the CPU mel (whisper/inference.py:46,58)
            nz = torch.randn(len(idx), nm, F)
        o = enc(enc.log_mel(wav, nz, 0.1))
        for j, i in enumerate(idx):
            outs[i] = o[j].cpu().float().numpy()
    rows: List[np.ndarray] = []
    for i, (_, _, n_rows) in enumerate(plan):
        rows.extend(outs[i][:n_rows])
    np.save(ppgPath, np.asarray(rows), allow_pickle=False)


# ------------------------------------------------------------------------------ dataset PPGs (prepare/preprocess_ppg.py)
def pad_or_trim(audio: np.ndarray, length_max: int = N_SAMPLES, length_min: int = N_SAMPLES // 2) -> np.ndarray:
    """whisper/audio.py:29-50 on a 1-D array: trimmed to at most 30 s, zero-padded to at least 15 s.  Clips of 15 s or
    less all become 15 s; clips between 15 and 30 s keep their length."""
    if audio.shape[-1] > length_max:
        audio = audio[..., :length_max]
    if audio.shape[-1] < length_min:
        audio = np.pad(audio, [(0, 0)] * (audio.ndim - 1) + [(0, length_min - audio.shape[-1])])
    return audio


def ppg_rows(audln: int) -> int:
    """Rows prepare/preprocess_ppg.py:29-39 keeps of a file of audln samples: ppg[:audln // 320] of the encoder's
    (F - 1) // 2 + 1 positions for the F = len(pad_or_trim(audio)) // 160 mel frames."""
    n = min(max(audln, N_SAMPLES // 2), N_SAMPLES)
    return min(audln // 320, (n // HOP_LENGTH - 1) // 2 + 1)


@torch.no_grad()
def ppg_batch(whisper: WhisperB200, audios: List[np.ndarray]) -> List[np.ndarray]:
    """prepare/preprocess_ppg.py:pred_ppg for several files in one ragged device batch: each 16 kHz array is
    pad_or_trim-ed, turned into its log-mel with no noise and encoded; item b -> float32 [ppg_rows(len), n_state].
    Each item's rows are those of a lone run of it."""
    enc = whisper.encoder
    padded = [pad_or_trim(np.asarray(a, dtype=np.float32)) for a in audios]
    lens = [p.shape[0] for p in padded]
    wav = np.zeros((len(padded), max(lens)), np.float32)
    for b, p in enumerate(padded):
        wav[b, :lens[b]] = p
    ppg = enc.encode_ragged(enc.log_mel_ragged(torch.from_numpy(wav), lens), [n // HOP_LENGTH for n in lens]).cpu()
    return [ppg[b, :ppg_rows(a.shape[0])].numpy() for b, a in enumerate(audios)]
