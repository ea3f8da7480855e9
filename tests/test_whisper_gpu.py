"""GPU parity of the PPG extractor (truncated Whisper encoder) against the oracle.
The encoder computes GEMMs/attention with bf16 operands (fp32 accumulate); the reference itself
runs fp16 on GPU (whisper/inference.py:22-23), so the gate is relative: rel-L2 <= 2e-2 and
cosine >= 0.999 against the fp32 oracle (SURVEY.md §8c tolerance plan)."""
import ctypes

import numpy as np

import pytest
import torch
import torch.nn.functional as F

from oracle import whisper_oracle as W
from tests.util import max_abs, rel_l2
from whisper_vits_svc_b200 import synth

pytestmark = pytest.mark.gpu


def _s():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _from_image(img, M, N):
    """GEMM tile image [ceil(M/128)][N/64][8][128][8] -> row-major [M, N]"""
    mt = (M + 127) // 128
    t = img.view(mt, N // 64, 8, 128, 8).permute(0, 3, 1, 2, 4).reshape(mt * 128, N)
    return t[:M]


@pytest.mark.parametrize("M,N,K,epi", [(128, 256, 64, 0), (300, 256, 128, 0), (1000, 512, 1280, 1), (257, 1280, 320, 2),
                                       (3000, 3840, 1280, 0), (24000, 1280, 1280, 2)])
def test_gemm_bf16(M, N, K, epi):
    from whisper_vits_svc_b200 import _lib
    g = torch.Generator().manual_seed(M + N + K)
    A = (torch.randn(M, K, generator=g)).bfloat16()
    Wt = (torch.randn(N, K, generator=g) / K ** 0.5).bfloat16()
    bias = torch.randn(N, generator=g)
    res = torch.randn(M, N, generator=g)
    Ad, Wd, bd, rd = A.cuda(), Wt.cuda(), bias.cuda(), res.cuda()
    ref = Ad.float() @ Wd.float().t() + bd          # fp32 reference on the device (same bf16 inputs)
    if epi == 1:
        ref = F.gelu(ref)
    if epi == 2:
        ref = ref + rd
    Mp = (M + 127) // 128 * 128
    lib = _lib.load()
    scratch = torch.empty(int(lib.svcb_op_gemm_bf16_scratch_bytes(M, N, K)), dtype=torch.uint8, device="cuda")
    if epi == 2:
        out = torch.zeros(M, N, device="cuda", dtype=torch.float32)
    else:
        out = torch.zeros(Mp if epi == 1 else M, N, device="cuda", dtype=torch.bfloat16)
    st = lib.svcb_op_gemm_bf16(Ad.data_ptr(), Wd.data_ptr(), bd.data_ptr(), out.data_ptr(),
                               rd.data_ptr() if epi == 2 else None, M, N, K, epi, scratch.data_ptr(),
                               scratch.numel(), _s())
    _lib.check(st, "svcb_op_gemm_bf16")
    torch.cuda.synchronize()
    got = _from_image(out, M, N) if epi == 1 else out
    tol = 2e-4 * K ** 0.5 if epi == 2 else 3e-2   # bf16 output rounding dominates for epi 0/1
    assert max_abs(got.float(), ref) <= tol


@pytest.mark.parametrize("B,T,heads,v_layout", [(2, 100, 2, 0), (1, 64, 4, 0), (2, 1500, 2, 0), (1, 333, 20, 0), (3, 129, 4, 0),
                                                (2, 100, 2, 1)])
def test_attention_tc_bf16(B, T, heads, v_layout):
    """The encoder's attention kernel (wgmma: S and O in registers, P fed from registers, V read as an MN-major operand) on its
    own, fed through the same tile image the QKV GEMM writes.  v_layout 1 exchanges LBO / SBO of the V
    descriptor: it must NOT match (pins the descriptor semantics the kernel relies on)."""
    from whisper_vits_svc_b200 import _lib
    D = heads * 64
    g = torch.Generator().manual_seed(T + heads)
    qkv = torch.randn(B, T, 3 * D, generator=g).bfloat16()
    q, k, v = [t.float().view(B, T, heads, 64).permute(0, 2, 1, 3) for t in qkv.split(D, dim=-1)]
    ref = (F.softmax(q @ k.transpose(-1, -2) / 8.0, dim=-1) @ v).permute(0, 2, 1, 3).reshape(B, T, D)
    qd = qkv.cuda()
    out = torch.zeros(B, T, D, device="cuda", dtype=torch.bfloat16)
    lib = _lib.load()
    scratch = torch.empty(int(lib.svcb_op_attention_tc_bf16_scratch_bytes(B, T, D)), dtype=torch.uint8, device="cuda")
    st = lib.svcb_op_attention_tc_bf16(qd.data_ptr(), out.data_ptr(), B, T, D, heads, v_layout, scratch.data_ptr(),
                                       scratch.numel(), _s())
    _lib.check(st, "svcb_op_attention_tc_bf16")
    torch.cuda.synchronize()
    err = max_abs(out.float(), ref)
    print(f"attention_tc B={B} T={T} heads={heads} v_layout={v_layout}: max-abs {err:.3e}")
    if v_layout == 0:
        assert err <= 2e-2
    else:
        assert err > 2e-2


@pytest.mark.parametrize("state,heads,layers,B,n", [(256, 4, 4, 2, 200), (512, 8, 4, 1, 301), (1280, 20, 4, 1, 400)])
def test_encoder_vs_oracle(state, heads, layers, B, n):
    from whisper_vits_svc_b200 import whisper_infer
    dims = dict(synth.WHISPER_LARGE_V2_DIMS, n_audio_state=state, n_audio_head=heads, n_audio_layer=layers)
    ck = synth.whisper_checkpoint(dims, seed=state)
    g = torch.Generator().manual_seed(n)
    mel = torch.randn(B, 80, n, generator=g).clamp(-1, 1.5)
    ref = W.audio_encoder(ck, mel)
    enc = whisper_infer.WhisperB200(ck, "cuda").encoder
    got = enc(mel).cpu()
    assert got.shape == ref.shape
    r = rel_l2(got, ref)
    cos = float(F.cosine_similarity(got.flatten(), ref.flatten(), dim=0))
    print(f"whisper D={state} layers={W.kept_layers(dims)}: rel-l2 {r:.3e}, cosine {cos:.6f}, max-abs {max_abs(got, ref):.3e}")
    assert r <= 2e-2 and cos >= 0.999


@pytest.mark.parametrize("name", ["whisper_d256_l8_b2_n200", "whisper_d512_l4_b1_n301"])
def test_encoder_vs_reference_golden(name):
    """tests/golden/whisper_*.npz = `Whisper.encoder(mel)` of the UNMODIFIED reference after the loader
    surgery (oracle/make_golden.py:whisper_case, fp32 CPU).  The device encoder (bf16 operands, fp32
    accumulate) against it, same relative gate as against the oracle."""
    import os
    from oracle import make_golden as mg
    from tests.util import GOLDEN
    from whisper_vits_svc_b200 import whisper_infer
    over, ck_seed, B, n, in_seed = mg.WHISPER_CASES[name]
    ck = synth.whisper_checkpoint(mg.whisper_dims(over), seed=ck_seed)
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    got = whisper_infer.WhisperB200(ck, "cuda").encoder(torch.from_numpy(g["mel"])).cpu()
    ref = torch.from_numpy(g["ppg"])
    assert got.shape == ref.shape
    r = rel_l2(got, ref)
    cos = float(F.cosine_similarity(got.flatten(), ref.flatten(), dim=0))
    print(f"{name}: rel-l2 {r:.3e}, cosine {cos:.6f}, max-abs {max_abs(got, ref):.3e}")
    assert r <= 2e-2 and cos >= 0.999


def test_encoder_full_size_vs_oracle():
    """BASELINE config #3 geometry: large-v2 dims (D=1280, 20 heads, 32 layers -> 24 kept), 30 s items
    (n=3000 frames -> all 1500 positions), B=2 so the M dimension spans many 128-row tiles and an item
    boundary.  bf16 rounding accumulates through 24 residual blocks; the gate stays rel-L2 <= 2e-2 and
    cosine >= 0.999 against the fp32 oracle (the reference itself runs fp16 on GPU)."""
    from whisper_vits_svc_b200 import whisper_infer
    ck = synth.whisper_checkpoint(seed=77)
    assert W.kept_layers(ck["dims"]) == 24
    mel = torch.randn(2, 80, 3000, generator=torch.Generator().manual_seed(9)).clamp(-1, 1.5)
    enc = whisper_infer.WhisperB200(ck, "cuda").encoder
    got = enc(mel).cpu()
    del enc
    torch.cuda.empty_cache()
    ref = W.audio_encoder(ck, mel[:1])        # one item on the host: ~1.7 TFLOP of fp32
    assert got.shape == (2, 1500, 1280)
    r = rel_l2(got[:1], ref)
    cos = float(F.cosine_similarity(got[:1].flatten(), ref.flatten(), dim=0))
    print(f"whisper large-v2 geometry, 24 layers, 30 s: rel-l2 {r:.3e}, cosine {cos:.6f}, max-abs {max_abs(got[:1], ref):.3e}")
    assert torch.isfinite(got).all()
    assert r <= 2e-2 and cos >= 0.999
    # item independence at full size: the second item alone == in the batch
    one = whisper_infer.WhisperB200(ck, "cuda").encoder(mel[1:2]).cpu()
    assert max_abs(one, got[1:2]) <= 1e-5


def _small_encoder():
    from whisper_vits_svc_b200 import whisper_infer
    dims = dict(synth.WHISPER_LARGE_V2_DIMS, n_audio_state=256, n_audio_head=4, n_audio_layer=4)
    ck = synth.whisper_checkpoint(dims, seed=11)
    return ck, whisper_infer.WhisperB200(ck, "cuda")


@pytest.mark.parametrize("B,N", [(1, 16000 * 3), (3, 16000 * 15), (2, 16000 * 2 + 37), (1, 201), (2, 480000)])
def test_log_mel_device_vs_oracle(B, N):
    """svcb_whisper_log_mel vs the torch restatement of whisper/audio.py:68-100 (itself pinned on the
    transformers implementation in the CPU suite).  White noise, a tone over a noise floor, silence."""
    _, wm = _small_encoder()
    rs = np.random.RandomState(N % 9973)
    t = np.arange(N) / 16000.0
    items = []
    for b in range(B):
        if b % 3 == 0:
            items.append(rs.randn(N).astype(np.float32) * 0.1)
        elif b % 3 == 1:
            items.append((0.3 * np.sin(2 * np.pi * (220.0 * (b + 1)) * t) + 0.01 * rs.randn(N)).astype(np.float32))
        else:
            items.append(np.zeros(N, np.float32))
    audio = torch.from_numpy(np.stack(items))
    ref = torch.stack([W.log_mel_spectrogram(a) for a in audio])
    got = wm.encoder.log_mel(audio).cpu()
    assert got.shape == ref.shape == (B, 80, N // 160)
    d = (got - ref).abs()
    print(f"log-mel B={B} N={N}: max-abs {float(d.max()):.3e}, mean-abs {float(d.mean()):.3e}")
    # direct fp32 DFT vs torch's FFT: bins near the max-8 floor of a tonal frame differ most
    assert float(d.max()) <= 5e-3 and float(d.mean()) <= 1e-4
    # the extractor's noise term is fused into the same pass (whisper/inference.py:46,58)
    nz = torch.randn(B, 80, N // 160, generator=torch.Generator().manual_seed(5))
    got_n = wm.encoder.log_mel(audio, nz, 0.1).cpu()
    assert max_abs(got_n, got + 0.1 * nz) <= 1e-6


def test_pred_ppg_end_to_end_vs_oracle(tmp_path):
    """pred_ppg (whisper/inference.py:32-62): wav file -> 15 s chunks + remainder -> device log-mel
    (+ the given noise) -> encoder -> row trim -> .npy, against the oracle on the same noise."""
    from scipy.io import wavfile
    from whisper_vits_svc_b200 import whisper_infer
    ck, wm = _small_encoder()
    rs = np.random.RandomState(2)
    n = 16000 * 33 + 1234                       # two full chunks + a remainder
    wav = (rs.randn(n) * 0.05).astype(np.float32)
    path = str(tmp_path / "a.wav")
    wavfile.write(path, 16000, (wav * 32767).astype(np.int16))
    audio = whisper_infer.load_audio(path)
    plan = whisper_infer.chunk_plan(audio.shape[0])
    assert [e - s for s, e, _ in plan] == [240000, 240000, n - 480000]
    g = torch.Generator().manual_seed(8)
    noise = [torch.randn(80, (e - s) // 160, generator=g) for s, e, _ in plan]
    out = str(tmp_path / "a.ppg.npy")
    whisper_infer.pred_ppg(wm, path, out, "cuda", mel_noise=noise)
    got = np.load(out)
    rows = []
    for (s, e, n_rows), nz in zip(plan, noise):
        mel = W.log_mel_spectrogram(torch.from_numpy(audio[s:e])) + nz * 0.1
        rows.append(W.audio_encoder(ck, mel.unsqueeze(0))[0][:n_rows])
    ref = torch.cat(rows).numpy()
    assert got.shape == ref.shape and got.shape[0] == 750 + 750 + (audio.shape[0] - 480000) // 320
    r = float(np.linalg.norm(got - ref) / np.linalg.norm(ref))
    print(f"pred_ppg: rows {got.shape[0]}, rel-l2 {r:.3e}")
    assert r <= 2e-2
