"""Ragged device batches for dataset feature preparation (preprocess_ppg.py, preprocess_hubert.py).

Every item of a ragged batch must be bitwise equal to a lone run of it through the existing entry points, and within
the encoders' relative gate (rel-L2 <= 2e-2, cosine >= 0.999) of the fp32 oracles.  The CLIs then run end to end on a
small dataset and their features build both retrieval indexes."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import hubert_oracle as HO, preprocess_oracle as PO, whisper_oracle as WO
from tests.util import GOLDEN, ROOT, rel_l2
from whisper_vits_svc_b200 import _lib, synth

pytestmark = pytest.mark.gpu


def _cos(a, b):
    a, b = torch.as_tensor(a).double().flatten(), torch.as_tensor(b).double().flatten()
    return float((a @ b) / (a.norm() * b.norm()))


def _audio(seed, n, sr=16000):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / sr
    x = 0.3 * np.sin(2 * np.pi * (150.0 + 40 * (seed % 7)) * t) * (1.0 + 0.5 * np.sin(2 * np.pi * 2.5 * t))
    return (x + 0.05 * rng.standard_normal(n)).astype(np.float32)


def _ragged(items):
    lens = [a.shape[0] for a in items]
    wav = np.zeros((len(items), max(lens)), np.float32)
    for b, a in enumerate(items):
        wav[b, :lens[b]] = a
    return torch.from_numpy(wav), lens


def _same(tag, got, want):
    d = float((got - want).abs().max()) if got.shape == want.shape else float("nan")
    print(f"{tag}: ragged vs lone max-abs {d:.3e}")
    assert got.shape == want.shape and torch.equal(got, want), tag


# ------------------------------------------------------------------------------------------------ HuBERT
@pytest.fixture(scope="module")
def hubert():
    from whisper_vits_svc_b200 import hubert_infer
    cache = {}

    def get(seed):
        if seed not in cache:
            sd = synth.hubert_checkpoint(seed)
            cache[seed] = (sd, hubert_infer.HubertSoftB200(sd, "cuda"))
        return cache[seed]
    return get


def test_hubert_ragged_equals_lone_and_oracle(hubert):
    """Frame counts straddling the 64- and 128-row tiles of attention and the GEMMs, one frame, and 20 s+ (frames(320 T)
    = T; +157 samples gives an item whose length is not a whole frame)."""
    sd, model = hubert(31)
    frames = [1, 63, 64, 65, 127, 128, 129, 100, 1001]
    lens = [320 * t for t in frames]
    lens[7] += 157
    items = [_audio(i, n) for i, n in enumerate(lens)]
    wav, lens = _ragged(items)
    out = model.units_ragged(wav, lens).cpu()
    T = model.frames(wav.shape[1])
    assert out.shape == (len(items), T, 256)
    for b, a in enumerate(items):
        t = model.frames(lens[b])
        assert t == frames[b]
        lone = model.units(torch.from_numpy(a)[None]).cpu()[0]
        _same(f"hubert item {b} ({t} frames)", out[b, :t], lone)
        assert not out[b, t:].any()
        ref = HO.units(sd, torch.from_numpy(a)[None, None])[0]
        r, c = rel_l2(out[b, :t], ref), _cos(out[b, :t], ref)
        print(f"hubert item {b}: vs oracle rel-l2 {r:.3e}, cosine {c:.6f}")
        assert r <= 2e-2 and c >= 0.999


@pytest.mark.parametrize("name", ["hubert_soft_b2_n8000", "hubert_soft_b1_n16123"])
def test_hubert_ragged_goldens(hubert, name):
    """The three items of the two HuBERT goldens in one ragged batch.  The goldens come from two checkpoints, so the
    batch runs once per checkpoint and the items of that checkpoint's golden are held to its gate."""
    from oracle import make_golden as mg
    gs = {n: np.load(f"{GOLDEN}/{n}.npz") for n in ("hubert_soft_b2_n8000", "hubert_soft_b1_n16123")}
    items = [(n, i, gs[n]["wav"][i, 0]) for n in gs for i in range(gs[n]["wav"].shape[0])]
    _, model = hubert(mg.HUBERT_CASES[name][0])
    wav, lens = _ragged([a for _, _, a in items])
    out = model.units_ragged(wav, lens).cpu()
    for b, (n, i, a) in enumerate(items):
        if n != name:
            continue
        ref = torch.from_numpy(gs[n]["units"][i])
        got = out[b, :ref.shape[0]]
        r, c = rel_l2(got, ref), _cos(got, ref)
        print(f"{name}[{i}] in a ragged batch of {len(items)}: rel-l2 {r:.3e}, cosine {c:.6f}")
        assert model.frames(lens[b]) == ref.shape[0]
        assert r <= 2e-2 and c >= 0.999


def test_ragged_lengths_are_validated(hubert):
    from whisper_vits_svc_b200 import whisper_infer
    _, model = hubert(31)
    wav = torch.zeros(2, 16000)
    for bad in ([16000, 0], [16000, 16001], [16000, 100]):          # empty, too long, no frame
        with pytest.raises(_lib.SvcbError):
            model.units_ragged(wav, bad)
    dims = dict(synth.WHISPER_LARGE_V2_DIMS, n_audio_state=256, n_audio_head=4, n_audio_layer=4)
    enc = whisper_infer.WhisperB200(synth.whisper_checkpoint(dims, seed=11), "cuda").encoder
    for bad in ([16000, 200], [16000, 16001]):
        with pytest.raises(_lib.SvcbError):
            enc.log_mel_ragged(wav, bad)
    for bad in ([100, 0], [100, 101]):
        with pytest.raises(_lib.SvcbError):
            enc.encode_ragged(torch.zeros(2, 80, 100), bad)


# ------------------------------------------------------------------------------------------------ Whisper
def _whisper(state=256, heads=4, layers=4, seed=11):
    from whisper_vits_svc_b200 import whisper_infer
    dims = dict(synth.WHISPER_LARGE_V2_DIMS, n_audio_state=state, n_audio_head=heads, n_audio_layer=layers)
    ck = synth.whisper_checkpoint(dims, seed=seed) if state != 1280 else synth.whisper_checkpoint(seed=seed)
    return ck, whisper_infer.WhisperB200(ck, "cuda")


# device lengths: the 15 s floor, odd and even frame counts between 15 and 30 s (one not a whole hop), 30 s
W_LENS = [240000, 160 * 1999 + 50, 160 * 2400, 160 * 2001, 480000]


def test_whisper_ragged_log_mel_and_encoder_equal_lone():
    _, wm = _whisper()
    enc = wm.encoder
    items = [_audio(10 + i, n) for i, n in enumerate(W_LENS)]
    wav, lens = _ragged(items)
    mel = enc.log_mel_ragged(wav, lens)
    frames = [n // 160 for n in lens]
    out = enc.encode_ragged(mel, frames).cpu()
    mel = mel.cpu()
    for b, a in enumerate(items):
        F, T = frames[b], (frames[b] - 1) // 2 + 1
        lone_mel = enc.log_mel(torch.from_numpy(a)[None])
        _same(f"log-mel item {b} ({F} frames)", mel[b, :, :F], lone_mel.cpu()[0])
        assert not mel[b, :, F:].any()
        _same(f"encoder item {b} ({F} frames, {T} positions)", out[b, :T], enc(lone_mel).cpu()[0])
        assert not out[b, T:].any()


def test_ppg_batch_vs_oracle_and_lone():
    """whisper_infer.ppg_batch = prepare/preprocess_ppg.py:pred_ppg per file: against
    audio_encoder(log_mel_spectrogram(pad_or_trim(x)))[:len // 320] and against a lone run."""
    from whisper_vits_svc_b200 import whisper_infer
    ck, wm = _whisper()
    lens = [16000 * 3 + 11, 240000, 160 * 2001 + 7, 16000 * 25, 480000, 16000 * 33]
    items = [_audio(20 + i, n) for i, n in enumerate(lens)]
    got = whisper_infer.ppg_batch(wm, items)
    for b, a in enumerate(items):
        rows = whisper_infer.ppg_rows(a.shape[0])
        assert got[b].shape == (rows, 256) and got[b].dtype == np.float32
        p = torch.from_numpy(PO.pad_or_trim(a))
        ref = WO.audio_encoder(ck, WO.log_mel_spectrogram(p)[None])[0][:rows]
        r, c = rel_l2(torch.from_numpy(got[b]), ref), _cos(got[b], ref)
        print(f"ppg item {b} ({a.shape[0]} samples, {rows} rows): vs oracle rel-l2 {r:.3e}, cosine {c:.6f}")
        assert r <= 2e-2 and c >= 0.999
        lone = wm.encoder(wm.encoder.log_mel(p[None])).cpu()[0][:rows].numpy()
        assert np.array_equal(got[b], lone)


def test_whisper_ragged_full_size_equals_lone():
    """large-v2 geometry (D 1280, 20 heads, 24 kept layers): one ragged batch against lone runs."""
    ck, wm = _whisper(1280, 20, 32, seed=77)
    enc = wm.encoder
    items = [_audio(40 + i, n) for i, n in enumerate([240000, 160 * 2333 + 99, 480000])]
    wav, lens = _ragged(items)
    frames = [n // 160 for n in lens]
    out = enc.encode_ragged(enc.log_mel_ragged(wav, lens), frames).cpu()
    assert torch.isfinite(out).all()
    for b, a in enumerate(items):
        T = (frames[b] - 1) // 2 + 1
        _same(f"large-v2 item {b} ({frames[b]} frames)", out[b, :T], enc(enc.log_mel(torch.from_numpy(a)[None])).cpu()[0])


# ------------------------------------------------------------------------------------------------ CLIs
def test_cli_wavs_to_indexes(tmp_path, hubert):
    from scipy.io import wavfile
    from whisper_vits_svc_b200 import hubert_infer, retrieval_train, whisper_infer
    ck, wm = _whisper()
    sd, model = hubert(31)
    (tmp_path / "whisper_pretrain").mkdir()
    (tmp_path / "hubert_pretrain").mkdir()
    torch.save(ck, tmp_path / "whisper_pretrain" / "large-v2.pt")
    torch.save(sd, tmp_path / "hubert_pretrain" / "hubert-soft-0d54a1f4.pt")
    wav = tmp_path / "wav"
    for s in ("spk_a", "spk_b"):
        (wav / s).mkdir(parents=True)

    def pcm(x):
        return (np.clip(x, -1, 1) * 32767).astype(np.int16)

    wavfile.write(wav / "spk_a" / "a3.wav", 16000, pcm(_audio(1, 16000 * 3)))
    wavfile.write(wav / "spk_a" / "a17.wav", 16000, pcm(_audio(2, 16000 * 17 + 333)))
    wavfile.write(wav / "spk_a" / "hi48k.wav", 48000, pcm(_audio(3, 48000 * 2, 48000)))
    wavfile.write(wav / "spk_b" / "stereo.wav", 16000, pcm(np.stack([_audio(4, 16000 * 4), _audio(5, 16000 * 4)], 1)))
    wavfile.write(wav / "spk_b" / "b21.wav", 16000, pcm(_audio(6, 16000 * 21 + 5)))
    wavfile.write(wav / "spk_b" / "short.wav", 16000, pcm(_audio(7, 100)))
    (wav / "spk_b" / "broken.wav").write_bytes(b"not a wav file")
    good = ["spk_a/a3", "spk_a/a17", "spk_a/hi48k", "spk_b/stereo", "spk_b/b21"]

    def cli(*args):
        r = subprocess.run([sys.executable, os.path.join(ROOT, args[0]), *args[1:], "-t", "2", "--batch", "3"],
                           cwd=tmp_path, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
        assert "short.wav" in r.stderr and "broken.wav" in r.stderr and "padding overhead" in r.stdout
        return r

    cli("preprocess_ppg.py", "-w", "wav", "-p", "data_svc/whisper")
    cli("preprocess_hubert.py", "-w", "wav", "-v", "data_svc/hubert")
    for g in good:
        audio = whisper_infer.load_audio(str(wav / f"{g}.wav"))
        ppg = np.load(tmp_path / "data_svc" / "whisper" / f"{g}.ppg.npy")
        assert ppg.dtype == np.float32 and ppg.shape == (whisper_infer.ppg_rows(audio.shape[0]), 256)
        assert np.array_equal(ppg, whisper_infer.ppg_batch(wm, [audio])[0]), g
        vec = np.load(tmp_path / "data_svc" / "hubert" / f"{g}.vec.npy")
        assert vec.dtype == np.float32 and vec.shape == (model.frames(audio.shape[0]), 256)
        assert np.array_equal(vec, hubert_infer.units_batch(model, [audio])[0]), g
    for d in ("whisper", "hubert"):
        assert sorted(os.listdir(tmp_path / "data_svc" / d / "spk_b")) == sorted(
            f"{n}.{'ppg' if d == 'whisper' else 'vec'}.npy" for n in ("stereo", "b21"))
    stamp = {p: p.stat().st_mtime_ns for p in (tmp_path / "data_svc" / "whisper").rglob("*.npy")}
    r = cli("preprocess_ppg.py", "-w", "wav", "-p", "data_svc/whisper")         # existing outputs are skipped
    assert "2/2" in r.stdout
    assert {p: p.stat().st_mtime_ns for p in (tmp_path / "data_svc" / "whisper").rglob("*.npy")} == stamp
    for s in ("spk_a", "spk_b"):
        for d, width in (("hubert", 256), ("whisper", 256)):
            out = tmp_path / "idx" / s / f"{d}.index"
            out.parent.mkdir(parents=True, exist_ok=True)
            ix = retrieval_train.train_index(tmp_path / "data_svc" / d / s, out)
            rows = sum(np.load(p).shape[0] for p in (tmp_path / "data_svc" / d / s).glob("*.npy"))
            assert out.is_file() and ix.ntotal == rows and ix.vectors.shape[1] == width
