"""Speaker encoder host side: the oracle (oracle/speaker_oracle.py) against the goldens and the live reference, the pins
of its librosa restatements, window offsets, config reading and rejection, the dataset path rules and the packer."""
import importlib.util
import json
import os

import numpy as np
import pytest
import torch

from oracle import ref_import
from oracle import speaker_oracle as SO
from tests.util import ROOT
from whisper_vits_svc_b200 import synth
from whisper_vits_svc_b200 import speaker_infer as S

CONFIG = os.path.join(ref_import.REF_ROOT, "speaker_pretrain", "config.json")


# ------------------------------------------------------------------------------------------------ oracle
@pytest.mark.parametrize("name", tuple(SO.SPEAKER_CASES))
def test_oracle_against_goldens(name):
    g = SO.load_golden(name)
    x = g["wav"].astype(np.float32) / np.float32(32768)
    wav = SO.prepare(x)
    assert np.array_equal(wav, S.prepare_wav(x))
    mel = SO.melspectrogram(wav).T
    assert mel.shape == g["mel"].shape and np.abs(mel - g["mel"]).max() <= 1e-5
    emb, win = SO.compute_embedding(synth.speaker_checkpoint(int(g["seed"]))["model"], g["mel"])
    assert np.abs(emb - g["embedding"]).max() <= 1e-6 and np.abs(win - g["windows"]).max() <= 1e-6
    assert np.allclose(np.linalg.norm(win, axis=1), 1.0, atol=1e-6)


def test_golden_shapes():
    short, long_ = SO.load_golden("speaker_short_trim"), SO.load_golden("speaker_10s")
    assert short["mel"].shape[0] < 250 and long_["mel"].shape[0] == 626
    # trim acts on the short clip: fewer frames than its length after the margins alone would give
    assert short["mel"].shape[0] < 1 + (short["wav"].shape[0] - 320) // 256
    assert sum(os.path.getsize(os.path.join(SO.GOLDEN, n + ".npz")) for n in SO.SPEAKER_CASES) < 1_100_000


@pytest.mark.skipif(not ref_import.available(), reason="reference tree absent")
def test_oracle_against_live_reference(monkeypatch, tmp_path):
    from scipy.io import wavfile
    lstm, audio = SO.import_reference(monkeypatch)
    sd = synth.speaker_checkpoint(5)["model"]
    wav = SO.synth_voice(5, 3.0, 0.3)
    wavfile.write(tmp_path / "x.wav", 16000, wav)
    mel, emb, win = SO.reference_embedding(lstm, audio, sd, str(tmp_path / "x.wav"))
    ours = SO.melspectrogram(SO.prepare(wav.astype(np.float32) / np.float32(32768))).T
    assert np.abs(ours - mel).max() <= 1e-6
    e, w = SO.compute_embedding(sd, mel)
    assert np.abs(e - emb).max() <= 2e-6 and np.abs(w - win).max() <= 2e-6


# ------------------------------------------------------------------------------------------------ pins
def test_stft_pinned_on_torch():
    rng = np.random.default_rng(1)
    for n in (513, 1024, 5000, 16001):
        y = rng.standard_normal(n)
        ref = torch.stft(torch.from_numpy(y), 1024, 256, window=torch.hann_window(1024, dtype=torch.float64), center=True,
                         pad_mode="reflect", return_complex=True).abs().numpy()
        ours = SO.stft_magnitude(y)
        assert ours.shape == ref.shape == (513, 1 + n // 256)
        assert np.abs(ours - ref).max() <= 1e-9 * max(1.0, np.abs(ref).max())


def test_mel_basis_pinned_on_transformers():
    au = pytest.importorskip("transformers.audio_utils")
    fb = au.mel_filter_bank(num_frequency_bins=513, num_mel_filters=80, min_frequency=0.0, max_frequency=8000.0,
                            sampling_rate=16000, norm="slaney", mel_scale="slaney")
    assert np.abs(SO.mel_basis() - fb.T).max() < 1e-8
    assert np.abs(S.mel_filters(80, 16000, 1024).numpy() - fb.T).max() < 1e-6   # the blob's fp32 copy


def _tone(n, amp, rng):
    return (amp * np.sin(np.arange(n) * 0.05) + 0.01 * amp * rng.standard_normal(n)).astype(np.float32)


@pytest.mark.parametrize("trim_fn", [lambda y: SO.trim(y)[0], S.trim], ids=["oracle", "product"])
def test_trim_on_known_boundaries(trim_fn):
    rng = np.random.default_rng(2)
    sil = lambda n: np.zeros(n, np.float32)   # noqa: E731
    y = np.concatenate([sil(8192), _tone(16384, 0.5, rng), sil(8192)])
    out = trim_fn(y)
    # the cut falls on frame boundaries (hop 256) within one frame (1024 samples, centred) of the tone's ends
    start = int(np.flatnonzero(np.all(np.lib.stride_tricks.sliding_window_view(y, out.shape[0]) == out, axis=1))[0])
    end = start + out.shape[0]
    assert start % 256 == 0 and 8192 - 1024 < start <= 8192 and 8192 + 16384 <= end < 8192 + 16384 + 1024
    # nothing to trim: loud throughout
    z = _tone(20000, 0.3, rng)
    assert np.array_equal(trim_fn(z), z)
    # a -70 dB tail is below top_db = 60 and goes; a -50 dB tail stays
    for db, kept in ((-70, False), (-50, True)):
        w = np.concatenate([_tone(16000, 1.0, rng), _tone(16000, 10 ** (db / 20), rng)])
        assert (trim_fn(w).shape[0] > 24000) == kept


def test_product_and_oracle_trim_agree():
    rng = np.random.default_rng(4)
    for _ in range(5):
        n = int(rng.integers(2000, 40000))
        y = (rng.standard_normal(n) * np.exp(-((np.arange(n) - n / 2) / (n / 6)) ** 2)).astype(np.float32)
        assert np.array_equal(S.trim(y), SO.trim(y)[0])


# ------------------------------------------------------------------------------------------------ windows
@pytest.mark.parametrize("T", [1, 249, 250, 251, 626, 1000, 5000])
def test_window_offsets_match_linspace(T):
    L = min(250, T)
    ref = [int(o) for o in np.linspace(0, T - L, num=10)]
    assert S.window_offsets(T) == ref == SO.window_offsets(T)[0]
    # the device formula (csrc/speaker_api.cu spk_win_offset): w * (S / 9) in float64, the last point S
    S_ = T - L
    dev = [S_ if w == 9 else int(float(w) * (float(S_) / 9.0)) for w in range(10)]
    assert dev == ref


# ------------------------------------------------------------------------------------------------ config
def test_read_json_with_comments(tmp_path):
    p = tmp_path / "c.json"
    p.write_text('{\n "a": 1, // one\n "b": "x\\\ny", // the continuation joins the string\n "c": [1, 2] // list\n}\n')
    assert S.read_json(str(p)) == {"a": 1, "b": "xy", "c": [1, 2]}
    p.write_text(json.dumps({"a": 2}))
    assert S.read_json(str(p)) == {"a": 2}


@pytest.mark.skipif(not ref_import.available(), reason="reference tree absent")
def test_reference_config_accepted():
    assert S.audio_params(S.read_json(CONFIG)) == dict(preemphasis=0.98, ref_level_db=20.0, min_level_db=-100.0, max_norm=4.0,
                                                       trim_db=60.0)


BASE = {"model_name": "lstm",
        "audio": {"num_mels": 80, "fft_size": 1024, "sample_rate": 16000, "win_length": 1024, "hop_length": 256,
                  "preemphasis": 0.98, "min_level_db": -100, "ref_level_db": 20, "signal_norm": True, "symmetric_norm": True,
                  "max_norm": 4.0, "clip_norm": True, "mel_fmin": 0.0, "mel_fmax": 8000.0, "trim_db": 60},
        "model": {"input_dim": 80, "proj_dim": 256, "lstm_dim": 768, "num_lstm_layers": 3, "use_lstm_with_projection": True}}


@pytest.mark.parametrize("edit", [
    ("model_name", "resnet"), ("model.use_lstm_with_projection", False), ("model.lstm_dim", 512), ("model.num_lstm_layers", 2),
    ("audio.num_mels", 64), ("audio.sample_rate", 22050), ("audio.fft_size", 2048), ("audio.win_length", 800),
    ("audio.hop_length", 160), ("audio.log_func", "np.log"), ("audio.symmetric_norm", False), ("audio.signal_norm", False),
    ("audio.clip_norm", False), ("audio.mel_fmax", 7600.0), ("audio.mel_fmin", 50.0), ("audio.stats_path", "s.npy"),
    ("audio.min_level_db", 0), ("audio", None),
])
def test_config_rejection(edit):
    import copy
    cfg = copy.deepcopy(BASE)
    S.audio_params(cfg)
    key, val = edit
    d = cfg
    *path, last = key.split(".")
    for k in path:
        d = d[k]
    d[last] = val
    with pytest.raises(ValueError):
        S.audio_params(cfg)


# ------------------------------------------------------------------------------------------------ dataset paths
def _preprocess_module():
    spec = importlib.util.spec_from_file_location("preprocess_speaker_cli", os.path.join(ROOT, "preprocess_speaker.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_preprocess_speaker_path_mapping(tmp_path, monkeypatch):
    m = _preprocess_module()
    monkeypatch.chdir(tmp_path)
    for s in ("alice", "bob"):
        (tmp_path / "data" / s).mkdir(parents=True)
        for f in ("a.wav", "b.wav", "c.txt"):
            (tmp_path / "data" / s / f).write_bytes(b"")
    (tmp_path / "data" / "top.wav").write_bytes(b"")
    (tmp_path / "data" / "readme.md").write_bytes(b"")
    files = sorted(m.get_spk_wavs("data", "out"))
    assert files == sorted(["./data/alice/a.wav", "./data/alice/b.wav", "./data/bob/a.wav", "./data/bob/b.wav", "./data/top.wav"])
    assert (tmp_path / "out" / "alice").is_dir() and (tmp_path / "out" / "bob").is_dir()
    assert m.embed_path("./data/alice/a.wav", "data", "out") == "./out/alice/a.spk"
    assert m.embed_path("./data/top.wav", "data", "out") == "./out/top.spk"


# ------------------------------------------------------------------------------------------------ packer
def test_packer_names_and_shapes():
    sd = synth.speaker_checkpoint(3)["model"]
    assert sorted(sd) == sorted(f"layers.{l}.{n}" for l in range(3) for n in
                                ("lstm.weight_ih_l0", "lstm.weight_hh_l0", "lstm.bias_ih_l0", "lstm.bias_hh_l0", "linear.weight"))
    assert all(sd[f"layers.{l}.lstm.bias_ih_l0"].abs().sum() > 0 for l in range(3))
    items = dict(S.pack_speaker(sd, dict(preemphasis=0.98, ref_level_db=20.0, min_level_db=-100.0, max_norm=4.0, trim_db=60.0)))
    want = {"spk.mel_fb": 80 * 513, "spk.audio": 4}
    for l in range(3):
        kin = 128 if l == 0 else 256
        want.update({f"spk.l{l}.wih": 3072 * 3 * kin // 2, f"spk.l{l}.b": 3072, f"spk.l{l}.whh": 128 * 2 * 768 * 24 // 2,
                     f"spk.l{l}.wproj": 256 * 3 * 768 // 2})
    assert {k: v.numel() for k, v in items.items()} == want
    assert all(v.dtype == torch.float32 for v in items.values())
    assert items["spk.audio"].tolist() == pytest.approx([0.98, 20.0, -100.0, 4.0])


def test_packed_recurrent_weights_decode():
    """W_hh slices: CTA c, [hi, lo][k / 8][24][8] bf16; gate column 4 u + g is nn.LSTM row g * 768 + 6 c + u; hi + lo
    recovers the fp32 weight to bf16x2 precision."""
    sd = synth.speaker_checkpoint(4)["model"]
    items = dict(S.pack_speaker(sd, dict(preemphasis=0.98, ref_level_db=20.0, min_level_db=-100.0, max_norm=4.0, trim_db=60.0)))
    whh = sd["layers.1.lstm.weight_hh_l0"]
    img = items["spk.l1.whh"].view(torch.bfloat16).float().view(128, 2, 96, 24, 8).permute(0, 1, 3, 2, 4).reshape(128, 2, 24, 768)
    order = S.gate_order()
    for c in (0, 57, 127):
        for n in (0, 5, 23):
            ref = whh[order[24 * c + n]]
            assert torch.equal(img[c, 0, n], ref.bfloat16().float())
            assert (img[c, 0, n] + img[c, 1, n] - ref).abs().max() <= 2e-5 * ref.abs().max()
    b = items["spk.l1.b"]
    bias = sd["layers.1.lstm.bias_ih_l0"] + sd["layers.1.lstm.bias_hh_l0"]
    assert torch.equal(b, bias[torch.from_numpy(order)])


def test_prepare_wav_rejects_unframeable_audio():
    from whisper_vits_svc_b200 import _lib
    tone = (0.5 * np.sin(np.arange(1200) * 0.05)).astype(np.float32)
    assert S.prepare_wav(tone[:320 + 513]).shape == (513,)
    with pytest.raises(_lib.SvcbError):
        S.prepare_wav(tone[:320 + 512])   # 512 samples left: the reflect padding of one frame needs more
    with pytest.raises(_lib.SvcbError):
        S.prepare_wav(np.zeros(32000, np.float32))


def test_preprocess_speaker_skips_only_the_failing_file(tmp_path, monkeypatch):
    """A batch that fails on the device is retried file by file: only the culprit is lost, and it is named."""
    m = _preprocess_module()
    monkeypatch.chdir(tmp_path)
    (tmp_path / "data").mkdir()
    names = [f"f{i}.wav" for i in range(7)]
    for n in names:
        (tmp_path / "data" / n).write_bytes(b"")

    class Fake:
        def load_wav(self, f):
            if f.endswith("f1.wav"):
                raise ValueError("unreadable")
            return np.full(4, float(f[-5]), np.float32)

        def embed(self, wavs):
            if any(w[0] == 4 for w in wavs):
                raise RuntimeError("device rejected f4")
            return torch.stack([torch.full((256,), float(w[0])) for w in wavs])

    files = m.get_spk_wavs("data", "out")
    import io
    import contextlib
    err = io.StringIO()
    with contextlib.redirect_stderr(err):
        failed = m.extract_speaker_embeddings(files, "data", "out", Fake(), 3, batch=3)
    assert failed == 2 and "f1.wav" in err.getvalue() and "f4.wav: device rejected" in err.getvalue()
    written = sorted(os.listdir(tmp_path / "out"))
    assert written == sorted(f"f{i}.spk.npy" for i in (0, 2, 3, 5, 6))
    assert np.load(tmp_path / "out" / "f5.spk.npy")[0] == 5.0
