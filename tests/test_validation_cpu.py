"""The validation score and the export, on the CPU: the oracle's filterbank and mel against transformers and the live
reference, the oracle's validation loop against the reference's own validate(), and svc_export.py against the
reference's.  Tests that use the reference skip where it is absent."""
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from oracle import ref_import
from oracle import validation_oracle as V
from tests.util import ROOT
from whisper_vits_svc_b200 import whisper_infer

needs_ref = pytest.mark.skipif(not ref_import.available(), reason="reference tree not present")


def test_filterbank_against_transformers():
    audio_utils = pytest.importorskip("transformers.audio_utils")
    ours = V.mel_filter_bank(32000, 1024, 100, 50, 16000)
    theirs = audio_utils.mel_filter_bank(513, 100, 50, 16000, 32000, norm="slaney", mel_scale="slaney").T
    assert ours.shape == theirs.shape == (100, 513)
    assert np.abs(ours - theirs).max() <= 1e-9


def test_mel_filters_fmin_fmax():
    got = whisper_infer.mel_filters(100, 32000, 1024, fmin=50.0, fmax=16000.0).numpy()
    want = V.mel_filter_bank(32000, 1024, 100, 50.0, 16000.0).astype(np.float32)
    assert np.abs(got - want).max() <= 1e-6 * np.abs(want).max()


def _whisper_matrix_before(n_mels, sr, n_fft):
    """whisper_infer.mel_filters as it was before fmin / fmax were added."""
    fftfreqs = np.linspace(0, sr / 2, n_fft // 2 + 1)
    mel_pts = whisper_infer._mel_to_hz_slaney(np.linspace(whisper_infer._hz_to_mel_slaney(0.0),
                                                          whisper_infer._hz_to_mel_slaney(sr / 2), n_mels + 2))
    fdiff = np.diff(mel_pts)
    ramps = mel_pts[:, None] - fftfreqs[None, :]
    w = np.zeros((n_mels, n_fft // 2 + 1))
    for i in range(n_mels):
        w[i] = np.maximum(0, np.minimum(-ramps[i] / fdiff[i], ramps[i + 2] / fdiff[i + 1]))
    return (w * (2.0 / (mel_pts[2:n_mels + 2] - mel_pts[:n_mels]))[:, None]).astype(np.float32)


@pytest.mark.parametrize("n_mels", [80, 128])
def test_mel_filters_whisper_defaults_unchanged(n_mels):
    got = whisper_infer.mel_filters(n_mels).numpy()
    assert np.array_equal(got, _whisper_matrix_before(n_mels, 16000, 400))


def test_mel_silence_is_the_clip():
    hp = V.load_hp()
    mel = V.mel_spectrogram(torch.zeros(2, 4000), V.basis32(hp))
    assert mel.shape == (2, 100, 12)
    assert torch.all(mel == torch.tensor(V.LOG_CLIP, dtype=torch.float32))


def _ref_stft(monkeypatch, hp):
    """vits_extend/stft.py with librosa.util and librosa.filters stubbed, the filterbank the oracle's."""
    ref_import._ensure_path()
    for name in ("librosa", "librosa.util", "librosa.filters"):
        ref_import._stub(name)
    lib = sys.modules["librosa"]
    monkeypatch.setattr(lib, "util", sys.modules["librosa.util"], raising=False)
    monkeypatch.setattr(lib, "filters", sys.modules["librosa.filters"], raising=False)
    monkeypatch.setattr(sys.modules["librosa.util"], "normalize", lambda x, *a, **k: x, raising=False)
    mel_fn = lambda sr, n_fft, n_mels, fmin, fmax: V.mel_filter_bank(sr, n_fft, n_mels, fmin, fmax)
    monkeypatch.setattr(sys.modules["librosa.filters"], "mel", mel_fn, raising=False)
    import vits_extend.stft as stft
    monkeypatch.setattr(stft, "librosa_mel_fn", mel_fn)
    d = hp.data
    return stft.TacotronSTFT(d.filter_length, d.hop_length, d.win_length, d.mel_channels, d.sampling_rate, d.mel_fmin,
                             d.mel_fmax, center=False)


@needs_ref
def test_mel_against_reference(monkeypatch):
    hp = ref_import.load_hp()
    ref = _ref_stft(monkeypatch, hp)
    g = torch.Generator().manual_seed(5)
    y = (torch.rand(3, 32000 + 171, generator=g) * 2 - 1) * torch.linspace(0, 1, 32171)
    y[1, 5000:9000] = 0.0
    with torch.no_grad():
        want = ref.mel_spectrogram(y)
    got = V.mel_spectrogram(y, V.basis32(hp))
    assert got.shape == want.shape == (3, 100, 32171 // 320)
    assert float((got - want).abs().max()) <= 1e-6


class _Writer:
    def __init__(self):
        self.audio, self.loss = [], None

    def log_fig_audio(self, real, fake, spec_fake, spec_real, idx, step):
        self.audio.append((idx, np.array(real), np.array(fake)))

    def log_validation(self, loss, generator, discriminator, step):
        self.loss = loss


def _ref_trn(hp, sd_g, seed=3):
    ref_import._ensure_path()
    from vits.models import SynthesizerTrn
    torch.manual_seed(seed)
    m = SynthesizerTrn(hp.data.filter_length // 2 + 1, hp.data.segment_size // hp.data.hop_length, hp)
    missing = set(sd_g) - set(m.state_dict())
    assert not missing, sorted(missing)[:5]
    m.load_state_dict(sd_g, strict=False)
    return m


@needs_ref
def test_validate_against_reference(monkeypatch, tmp_path):
    import random
    from whisper_vits_svc_b200 import synth
    hp = ref_import.load_hp()
    stft = _ref_stft(monkeypatch, hp)
    files = V.write_dataset(str(tmp_path), hp)
    sd = synth.svc_state_dict(hp, V.WEIGHT_SEED)
    trn = _ref_trn(hp, sd)
    from vits.data_utils import TextAudioSpeakerCollate, TextAudioSpeakerSet
    import vits_extend.validation as rv
    random.seed(V.CROP_SEED)
    ds = TextAudioSpeakerSet(files, hp.data)
    loader = torch.utils.data.DataLoader(ds, num_workers=0, shuffle=False, batch_size=V.BATCH, drop_last=False,
                                         collate_fn=TextAudioSpeakerCollate())
    writer, log = _Writer(), []
    disc = types.SimpleNamespace(eval=lambda: None)
    torch.manual_seed(99)
    with torch.no_grad(), ref_import.record_rng(log):
        rv.validate(hp, None, trn, disc, loader, stft, writer, 0, "cpu")
    assert [k for k, _ in log] == ["randn_like", "randn_like", "randn_like", "rand", "randn_like"] * len(loader)
    draws = [t for _, t in log]

    def replay(bi, shapes):
        return dict(zip(shapes, draws[5 * bi:5 * bi + 5]))

    batches, n = V.read_batches(files, hp, V.CROP_SEED, V.BATCH)
    loss, _, logged = V.validate(sd, hp, batches, n, replay, V.basis32(hp))
    assert abs(loss - writer.loss) <= 1e-5 * abs(writer.loss), (loss, writer.loss)
    assert [idx for idx, _, _ in writer.audio] == sorted(logged)
    for idx, real, fake in writer.audio:
        assert np.array_equal(real, logged[idx][0])
        assert np.abs(fake - logged[idx][1]).max() <= 1e-4


def _trainer_checkpoint(path, hp, seed=5):
    """A trainer-format checkpoint: model_g of a reference-shaped SynthesizerTrn (synthetic SynthesizerInfer weights plus
    seeded enc_q / emb_g / speaker_classifier entries), small model_d / optimizer stand-ins."""
    from whisper_vits_svc_b200 import synth
    sd = synth.svc_state_dict(hp, seed)
    g = torch.Generator().manual_seed(seed)
    sd["enc_q.pre.weight"] = torch.randn(192, 513, 1, generator=g)
    sd["emb_g.weight"] = torch.randn(256, 256, generator=g)
    sd["speaker_classifier.classifier.1.weight"] = torch.randn(256, 192, 1, generator=g)
    torch.save({"model_g": sd, "model_d": {"w": torch.randn(4, generator=g)}, "optim_g": {}, "optim_d": {}, "step": 7,
                "epoch": 1, "hp_str": "x"}, path)
    return sd


def test_export_cli(tmp_path):
    hp = V.load_hp()
    ck = tmp_path / "ck.pt"
    sd = _trainer_checkpoint(ck, hp)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "svc_export.py"), "-c", os.path.join(ROOT, "configs", "base.yaml"),
                        "-p", str(ck)], cwd=tmp_path, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert "is not in the checkpoint" not in r.stdout
    out = torch.load(tmp_path / "sovits5.0.pth", map_location="cpu")
    assert list(out) == ["model_g"] and len(out["model_g"]) == 903
    for k, v in out["model_g"].items():
        assert torch.equal(v, sd[k]), k
    from whisper_vits_svc_b200 import hostio, models
    m = models.SynthesizerInfer(513, 25, hp)
    import contextlib
    import io
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        hostio.load_svc_model(str(tmp_path / "sovits5.0.pth"), m)
    assert "is not in the checkpoint" not in buf.getvalue()


@needs_ref
def test_export_against_reference(monkeypatch, tmp_path):
    hp = ref_import.load_hp()
    ref_import._ensure_path()
    om = types.ModuleType("omegaconf")
    om.OmegaConf = types.SimpleNamespace(load=ref_import.load_hp)
    monkeypatch.setitem(sys.modules, "omegaconf", om)
    from whisper_vits_svc_b200 import synth
    ref_trn = _ref_trn(hp, synth.svc_state_dict(hp, 5))
    ck = tmp_path / "ck.pt"
    torch.save({"model_g": ref_trn.state_dict(), "model_d": {}, "optim_g": {}, "optim_d": {}, "step": 1, "epoch": 1,
                "hp_str": ""}, ck)
    (tmp_path / "ref").mkdir()
    (tmp_path / "ours").mkdir()
    monkeypatch.chdir(tmp_path / "ref")
    import importlib.util
    spec = importlib.util.spec_from_file_location("ref_svc_export", os.path.join(ref_import.REF_ROOT, "svc_export.py"))
    ref_export = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref_export)
    ref_export.main(types.SimpleNamespace(config=os.path.join(ROOT, "configs", "base.yaml"), checkpoint_path=str(ck)))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "svc_export.py"), "-c", os.path.join(ROOT, "configs", "base.yaml"),
                        "-p", str(ck)], cwd=tmp_path / "ours", capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    want = torch.load(tmp_path / "ref" / "sovits5.0.pth", map_location="cpu")["model_g"]
    got = torch.load(tmp_path / "ours" / "sovits5.0.pth", map_location="cpu")["model_g"]
    assert set(got) == set(want)
    held = torch.load(ck, map_location="cpu")["model_g"]
    for k in got:
        assert k in held
        assert torch.equal(got[k], held[k]) and torch.equal(want[k], held[k]), k
