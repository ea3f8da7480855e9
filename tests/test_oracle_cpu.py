"""CPU tests: the oracle against the committed golden fixtures, generated from the unmodified
reference by oracle/make_golden.py (tests/golden/reference_pins.npz holds the reference outputs the
pins below compare with)."""
import os

import numpy as np
import pytest
import torch

from oracle import svc_oracle as O
from tests.util import GOLDEN, make_inputs, max_abs
from whisper_vits_svc_b200 import hparams, synth

FULL = ["infer_b2_t48", "infer_b3_t70_ragged"]


def _load(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"))


def max_abs64(a, b):
    return float(np.abs(np.asarray(a, dtype=np.float64) - np.asarray(b, dtype=np.float64)).max())


@pytest.fixture(scope="module")
def pins():
    return _load("reference_pins")


@pytest.mark.parametrize("name", FULL)
def test_oracle_matches_golden_full(name, hp, sd):
    g = _load(name)
    d = make_inputs(int(g["seed"]), int(g["B"]), int(g["T"]), hp, ragged=bool(g["ragged"]))
    src = O.pitch2source(sd, hp, d["pit"], d["rand_ini"], d["noise"])
    assert max_abs(src, g["source"]) <= 1e-6
    st = {}
    wave = O.synthesizer_infer(sd, hp, d["ppg"], d["vec"], d["pit"], d["spk"], d["ppg_l"], src, d["eps"], stages=st)
    assert max_abs(st["z_p"], g["z_p"]) <= 1e-5
    assert max_abs(st["z"], g["z"]) <= 1e-5
    assert max_abs(wave, g["wave"]) <= 1e-5
    assert np.array_equal(O.source2wav(src[:1]), g["pcm"])


@pytest.mark.parametrize("name,over", [("gen80_b2_t36", dict(gen__upsample_input=80, data__sampling_rate=24000)),
                                       ("gen192_b1_t64", {})])
def test_oracle_matches_golden_generator(name, over, hp):
    g = _load(name)
    hpx = hparams.override(hp, **over)
    sdx = synth.svc_state_dict(hpx, 1234)
    d = make_inputs(int(g["seed"]), int(g["B"]), int(g["T"]), hpx, gen_only=True)
    src = O.pitch2source(sdx, hpx, d["pit"], d["rand_ini"], d["noise"])
    assert max_abs(src, g["source"]) <= 1e-6
    wave = O.generator(sdx, hpx, d["spk"], d["z"], src)
    assert max_abs(wave, g["wave"]) <= 1e-5


def test_oracle_matches_reference_live(hp, sd, pins):
    """Float64 on both sides (oracle/make_golden.py:reference_pins): host-independent to ~1e-15."""
    from oracle.make_golden import to_float64
    d = to_float64(make_inputs(77, 2, 33, hp, ragged=True))
    sd = to_float64(sd)
    src, wave = pins["svc_source"], pins["svc_wave"]
    src_o = O.pitch2source(sd, hp, d["pit"], d["rand_ini"], d["noise"])
    wave_o = O.synthesizer_infer(sd, hp, d["ppg"], d["vec"], d["pit"], d["spk"], d["ppg_l"], src_o, d["eps"])
    assert max_abs64(src, src_o) <= 1e-6
    assert max_abs64(wave, wave_o) <= 1e-6


def test_synthetic_checkpoint_has_reference_keys(sd, pins):
    keys = [str(k) for k in pins["sd_keys"]]
    assert set(keys) == set(sd)
    for k, shp in zip(keys, pins["sd_shapes"]):
        assert ",".join(map(str, sd[k].shape)) == str(shp), k
    # the alias-filter buffers are the reference's own Kaiser-sinc taps
    assert np.array_equal(pins["up_filter"], sd["dec.activation_post.upsample.filter"].numpy())


def test_f0_to_coarse_integer_hz_is_rounding_safe():
    """The CUDA path evaluates the mel mapping in fp32 with a correctly rounded log; for every
    integer-Hz pitch (the reference's CSV format) that equals torch's fp32 result."""
    f = torch.arange(0, 1101, dtype=torch.float32)
    ref = O.f0_to_coarse(f)
    mel = 1127 * torch.log((1 + f / 700).double()).float()
    mel = torch.where(mel > 0, (mel - np.float32(77.75496616579426)) * 254 / np.float32(986.6532670978451) + 1, mel)
    mel = mel.clamp(min=1.0, max=255.0)
    assert torch.equal((mel + 0.5).long(), ref)
    assert ref.min() >= 1 and ref.max() <= 255


# ------------------------------------------------------------------ log-mel front end (whisper/audio.py:54-100)
def test_mel_filterbank_pinned_by_third_party():
    """librosa (the reference's source of the matrix, whisper/audio.py:54-65) is absent: pin the
    restated Slaney filterbank on transformers' independent implementation of the same definition."""
    au = pytest.importorskip("transformers.audio_utils")
    from oracle import whisper_oracle as wo
    fb = au.mel_filter_bank(num_frequency_bins=201, num_mel_filters=80, min_frequency=0.0, max_frequency=8000.0,
                            sampling_rate=16000, norm="slaney", mel_scale="slaney")
    ours = wo.slaney_mel_filterbank()
    assert ours.shape == (80, 201)
    assert np.abs(ours - fb.T).max() < 1e-8
    # structure: non-negative triangles, one peak each, area ~ 1 under the Slaney normalisation
    assert (ours >= 0).all()
    assert np.all(np.diff(ours.argmax(axis=1)) >= 0)
    assert np.allclose(ours.sum(axis=1) * (16000 / 400), 1.0, atol=0.1)   # 40 Hz bins sample narrow triangles coarsely


def test_log_mel_oracle_pinned_by_third_party():
    tr = pytest.importorskip("transformers")
    from oracle import whisper_oracle as wo
    fe = tr.WhisperFeatureExtractor(feature_size=80)
    rs = np.random.RandomState(3)
    t = np.arange(16000 * 4) / 16000.0
    for x in (rs.randn(16000 * 4).astype(np.float32) * 0.1,
              (0.3 * np.sin(2 * np.pi * 440.0 * t) + 0.01 * rs.randn(t.size)).astype(np.float32),
              np.zeros(16000 * 2 + 37, np.float32)):
        ref = fe._np_extract_fbank_features(x[None, :], "cpu")[0]
        got = wo.log_mel_spectrogram(torch.from_numpy(x)).numpy()
        assert got.shape == ref.shape == (80, x.size // 160)
        assert np.abs(got - ref).max() < 2e-4   # near-floor bins of the tone: fp32 FFT vs numpy float64


def test_product_mel_filters_match_oracle():
    from oracle import whisper_oracle as wo
    from whisper_vits_svc_b200 import whisper_infer
    assert np.array_equal(whisper_infer.mel_filters().numpy(), wo.slaney_mel_filterbank())


# ------------------------------------------------------------------ PPG extractor oracle (whisper/model.py:144-163)
WHISPER_GOLDEN = ["whisper_d256_l8_b2_n200", "whisper_d512_l4_b1_n301"]


def _whisper_case(name):
    from oracle import make_golden as mg
    over, ck_seed, B, n, in_seed = mg.WHISPER_CASES[name]
    return synth.whisper_checkpoint(mg.whisper_dims(over), seed=ck_seed), mg.whisper_mel(in_seed, B, n)


@pytest.mark.parametrize("name", WHISPER_GOLDEN)
def test_whisper_oracle_matches_golden(name):
    """tests/golden/whisper_*.npz are outputs of the unmodified reference `Whisper.encoder` after the
    loader surgery (oracle/make_golden.py:whisper_case); the restatement must reproduce them."""
    from oracle import whisper_oracle as wo
    g = _load(name)
    ck, mel = _whisper_case(name)
    assert np.array_equal(mel.numpy(), g["mel"])          # the input recipe is reproducible
    got = wo.audio_encoder(ck, mel)
    assert got.shape == g["ppg"].shape
    assert max_abs(got, g["ppg"]) <= 1e-5


@pytest.mark.parametrize("over,B,n", [(dict(n_audio_state=256, n_audio_head=4, n_audio_layer=8), 2, 120),
                                      (dict(n_audio_state=384, n_audio_head=6, n_audio_layer=4), 1, 77)])
def test_whisper_oracle_matches_reference_live(over, B, n, pins):
    """The pin itself: reference `Whisper(dims)` -> `del decoder`, `del encoder.blocks[-(n//4):]`,
    `load_state_dict(strict=False)` exactly as whisper/inference.py:11-20, then `model.encoder(mel)`
    against `whisper_oracle.audio_encoder` on the same checkpoint and mel."""
    from oracle import make_golden as mg, whisper_oracle as wo
    ck = synth.whisper_checkpoint(mg.whisper_dims(over), seed=5)
    mel = mg.whisper_mel(6, B, n)
    case = mg.WHISPER_PIN_CASES.index((over, B, n))   # the stored reference output of these dims and shapes
    assert int(pins[f"whisper{case}_kept_layers"]) == wo.kept_layers(ck["dims"])
    ref = pins[f"whisper{case}_ppg"]                 # float64, as the oracle below (make_golden.py:reference_pins)
    got = wo.audio_encoder(mg.to_float64(ck), mel.double())
    assert got.shape == ref.shape == (B, (n - 1) // 2 + 1, over["n_audio_state"])
    assert max_abs64(got, ref) <= 1e-6


# ----------------------------------------------------------------------------- HuBERT-Soft (SURVEY §8f-2)
HUBERT_GOLDEN = ["hubert_soft_b2_n8000", "hubert_soft_b1_n16123"]


def _hubert_case(name):
    from oracle import make_golden as mg
    ck_seed, B, n, in_seed = mg.HUBERT_CASES[name]
    return synth.hubert_checkpoint(ck_seed), mg.hubert_wav(in_seed, B, n)


@pytest.mark.parametrize("name", HUBERT_GOLDEN)
def test_hubert_oracle_matches_golden(name):
    """tests/golden/hubert_*.npz are outputs of the unmodified reference `HubertSoft.units`
    (oracle/make_golden.py:hubert_case); the restatement must reproduce them."""
    from oracle import hubert_oracle as ho
    g = _load(name)
    sd, wav = _hubert_case(name)
    assert np.array_equal(wav.numpy(), g["wav"])           # the input recipe is reproducible
    got = ho.units(sd, wav)
    assert got.shape == g["units"].shape == (wav.shape[0], ho.frames(wav.shape[-1]), 256)
    assert max_abs(got, g["units"]) <= 2e-5


def test_hubert_oracle_matches_reference_live(pins):
    """The pin itself: the reference's `HubertSoft()` with the synthetic state dict loaded (strict), `units(wav)`
    (hubert/hubert_model.py:68-72) against `hubert_oracle.units` on the same state dict and audio."""
    from oracle import hubert_oracle as ho, make_golden as mg
    sd = synth.hubert_checkpoint(7)
    wav = mg.hubert_wav(8, 1, 5003)
    ref = pins["hubert_units"]
    got = ho.units(sd, wav)
    assert got.shape == ref.shape == (1, ho.frames(5003), 256)
    assert max_abs(got, ref) <= 2e-5
