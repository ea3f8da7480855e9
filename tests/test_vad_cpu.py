"""Silero VAD, host side: the oracle against the fixtures and the live model, get_speech_timestamps against the live
reference, the post-processing mask and the model-file checks (no GPU)."""
import numpy as np
import pytest
import torch

from oracle import ref_import
from oracle import vad_oracle as VO
from whisper_vits_svc_b200 import vad_infer as V

needs_ref = pytest.mark.skipif(not ref_import.available(), reason="reference tree not present")


@pytest.fixture(scope="module")
def sd():
    return VO.load_tensors()


@pytest.mark.parametrize("name", VO.FIXTURES)
def test_oracle_against_fixtures(sd, name):
    g = VO.load_golden(name)
    for clip in VO.clips(g):
        p, e = VO.speech_probs(sd, g[f"{clip}.wav"])
        assert p.shape == g[f"{clip}.probs"].shape == (V.windows(g[f"{clip}.wav"].shape[0]),)
        dp = float(np.abs(p - g[f"{clip}.probs"]).max())
        de = float(np.abs(e - g[f"{clip}.enc"]).max())
        print(f"{name}/{clip}: prob max-abs {dp:.2e}, encoder max-abs {de:.2e}")
        assert dp <= 2e-6 and de <= 1e-5 * max(1.0, float(np.abs(g[f"{clip}.enc"]).max())), (clip, dp, de)


@needs_ref
def test_oracle_against_live_model(sd):
    model = VO.live_model()
    live_sd = {k[len("_model."):]: v for k, v in model.state_dict().items() if k.startswith("_model.")}
    for k, t in sd.items():
        assert torch.equal(t, live_sd[k]), k
    rng = np.random.default_rng(4)
    wavs = [VO.load_golden("vad_test10s")["test10s.wav"][:40000]]
    wavs += [(a * rng.standard_normal(n)).astype(np.float32) for a, n in ((0.05, 7000), (0.5, 9999), (1.0, 513))]
    for w in wavs:
        p, e = VO.live_probs(model, w)
        po, eo = VO.speech_probs(sd, w, per_window=True)
        dp, de = float(np.abs(p - po).max()), float(np.abs(e - eo).max())
        print(f"{w.shape[0]} samples: prob max-abs {dp:.2e}, encoder max-abs {de:.2e}")
        assert dp <= 2e-6 and de <= 1e-5 * max(1.0, float(np.abs(e).max()))


# ------------------------------------------------------------------------------------------------ timestamps
def _ours(probs, n, **kw):
    return V.get_speech_timestamps(np.asarray(probs, np.float32), n, **kw)


def _ref(probs, n, **kw):
    return VO.reference_timestamps(np.asarray(probs, np.float32), n, **kw)


def _random_probs(rng, W):
    """Runs of speech-like, silence-like and in-between probabilities, with exact threshold values sprinkled in."""
    out = []
    while len(out) < W:
        kind = rng.integers(4)
        n = int(rng.integers(1, 40))
        if kind == 0:
            out += list(rng.uniform(0.5, 1.0, n))
        elif kind == 1:
            out += list(rng.uniform(0.0, 0.05, n))
        elif kind == 2:
            out += list(rng.uniform(0.0, 1.0, n))
        else:
            out += list(rng.choice([0.2, 0.05, 0.5, 0.35, 0.19999], n))
    return np.array(out[:W], np.float32)


@needs_ref
def test_timestamps_random_sequences_equal_reference():
    rng = np.random.default_rng(17)
    for case in range(400):
        W = int(rng.integers(1, 400))
        n = W * 512 - int(rng.integers(0, 512))
        kw = dict(threshold=float(rng.choice([0.5, 0.2, 0.35])),
                  min_speech_duration_ms=int(rng.choice([250, 100, 0])),
                  max_speech_duration_s=float(rng.choice([float("inf"), 1.0, 2.5, 0.3])),
                  min_silence_duration_ms=int(rng.choice([100, 30, 300])),
                  speech_pad_ms=int(rng.choice([30, 0, 100])))
        p = _random_probs(rng, W)
        assert _ours(p, n, **kw) == _ref(p, n, **kw), (case, kw)


@needs_ref
@pytest.mark.parametrize("kw", [{}, {"threshold": 0.2}, {"max_speech_duration_s": 1.0}, {"max_speech_duration_s": 1.0, "threshold": 0.2}])
def test_timestamps_constructed_cases_equal_reference(kw):
    hi, lo, mid = 0.9, 0.01, 0.4
    cases = {
        "speech at both ends": [hi] * 20 + [lo] * 10 + [hi] * 20,
        "all speech": [hi] * 100,
        "blip shorter than 250 ms": [lo] * 10 + [hi] * 5 + [lo] * 20 + [hi] * 30 + [lo] * 10,
        "gap shorter than two pads": [hi] * 20 + [lo] * 4 + [hi] * 20 + [lo] * 1 + [hi] * 9 + [lo] * 10,
        "long speech, earlier silence": [hi] * 20 + [lo] * 5 + [hi] * 60 + [lo] * 3 + [hi] * 50,
        "long speech, no silence": [hi] * 150 + [lo] * 10,
        "long speech, still in silence at the limit": [hi] * 25 + [lo] * 4 + [mid] * 30 + [hi] * 10,
        "exactly at the thresholds": [0.5] * 10 + [0.35] * 10 + [0.2] * 10 + [0.05] * 10 + [0.5] * 12 + [0.0] * 8,
        "silence": [lo] * 50,
        "one window": [hi],
    }
    for name, p in cases.items():
        for tail in (0, 1, 511):
            n = len(p) * 512 - tail
            assert _ours(p, n, **kw) == _ref(p, n, **kw), (name, tail)


@pytest.mark.parametrize("name", VO.FIXTURES)
def test_timestamps_of_fixture_probabilities(name):
    g = VO.load_golden(name)
    for clip in VO.clips(g):
        ts = _ours(g[f"{clip}.probs"], g[f"{clip}.wav"].shape[0], threshold=0.2)
        assert np.array_equal(np.array([[t["start"], t["end"]] for t in ts], np.int64).reshape(-1, 2), g[f"{clip}.ts"]), clip


# ------------------------------------------------------------------------------------------------ the mask
def _reference_post(ref16, svc32, timestamps):
    """svc_inference_post.py:39-49 as the reference writes it."""
    ref_wave = np.array(ref16, np.float32)
    ref_wave[:] = 0
    for tag in timestamps:
        ref_wave[tag["start"]:tag["end"]] = 1
    ref_wave = np.repeat(ref_wave, 2, -1)
    svc_wave = np.array(svc32, np.float32)
    min_len = min(len(ref_wave), len(svc_wave))
    ref_wave = ref_wave[:min_len]
    svc_wave = svc_wave[:min_len]
    svc_wave[ref_wave == 0] = 0
    return svc_wave


@pytest.mark.parametrize("n16,n32,ts", [
    (16000, 40000, [{"start": 100, "end": 5000}, {"start": 9000, "end": 16000}]),   # the ref is shorter
    (16000, 20000, [{"start": 0, "end": 12000}]),                                   # the ref is longer
    (16000, 32000, []),                                                             # no speech
    (300, 1000, []),                                                                # shorter than one window
    (0, 1000, []),                                                                  # empty
])
def test_mask_rule(n16, n32, ts):
    rng = np.random.default_rng(n16 + n32)
    svc = rng.standard_normal(n32).astype(np.float32)
    svc0 = svc.copy()
    got = V.silence_outside_speech(ts, n16, svc)
    ref = _reference_post(np.ones(n16, np.float32), svc, ts)
    assert got.dtype == np.float32 and got.shape == (min(2 * n16, n32),)
    assert np.array_equal(got, ref)
    assert np.array_equal(svc, svc0)


# ------------------------------------------------------------------------------------------------ the model file
def test_read_model_round_trip(sd, tmp_path):
    path = str(tmp_path / "silero_vad.jit")
    VO.write_jit(path, sd)
    got = V.read_model(path)
    assert sorted(got) == sorted(V.SHAPES)
    for k in V.SHAPES:
        assert torch.equal(got[k], sd[k]), k
    names = [n for n, _ in V.pack_vad(got)]
    assert len(names) == len(set(names))


@needs_ref
def test_read_model_live_file(sd):
    got = V.read_model(VO.ref_model_path())
    for k in V.SHAPES:
        assert torch.equal(got[k], sd[k]), k


@pytest.mark.parametrize("change,match", [
    ("missing", "missing _model.decoder.rnn.weight_hh_l1"),
    ("shape", "encoder.12.weight has shape"),
    ("hop", "hop_length is 128"),
    ("to_pad", "to_pad is 2"),
    ("filter", "filter_length is 512"),
])
def test_read_model_rejections(sd, tmp_path, change, match):
    sd = dict(sd)
    kw = {}
    if change == "missing":
        del sd["decoder.rnn.weight_hh_l1"]
    elif change == "shape":
        sd["encoder.12.weight"] = torch.zeros(64, 32, 1)
    elif change == "hop":
        kw["hop_length"] = 128
    elif change == "to_pad":
        kw["to_pad"] = 2
    else:
        kw["filter_length"] = 512
    path = str(tmp_path / "m.jit")
    VO.write_jit(path, sd, **kw)
    with pytest.raises(ValueError, match=match):
        V.read_model(path)


def test_other_layout_rejected(tmp_path):
    path = str(tmp_path / "v5.jit")
    VO.write_jit(path, {"stft.forward_basis_buffer": torch.zeros(258, 1, 256), "decoder.rnn.weight_ih": torch.zeros(512, 128)})
    with pytest.raises(ValueError, match="not the Silero VAD 16 kHz model"):
        V.read_model(path)


def test_windows():
    assert [V.windows(n) for n in (0, 1, 511, 512, 513, 1024)] == [0, 1, 1, 1, 2, 2]
