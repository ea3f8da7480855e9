"""CREPE without a device: the oracle's Viterbi against exhaustive search, the oracle against the unmodified reference
and the stored goldens, the real `tiny` weights against the physics of steady tones, frame counts, the packer's layouts
and the command lines' no-device message."""
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import crepe_oracle as O
from tests.util import ROOT
from whisper_vits_svc_b200 import crepe_infer as C, synth

GOLD = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def tiny_sd():
    return O.tiny_weights()


@pytest.fixture(scope="module")
def tones():
    return dict(np.load(os.path.join(GOLD, "crepe_tiny_tones.npz")).items())


def _brute(prob, trans):
    S, T = prob.shape
    tiny = np.finfo(prob.dtype).tiny
    lp, lt, best, arg = np.log(prob.T.astype(np.float64) + tiny), np.log(trans + tiny), -np.inf, None
    for path in itertools.product(range(S), repeat=T):   # lexicographic, so the first maximum has the lowest last states
        v = lp[0, path[0]] + np.log(1.0 / S + tiny)
        for t in range(1, T):
            v = v + lt[path[t - 1], path[t]] + lp[t, path[t]]
        if v > best:
            best, arg = v, path
    return best, np.array(arg)


def _score(prob, trans, path):
    tiny = np.finfo(prob.dtype).tiny
    v = np.log(prob[path[0], 0].astype(np.float64) + tiny) + np.log(1.0 / prob.shape[0] + tiny)
    for t in range(1, len(path)):
        v += np.log(trans[path[t - 1], path[t]] + tiny) + np.log(prob[path[t], t].astype(np.float64) + tiny)
    return v


@pytest.mark.parametrize("seed", range(6))
def test_viterbi_equals_exhaustive_search(seed):
    g = np.random.default_rng(seed)
    trans = O.transition_matrix(4) if seed % 2 else g.random((4, 4))
    trans = trans / trans.sum(1, keepdims=True)
    prob = g.random((4, 6)).astype(np.float32)
    if seed >= 3:   # ties: repeated columns and a zero
        prob = np.round(prob * 2) / 2
    best, _ = _brute(prob, trans)
    path = O.viterbi(prob, trans)
    assert np.isclose(_score(prob, trans, path), best, rtol=0, atol=1e-12)
    if seed < 3:
        assert np.array_equal(path, _brute(prob, trans)[1])


def test_decode_restarts_every_segment(tones):
    masked = torch.from_numpy(tones["probs160"])
    masked = torch.cat([masked, masked.flip(0)])[:600]
    bins, _, _ = O.decode(masked, None)
    trans = O.transition_matrix()
    parts = [O.viterbi(torch.softmax(masked[s:s + 512].T, 0).numpy(), trans) for s in (0, 512)]
    assert np.array_equal(bins.numpy(), np.concatenate(parts))
    assert O.frequency_to_bins(50) == C.BIN_LO and O.frequency_to_bins(1000, True) == C.BIN_HI


def test_oracle_equals_goldens_and_reference(tiny_sd, tones):
    audio, noise = torch.from_numpy(tones["audio"]), torch.from_numpy(tones["noise"])
    for hop in (160, 320):
        dither = torch.from_numpy(tones[f"dither{hop}"])
        masked, bins, pitch, period = O.predict(tiny_sd, audio, hop, noise, dither)
        assert torch.allclose(masked[:, 39:299], torch.from_numpy(tones[f"probs{hop}"])[:, 39:299], atol=1e-6)
        assert torch.isinf(masked[:, :39]).all() and torch.isinf(masked[:, 299:]).all()
        assert np.array_equal(bins.numpy(), tones[f"bins{hop}"])
        assert np.allclose(pitch.numpy(), tones[f"pitch{hop}"], rtol=1e-6)
        assert np.allclose(period.numpy(), tones[f"periodicity{hop}"], atol=1e-6)
        if O.reference_available():
            r_probs, r_pitch, r_period = O.reference_predict(tiny_sd, "tiny", audio, hop, noise, dither)
            assert torch.equal(O.mask(r_probs), torch.from_numpy(tones[f"probs{hop}"]))
            assert torch.equal(r_pitch, torch.from_numpy(tones[f"pitch{hop}"]))
            assert torch.equal(r_period, torch.from_numpy(tones[f"periodicity{hop}"]))
    sing = O.compute_f0_sing(tiny_sd, audio, noise, torch.from_numpy(tones["dither320"]))
    assert O.csv_text(sing) == bytes(tones["csv"]).decode()
    assert np.allclose(O.compute_f0(tiny_sd, audio, noise, torch.from_numpy(tones["dither160"])), tones["pit"], rtol=1e-6,
                       equal_nan=True)


@pytest.mark.skipif(not O.reference_available(), reason="needs the reference tree")
def test_filters_equal_reference():
    crepe = O.import_reference()
    g = torch.Generator().manual_seed(1)
    x = torch.rand(1, 40, generator=g) * 300
    x[0, [3, 4, 17, 39]] = float("nan")
    x[0, [8, 9, 10, 11, 12]] = 0.0
    for ours, oracle, ref, win in ((C.mean, O.mean, crepe.filter.mean, 5), (C.median, O.median, crepe.filter.median, 7)):
        want = ref(x.clone(), win)[0].numpy()
        assert np.allclose(ours(x[0].clone(), win).numpy(), want, rtol=1e-6, equal_nan=True)
        assert np.allclose(oracle(x[0].numpy(), win), want, rtol=1e-6, equal_nan=True)


def test_host_filters_equal_oracle():
    g = torch.Generator().manual_seed(2)
    x = torch.rand(33, generator=g) * 300
    x[[0, 5, 6, 32]] = float("nan")
    x[[20, 21, 22, 23, 24]] = 0.0
    assert np.allclose(C.mean(x.clone(), 5).numpy(), O.mean(x.numpy(), 5), rtol=1e-6, equal_nan=True)
    assert np.allclose(C.median(x.clone(), 7).numpy(), O.median(x.numpy(), 7), rtol=1e-6, equal_nan=True)
    assert torch.isnan(C.mean(x.clone(), 5)[22])   # an exact zero becomes NaN


def test_tiny_weights_find_steady_tones(tiny_sd, tones):
    audio, noise = torch.from_numpy(tones["audio"]), torch.from_numpy(tones["noise"])
    pitch = O.predict(tiny_sd, audio, 160, noise, torch.zeros(1 + audio.numel() // 160))[2].numpy()
    for k, f in enumerate((110.0, 220.0, 440.0, 880.0)):
        assert np.abs(1200 * np.log2(pitch[k * 50 + 10:k * 50 + 40] / f)).max() <= 20.0, f


@pytest.mark.parametrize("n", [0, 1, 159, 160, 1023, 1024, 16000])
def test_frame_counts(n):
    for hop in (160, 320):
        assert C.frames_of(n, hop) == 1 + n // hop == O.frames(torch.zeros(n), hop).shape[0]
    assert torch.count_nonzero(O.frames(torch.zeros(n), 160)) == 0


@pytest.mark.parametrize("capacity", ["full", "tiny"])
def test_packer_layout(capacity):
    sd = synth.crepe_checkpoint(3, capacity)
    items = dict(C.pack_crepe(C.check_model(sd, capacity), capacity))
    ch = C.CHANNELS[capacity]
    assert items["crepe.cls.wt"].shape == (4 * ch[6], 360)
    for i in range(6):
        p = f"crepe.conv{i + 1}"
        w = sd[f"conv{i + 1}.weight"].squeeze(-1)
        bn = {n: sd[f"conv{i + 1}_BN.{n}"] for n in ("weight", "bias", "running_mean", "running_var")}
        x = torch.linspace(0, 2, 7)[:, None]
        want = (x - bn["running_mean"]) / torch.sqrt(bn["running_var"] + C.BN_EPS) * bn["weight"] + bn["bias"]
        assert torch.allclose(x * items[p + ".scale"] + items[p + ".shift"], want, atol=1e-5)
        assert (items[p + ".scale"] < 0).any()
        if capacity == "tiny":
            assert torch.equal(items[p + ".w"], w)
        elif i == 0:
            img = items[p + ".wimg"].view(torch.bfloat16).view(8, 64, 128, 8)
            assert torch.equal(img.permute(0, 2, 1, 3).reshape(1024, 512).float(), w.reshape(1024, 512).bfloat16().float())
        else:
            img = items[p + ".wimg"].view(torch.bfloat16)
            assert torch.equal(C.conv_image_unpack(img, ch[i + 1], ch[i], C.CONV_CK[i - 1]), w.bfloat16().float())
    with pytest.raises(ValueError, match="conv1.weight has shape"):
        C.check_model(sd, "tiny" if capacity == "full" else "full")


@pytest.mark.parametrize("cli", ["pitch_inference.py", "preprocess_crepe.py"])
def test_command_lines_need_a_device(cli, tmp_path):
    if torch.cuda.is_available():
        pytest.skip("a device is present")
    r = subprocess.run([sys.executable, os.path.join(ROOT, cli), "-w", "x", "-p", "y"], cwd=tmp_path, capture_output=True,
                       text=True, env=dict(os.environ, PYTHONPATH=ROOT))
    assert r.returncode != 0 and "this build has no CPU path: a CUDA (sm_90a) device is required" in r.stderr
