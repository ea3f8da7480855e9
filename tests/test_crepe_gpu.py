"""CREPE on the device against the fp32 oracle: framing, the network per layer and at the probabilities (`full` with
synthetic weights, `tiny` with the real ones), the decoder alone on golden probabilities, the tones end to end, ragged
batches and the two command lines."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import crepe_oracle as O
from tests.util import ROOT
from whisper_vits_svc_b200 import _lib, crepe_infer as C, hostio, synth

pytestmark = pytest.mark.gpu
GOLD = os.path.join(ROOT, "tests", "golden")
# measured on an H100 (DESIGN.md, CREPE): bf16 operands through K = 65,536 against the fp32 oracle
FULL_PROBS_MAX, FULL_LAYER_REL, TINY_PROBS_MAX = 1e-2, 1e-2, 2e-5


def _npz(name):
    return {k: v for k, v in np.load(os.path.join(GOLD, name)).items()}


@pytest.fixture(scope="module")
def tiny_sd():
    return O.tiny_weights()


@pytest.fixture(scope="module")
def tiny(tiny_sd):
    return C.CrepeB200(tiny_sd, "cuda", "tiny")


@pytest.fixture(scope="module")
def full_sd():
    return synth.crepe_checkpoint(int(_npz("crepe_full_synth.npz")["seed"]), "full")


@pytest.fixture(scope="module")
def full(full_sd):
    return C.CrepeB200(full_sd, "cuda", "full")


@pytest.fixture(scope="module")
def tones():
    return _npz("crepe_tiny_tones.npz")


def _inband(p):
    return p[:, C.BIN_LO:C.BIN_HI]


def test_framing():
    g = torch.Generator().manual_seed(3)
    clips = [torch.randn(5000, generator=g) * 0.1, torch.zeros(700), torch.randn(100, generator=g), torch.full((2048,), 0.5),
             torch.zeros(0)]
    noises = [torch.randn(c.numel(), generator=g) for c in clips]
    noises[3].zero_()   # a DC-only frame: with noise its deviation is 1e-3 and the quotient shows fp32 rounding of the mean
    for hop, nz in ((160, noises), (320, None)):
        fr, fo = C.frame_device(clips, hop, nz)
        fr = fr.cpu()
        assert list(fo) == list(np.cumsum([0] + [1 + c.numel() // hop for c in clips]))
        for b, c in enumerate(clips):
            want = O.frames(c, hop, None if nz is None else nz[b])
            assert (fr[fo[b]:fo[b + 1]] - want).abs().max() <= 1e-5, (hop, b)
    fr, fo = C.frame_device(clips, 320)
    assert torch.count_nonzero(fr[fo[1]:fo[2]]) == 0             # an all-zero file stays zeros
    assert torch.count_nonzero(fr[fo[3] + 2:fo[3] + 5]) == 0     # frames inside the DC run


def _full_images(model, n_frames):
    """The bf16 images conv2 .. conv6 read, from the model's workspace -> the outputs of conv1 .. conv5 as [F, C, P]."""
    chunk = max(16, -(-n_frames // 16) * 16)
    ws = model._handle._ws
    al = lambda x: -(-x // 256) * 256   # noqa: E731
    off = al(chunk * 4096) + al(chunk * 2048 * 4)
    outs = []
    for L in range(5):
        cin, G, R = C.CHANNELS["full"][L + 1], C.IMAGE_G[L], C.IMAGE_ROWS[L]
        nbytes = chunk // G * cin * R * 2
        img = ws[off:off + nbytes].view(torch.bfloat16).view(chunk // G, cin // 8, R, 8).float().cpu()
        P = 128 >> L
        rows = img[:, :, 31 * G:(31 + P) * G].reshape(chunk // G, cin // 8, P, G, 8)
        outs.append(rows.permute(0, 3, 1, 4, 2).reshape(chunk, cin, P)[:n_frames])
        off += al(nbytes)
    return outs


def test_full_layers_and_probs(full, full_sd):
    g = _npz("crepe_full_synth.npz")
    audio, noise = torch.from_numpy(g["audio"]), torch.from_numpy(g["noise"])
    probs, fo = full.probs_device([audio], int(g["hop"]), [noise])
    torch.cuda.synchronize()
    n = fo[-1]
    want, layers = O.network(full_sd, O.frames(audio, int(g["hop"]), noise), layers=True)
    assert torch.allclose(want, torch.from_numpy(g["probs"]), atol=1e-5)
    report = []
    for i, got in enumerate(_full_images(full, n)):
        ref = layers[i]
        rel = float((got - ref).norm() / ref.norm())
        report.append(f"conv{i + 1} max-abs {float((got - ref).abs().max()):.3e} rel-l2 {rel:.3e}")
        assert rel <= FULL_LAYER_REL, report
        if i >= 1:
            assert (ref - torch.from_numpy(g[f"layer{i + 1}"].astype(np.float32))).abs().max() <= 2e-2
    p = probs.cpu()
    assert torch.isinf(p[:, :C.BIN_LO]).all() and torch.isinf(p[:, C.BIN_HI:]).all()
    e = float((_inband(p) - _inband(want)).abs().max())
    rel = float((_inband(p) - _inband(want)).norm() / _inband(want).norm())
    report.append(f"probs max-abs {e:.3e} rel-l2 {rel:.3e}")
    print("\n".join(report))
    assert e <= FULL_PROBS_MAX, report


def test_tiny_probs(tiny, tiny_sd, tones):
    audio, noise = torch.from_numpy(tones["audio"]), torch.from_numpy(tones["noise"])
    for hop in (160, 320):
        probs, _ = tiny.probs_device([audio], hop, [noise])
        want = torch.from_numpy(tones[f"probs{hop}"])
        e = float((_inband(probs.cpu()) - _inband(want)).abs().max())
        print(f"tiny probs hop {hop} max-abs {e:.3e}")
        assert e <= TINY_PROBS_MAX


@pytest.mark.parametrize("lengths", [[1], [511], [512], [513], [1025], [1, 511, 512, 513, 1025, 7]])
def test_decoder_alone(tones, lengths):
    # the golden rows (426 frames) forwards, backwards and forwards again: long enough for three segments
    probs, dither = torch.from_numpy(tones["probs160"]), torch.from_numpy(tones["dither160"])
    probs, dither = torch.cat([probs, probs.flip(0), probs]), torch.cat([dither, dither.flip(0), dither])
    starts = [(37 * i) % 200 for i in range(len(lengths))]
    items = [probs[s:s + n] for s, n in zip(starts, lengths)]
    dith = [dither[s:s + n] for s, n in zip(starts, lengths)]
    fo = _lib.offsets(lengths)
    bins, pitch, period = C.decode_device(torch.cat(items).cuda(), fo, torch.cat(dith))
    for b, (p, d) in enumerate(zip(items, dith)):
        wb, wp, wq = O.decode(p, d)
        assert torch.equal(bins[fo[b]:fo[b + 1]].cpu().long(), wb), (b, lengths)
        assert (pitch[fo[b]:fo[b + 1]].cpu() - wp).abs().max() <= 1e-3
        assert torch.equal(period[fo[b]:fo[b + 1]].cpu(), wq)


def test_decoder_rejects_bad_arguments(tones):
    probs = torch.from_numpy(tones["probs160"][:10]).cuda()
    with pytest.raises(_lib.SvcbError, match="segment"):
        C.decode_device(probs, _lib.offsets([10]), None, segment=513)
    with pytest.raises(_lib.SvcbError, match="item 1 has 0 frames"):
        C.decode_device(probs, _lib.offsets([10, 0]), None)


def test_tones_end_to_end(tiny, tones):
    audio, noise, f0 = torch.from_numpy(tones["audio"]), torch.from_numpy(tones["noise"]), tones["f0"]
    for hop in (160, 320):
        dither = torch.from_numpy(tones[f"dither{hop}"])
        probs, fo = tiny.probs_device([audio], hop, [noise])
        bins, pitch, period = C.decode_device(probs, fo, dither)
        bins, ref = bins.cpu().numpy(), tones[f"bins{hop}"]
        assert np.mean(bins == ref) >= 0.99
        voiced = f0[np.minimum(np.arange(len(bins)) * hop, len(f0) - 1)] > 0
        assert np.abs(bins - ref)[voiced].max() <= 1
        assert np.abs(period.cpu().numpy() - tones[f"periodicity{hop}"])[bins == ref].max() <= 1e-4
    # steady tones, no dither: within one 20-cent bin of the truth
    pitch = C.predict(tiny, audio, 160, noise, torch.zeros(1 + audio.numel() // 160)).numpy()
    for k, f in enumerate((110.0, 220.0, 440.0, 880.0)):
        mid = pitch[k * 50 + 10:k * 50 + 40]
        assert np.abs(1200 * np.log2(mid / f)).max() <= 20.0, f
    text = O.csv_text(C.compute_f0_sing(tiny, audio, noise, torch.from_numpy(tones["dither320"])).numpy()).splitlines()
    gold = bytes(tones["csv"]).decode().splitlines()
    assert len(text) == len(gold) == 2 * (1 + audio.numel() // 320)
    diff = [(a, b) for a, b in zip(text, gold) if a != b]
    assert len(diff) <= 0.01 * len(gold)
    for a, b in diff:
        fa, fb = int(a.split(",")[1]), int(b.split(",")[1])
        assert abs(fa - fb) <= max(1, 0.0117 * max(fa, fb) + 1)
    pit = C.compute_f0(tiny, audio, noise, torch.from_numpy(tones["dither160"]))
    assert pit.dtype == np.float32 and pit.shape == tones["pit"].shape
    same = np.isclose(pit, tones["pit"], rtol=1e-5, atol=1e-3, equal_nan=True)
    assert same.mean() >= 0.99


@pytest.mark.parametrize("capacity", ["full", "tiny"])
def test_ragged_batch_is_bit_identical(capacity, full, tiny):
    model = full if capacity == "full" else tiny
    g = torch.Generator().manual_seed(5)
    clips = [torch.randn(n, generator=g) * 0.1 for n in (0, 100, 1600, 2999, 160, 5000, 1023)]
    noises = [torch.randn(c.numel(), generator=g) for c in clips]
    probs, fo = model.probs_device(clips, 160, noises)
    probs = probs.clone()
    for b, (c, nz) in enumerate(zip(clips, noises)):
        alone, _ = model.probs_device([c], 160, [nz])
        assert torch.equal(alone, probs[fo[b]:fo[b + 1]]), b


def test_command_lines(tmp_path, full_sd):
    import scipy.io.wavfile
    (tmp_path / "crepe" / "assets").mkdir(parents=True)
    torch.save(full_sd, tmp_path / "crepe" / "assets" / "full.pth")
    lengths = {"a/x.wav": 4000, "a/y.wav": 1000, "b/z.wav": 16000, "b/short.wav": 321}
    g = np.random.default_rng(0)
    for rel, n in lengths.items():
        (tmp_path / "waves" / os.path.dirname(rel)).mkdir(parents=True, exist_ok=True)
        scipy.io.wavfile.write(tmp_path / "waves" / rel, 16000, (g.standard_normal(n) * 3000).astype(np.int16))
    (tmp_path / "waves" / "a" / "bad.wav").write_bytes(b"not a wav")
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "preprocess_crepe.py"), "-w", "waves", "-p", "pitch", "--batch", "2"],
                       cwd=tmp_path, env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    # three frames are fewer than the median filter's reflect padding takes, in the reference too: reported and skipped
    assert "bad.wav" in r.stderr and "short.wav" in r.stderr
    assert not (tmp_path / "pitch" / "b" / "short.pit.npy").exists()
    del lengths["b/short.wav"]
    for rel, n in lengths.items():
        pit = np.load(tmp_path / "pitch" / (rel[:-4] + ".pit.npy"))
        assert pit.dtype == np.float32 and pit.shape == (1 + n // 160,)
    assert not (tmp_path / "pitch" / "a" / "bad.pit.npy").exists()
    r = subprocess.run([sys.executable, os.path.join(ROOT, "pitch_inference.py"), "-w", "waves/b/z.wav", "-p", "z.pit.csv"],
                       cwd=tmp_path, env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lines = (tmp_path / "z.pit.csv").read_text().splitlines()
    assert len(lines) == 2 * (1 + 16000 // 320)
    import re
    for i, line in enumerate(lines):
        m = re.fullmatch(r"(\d+)m (\d+)s ([ \d]{3}),(-?\d+)", line)
        assert m and int(m[1]) * 60000 + int(m[2]) * 1000 + int(m[3]) == 10 * i, line
    assert len(hostio.load_csv_pitch(str(tmp_path / "z.pit.csv"))) == len(lines)
