"""Linear spectrograms on the device (svcb_linear_spec_ragged, spectrogram.spec_batch, preprocess_spec.py).

Parity with the fixture made by the oracle, within max|dev - ref| <= 2e-5 * max(1, max|ref|) per clip; ragged batches
bitwise equal to lone runs; passes of more than one launch; silence; and the CLI end to end on a small dataset."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import spec_oracle as SO
from tests.util import ROOT
from whisper_vits_svc_b200 import _lib, hparams, spectrogram

pytestmark = pytest.mark.gpu

GROUP = 128   # items per launch (csrc/spec_api.cu SPEC_GROUP)


@pytest.fixture(scope="module")
def hp():
    return hparams.load_hparams(os.path.join(ROOT, "configs", "base.yaml"))


def _gate(tag, got, ref):
    ref = torch.as_tensor(ref)
    assert got.shape == ref.shape and got.dtype == torch.float32, (tag, got.shape, ref.shape)
    err, scale = float((got - ref).abs().max()), max(1.0, float(ref.abs().max()))
    print(f"{tag}: max|dev - ref| {err:.3e}, {err / scale:.3e} of max(1, max|ref|)")
    assert err <= 2e-5 * scale, tag
    return err / scale


def _clip(seed, n):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 32000
    x = 0.4 * np.sin(2 * np.pi * (120.0 + 37 * (seed % 11)) * t) + 0.05 * rng.standard_normal(n)
    return x.astype(np.float32)


def test_fixture_parity(hp):
    g = SO.load_golden()
    names = sorted(g)
    out = spectrogram.spec_batch([g[k][0] for k in names], hp)
    worst = max(_gate(k, o, g[k][1]) for k, o in zip(names, out))
    print(f"worst over the fixture: {worst:.3e}")


def test_ragged_equals_lone_in_two_orders(hp):
    lens = [353, 640, 320 * 8 + 1, 320 * 500 + 17, 32000 * 3, 354, 320 * 9 - 1]
    clips = [_clip(i, n) for i, n in enumerate(lens)]
    lone = [spectrogram.spec_batch([c], hp)[0] for c in clips]
    for order in (list(range(len(clips))), list(reversed(range(len(clips))))):
        out = spectrogram.spec_batch([clips[i] for i in order], hp)
        for o, i in zip(out, order):
            assert o.shape == (513, lens[i] // 320)
            assert torch.equal(o, lone[i]), (i, lens[i])


def test_more_than_one_pass_and_a_long_clip(hp):
    rng = np.random.default_rng(3)
    lens = [int(n) for n in rng.integers(353, 320 * 40, GROUP + 5)]
    clips = [_clip(100 + i, n) for i, n in enumerate(lens)] + [_clip(7, 60 * 32000)]
    out = spectrogram.spec_batch(clips, hp)
    assert len(out) == len(clips)
    for i in list(range(0, len(clips), 9)) + [GROUP - 1, GROUP, len(clips) - 1]:
        _gate(f"item {i} ({clips[i].shape[0]} samples)", out[i], SO.spectrogram(torch.from_numpy(clips[i])[None])[0])
    assert torch.equal(out[GROUP], spectrogram.spec_batch([clips[GROUP]], hp)[0])   # first item of the second pass


def test_silence(hp):
    s = spectrogram.spec_batch([np.zeros(320 * 12 + 5, np.float32)], hp)[0]
    assert s.shape == (513, 12)
    assert torch.equal(s, torch.full_like(s, float(torch.tensor(1e-6, dtype=torch.float32).sqrt())))


def test_lengths_are_validated(hp):
    for bad in ([np.zeros(352, np.float32)], [np.zeros(1000, np.float32), np.zeros(100, np.float32)]):
        with pytest.raises(_lib.SvcbError, match="352"):
            spectrogram.spec_batch(bad, hp)


def test_cli_end_to_end(tmp_path):
    from scipy.io import wavfile
    (tmp_path / "configs").mkdir()
    (tmp_path / "configs" / "base.yaml").write_text(open(os.path.join(ROOT, "configs", "base.yaml")).read())
    wav = tmp_path / "wav"
    for s in ("spk_a", "spk_b"):
        (wav / s).mkdir(parents=True)

    def pcm(x):
        return (np.clip(x, -1, 1) * 32767).astype(np.int16)

    good = {"spk_a/a2": 32000 * 2 + 17, "spk_a/a9": 32000 * 9, "spk_a/tiny": 353, "spk_b/b5": 32000 * 5 + 319}
    for i, (g, n) in enumerate(good.items()):
        wavfile.write(wav / f"{g}.wav", 32000, pcm(_clip(i, n)))
    wavfile.write(wav / "spk_a" / "sr16k.wav", 16000, pcm(_clip(10, 16000)))
    wavfile.write(wav / "spk_b" / "stereo.wav", 32000, pcm(np.stack([_clip(11, 32000), _clip(12, 32000)], 1)))
    wavfile.write(wav / "spk_b" / "short.wav", 32000, pcm(_clip(13, 300)))
    (tmp_path / "spe" / "spk_b").mkdir(parents=True)
    torch.save(torch.zeros(1), tmp_path / "spe" / "spk_b" / "b5.pt")        # overwritten
    r = subprocess.run([sys.executable, os.path.join(ROOT, "preprocess_spec.py"), "-w", "wav", "-s", "spe", "-t", "2",
                        "--batch", "2"], cwd=tmp_path, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert r.stdout.splitlines()[:2] == ["wav", "spe"]
    for bad in ("sr16k.wav", "stereo.wav", "short.wav"):
        assert bad in r.stderr, bad
    assert "3 of 7 files failed" in r.stderr
    for s in ("spk_a", "spk_b"):
        assert sorted(os.listdir(tmp_path / "spe" / s)) == sorted(f"{g.split('/')[1]}.pt" for g in good if g.startswith(s))
    for g, n in good.items():
        spec = torch.load(tmp_path / "spe" / f"{g}.pt")
        assert spec.dtype == torch.float32 and spec.shape == (513, n // 320) and spec.is_contiguous()
        assert spec.untyped_storage().nbytes() == 4 * 513 * (n // 320)   # not the whole batch's buffer
        _gate(f"cli {g}", spec, SO.compute_spec(str(wav / f"{g}.wav")))
