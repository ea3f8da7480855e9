"""The pitch-shift sweep (svc_inference_shift.py) on the device: every shift of one engine run is bitwise its lone run,
the extreme shifts match the oracle's chunk loop, and the CLI writes the reference's files."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy.io import wavfile

from oracle import svc_oracle as O
from tests.util import ROOT
from whisper_vits_svc_b200 import hostio

pytestmark = pytest.mark.gpu
HOP = 320
N = 2600                      # -> chunks (0, 2510) and (2490, 2600)
SHIFTS = [-12, -5, 0, 7, 12]


class Quiet:   # the random draws silenced, so that every run is deterministic
    def __init__(self, m, C):
        self.m, self.C = m, C

    def pitch2source(self, f0, **kw):
        B, T = f0.shape
        return self.m.pitch2source(f0, rand_ini=torch.zeros(B, 11), noise=torch.zeros(B, T * HOP, 11))

    def inference_ragged(self, ppg, vec, pit, spk, n_frames, source, eps=None):
        return self.m.inference_ragged(ppg, vec, pit, spk, n_frames, source,
                                       eps=torch.zeros(ppg.shape[0], self.C, ppg.shape[1]))


@pytest.fixture(scope="module")
def model_tc(hp, sd):
    from whisper_vits_svc_b200 import models
    m = models.SynthesizerInfer(513, 25, hp, precision=3)
    m.load_state_dict(sd)
    return m.to("cuda")


@pytest.fixture(scope="module")
def utterance(hp):
    g = torch.Generator().manual_seed(23)
    pit = [int(v) for v in torch.randint(100, 500, (N,), generator=g)]
    pit[700:900] = [0] * 200
    return (torch.randn(hp.vits.spk_dim, generator=g) * 0.05, pit, torch.randn(N, hp.vits.ppg_dim, generator=g),
            torch.randn(N, hp.vits.vec_dim, generator=g))


def _jobs(utt, shifts):
    spk, pit, ppg, vec = utt
    return [(s, spk, hostio.shift_pitch(pit, s), ppg, vec) for s in shifts]


@pytest.fixture(scope="module")
def sweep(model_tc, hp, utterance):
    eng = hostio.BatchEngine(Quiet(model_tc, hp.vits.inter_channels), hp, "cuda", ragged=True)
    return eng, dict(eng.run(iter(_jobs(utterance, SHIFTS))))


def test_each_shift_equals_its_lone_run(model_tc, hp, utterance, sweep):
    eng, got = sweep
    assert list(got) == SHIFTS
    lone_calls = 0
    for s in SHIFTS:
        lone = hostio.BatchEngine(Quiet(model_tc, hp.vits.inter_channels), hp, "cuda", ragged=True)
        (key, want), = lone.run(iter(_jobs(utterance, [s])))
        lone_calls += lone.batches
        assert key == s and got[s].shape == want.shape == (N * HOP - 1,)
        assert np.array_equal(got[s], want), (s, float(np.abs(got[s] - want).max()))
    assert eng.batches < lone_calls, (eng.batches, lone_calls)
    assert not np.array_equal(got[-12], got[12])


@pytest.mark.parametrize("shift", [-12, 12])
def test_extreme_shifts_match_the_oracle_chunk_loop(hp, sd, utterance, sweep, shift):
    spk, pit, ppg, vec = utterance
    p = hostio.shift_pitch(pit, shift)
    src = O.pitch2source(sd, hp, p[None], torch.zeros(1, 11), torch.zeros(1, N * HOP, 11))
    ref = []
    for cs, ce, so, eo in hostio.chunk_plan(N, HOP):
        w = O.synthesizer_infer(sd, hp, ppg[None, cs:ce], vec[None, cs:ce], p[None, cs:ce], spk[None],
                                torch.tensor([ce - cs]), src[:, :, cs * HOP:ce * HOP],
                                torch.zeros(1, hp.vits.inter_channels, ce - cs))
        ref.append(w[0, 0].numpy()[so:eo])
    ref = np.concatenate(ref)
    err = float(np.abs(sweep[1][shift] - ref).max())
    print(f"shift {shift}, 26 s utterance in the sweep: max-abs {err:.3e} against the oracle")
    assert err <= 2e-4


def test_cli_writes_every_shift(tmp_path, hp, sd):
    from whisper_vits_svc_b200 import models
    m = models.SynthesizerInfer(513, 25, hp)
    m.load_state_dict(sd)
    hostio.save_svc_model(m, str(tmp_path / "g.pth"))
    rs = np.random.RandomState(4)
    n = 300                                             # the frames all features share (20 ms rows are repeated x2)
    np.save(tmp_path / "x.ppg.npy", rs.randn(n // 2, hp.vits.ppg_dim).astype(np.float32))
    np.save(tmp_path / "x.vec.npy", rs.randn(n // 2 + 1, hp.vits.vec_dim).astype(np.float32))
    np.save(tmp_path / "x.spk.npy", (rs.randn(hp.vits.spk_dim) * 0.05).astype(np.float32))
    pit = rs.randint(100, 500, size=n + 5)
    pit[40:90] = 0
    hostio.save_csv_pitch(pit, str(tmp_path / "x.pit.csv"))
    cmd = [sys.executable, os.path.join(ROOT, "svc_inference_shift.py"), "--config", os.path.join(ROOT, "configs", "base.yaml"),
           "--model", "g.pth", "--wave", "x.wav", "--spk", "x.spk.npy", "--ppg", "x.ppg.npy", "--vec", "x.vec.npy",
           "--pit", "x.pit.csv", "--shift_l", "-2", "--shift_r", "1"]
    r = subprocess.run(cmd, cwd=tmp_path, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = r.stdout.splitlines()
    assert "pitch shift: [-2, 1]" in lines
    assert lines[lines.index("pitch shift: [-2, 1]") + 1:][:4] == ["-2", "-1", "0", "1"]
    assert sorted(os.listdir(tmp_path / "_svc_out")) == sorted(f"svc_out_{s}.wav" for s in (-2, -1, 0, 1))
    waves = {}
    for s in (-2, -1, 0, 1):
        rate, w = wavfile.read(tmp_path / "_svc_out" / f"svc_out_{s}.wav")
        assert rate == 32000 and w.dtype == np.float32 and w.shape == (n * HOP - 1,) and np.isfinite(w).all(), s
        waves[s] = w
    assert all(not np.array_equal(waves[a], waves[b]) for a in waves for b in waves if a < b)
    rate, pw = wavfile.read(tmp_path / "svc_out_pit.wav")
    assert rate == 32000 and pw.dtype == np.int16 and pw.shape == (n * HOP,)
