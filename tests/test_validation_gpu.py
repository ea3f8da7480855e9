"""The validation score on the device (svcb_tacotron_mel, validation.py, svc_validate.py).

The device mels of the fixture's audio match the oracle's (tests/golden/validation_synth.npz): within 1e-3 where the
mel is at least 1e-3 and exactly ln(1e-5) on digital silence.  Each item's mel is bitwise the same alone and at any
position of any batch; bad input is refused before any launch.  The validation pass with the fixture's draws gives the
fixture's mel_loss within 1e-4 relative and hands over the logged audio of item 0 of each batch.  A checkpoint scores
bitwise the same alone, twice and after another, and as its export; the peak device memory does not grow with the
number of checkpoints; the CLI scores a set of checkpoints, reports a corrupt one and exits with 1."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import yaml

from oracle import validation_oracle as V
from tests.util import ROOT
from whisper_vits_svc_b200 import _lib, synth, validation

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def hp():
    return V.load_hp()


@pytest.fixture(scope="module")
def data(hp, tmp_path_factory):
    files = V.write_dataset(str(tmp_path_factory.mktemp("valid")), hp)
    batches, n = V.read_batches(files, hp, V.CROP_SEED, V.BATCH)
    return files, batches, n


@pytest.fixture(scope="module")
def scorer(hp):
    s = validation.Scorer(hp, "cuda")
    yield s
    s.close()


def _silent_frames(x):
    """Frames (L // 320 of a row x) whose reflect-padded 1024-sample window is all zeros."""
    p = np.pad(x, (V.PAD, V.PAD), mode="reflect")
    T = x.size // V.HOP
    return np.array([not np.any(p[t * V.HOP:t * V.HOP + V.N_FFT]) for t in range(T)])


def _check_mel(got, want, audio, what):
    got, want = got.cpu().numpy(), np.asarray(want)
    assert got.shape == want.shape
    big = want >= np.log(1e-3)
    err_big = float(np.abs(got - want)[big].max())
    err_all = float(np.abs(got - want).max())
    print(f"{what}: max-abs {err_big:.2e} where mel >= 1e-3 ({big.mean():.1%} of values), {err_all:.2e} overall")
    assert err_big <= 1e-3
    for b in range(audio.shape[0]):
        sil = _silent_frames(audio[b])
        assert sil.any() or what.startswith("fake")
        assert np.all(got[b][:, sil] == np.float32(V.LOG_CLIP))


def test_mel_against_fixture(hp, data):
    g = V.load_golden()
    basis = validation.mel_basis(hp).cuda()
    _, batches, _ = data
    for i, bt in enumerate(batches):
        audio = bt[7].squeeze(1)
        _check_mel(validation.tacotron_mel(audio.cuda(), basis), g[f"mel_real_{i}"], audio.numpy(), f"real {i}")
        fake = torch.from_numpy(g[f"fake_audio_{i}"])[None]
        _check_mel(validation.tacotron_mel(fake.cuda(), basis), g[f"mel_fake_{i}"][:1], fake.numpy(), f"fake {i}")


def test_mel_items_independent(hp):
    basis = validation.mel_basis(hp).cuda()
    g = torch.Generator().manual_seed(3)
    L = 320 * 77 + 13
    rows = (torch.rand(5, L, generator=g) * 2 - 1) * 0.8
    rows[2, 4000:9000] = 0.0
    alone = [validation.tacotron_mel(rows[i:i + 1].cuda(), basis) for i in range(5)]
    for perm in ([0, 1, 2, 3, 4], [4, 2, 0, 3, 1], [3, 3, 1]):
        mel = validation.tacotron_mel(rows[perm].cuda(), basis)
        for pos, i in enumerate(perm):
            assert torch.equal(mel[pos], alone[i][0]), (perm, pos)


def test_mel_bad_input(hp):
    basis = validation.mel_basis(hp).cuda()
    x = torch.zeros(2, 4000, device="cuda")
    out = torch.empty(2, 100, 12, device="cuda")
    lib = _lib.load()
    n0 = _lib.last_launch_count()
    cases = [(x.data_ptr(), 0, 4000, basis.data_ptr(), 100, out.data_ptr(), -1),   # SVCB_E_BAD_SHAPE
             (x.data_ptr(), 2, 352, basis.data_ptr(), 100, out.data_ptr(), -1),
             (x.data_ptr(), 2, 4000, basis.data_ptr(), 0, out.data_ptr(), -3),   # SVCB_E_UNSUPPORTED
             (x.data_ptr(), 2, 4000, basis.data_ptr(), 129, out.data_ptr(), -3),
             (None, 2, 4000, basis.data_ptr(), 100, out.data_ptr(), -1),
             (x.data_ptr(), 2, 4000, None, 100, out.data_ptr(), -1),
             (x.data_ptr(), 2, 4000, basis.data_ptr(), 100, None, -1)]
    for *args, code in cases:
        assert lib.svcb_tacotron_mel(*args, _lib.stream()) == code, args
    assert _lib.last_launch_count() == n0
    with pytest.raises(ValueError, match="leaves"):
        validation.tacotron_mel(torch.full((1, 4000), 1.5, device="cuda"), basis)


def _exported(path, hp, seed):
    torch.save({"model_g": synth.svc_state_dict(hp, seed)}, path)
    return str(path)


def _fixture_set(hp, data):
    files, _, _ = data
    return validation.load_set(hp, files, V.CROP_SEED, V.BATCH, "cuda", draw=V.cpu_draws(V.DRAW_SEED))


def _scores(scorer, paths, vset, on_audio=None):
    out = []
    scorer.score_paths(paths, vset, lambda p, loss, err: out.append((p, loss, err)), on_audio)
    return out


def test_loss_against_fixture(hp, data, scorer, tmp_path):
    g = V.load_golden()
    vset = _fixture_set(hp, data)
    assert vset.n_items == len(V.ITEM_FRAMES) and len(vset.batches) == 2
    ck = _exported(tmp_path / "w.pth", hp, V.WEIGHT_SEED)
    logged = {}
    (p, loss, err), = _scores(scorer, [ck], vset, lambda p, idx, r, f: logged.setdefault(idx, (r, f)))
    assert err is None
    want = float(g["mel_loss"])
    print(f"mel_loss device {loss!r}, oracle {want!r}, rel {abs(loss - want) / want:.2e}")
    assert abs(loss - want) <= 1e-4 * want
    assert sorted(logged) == [0, 1]
    _, batches, _ = data
    for idx, (real, fake) in logged.items():
        assert np.array_equal(real, batches[idx][7][0, 0].numpy())
        e = float(np.abs(fake - g[f"fake_audio_{idx}"]).max())
        print(f"logged fake audio {idx}: max-abs {e:.2e}")
        assert e <= 1e-3


def test_scores_deterministic(hp, data, scorer, tmp_path):
    vset = validation.load_set(hp, data[0], 5, 2, "cuda")
    a = _exported(tmp_path / "a.pth", hp, 21)
    b = _exported(tmp_path / "b.pth", hp, 22)
    alone = _scores(scorer, [a], vset)[0][1]
    twice = [s[1] for s in _scores(scorer, [a, a], vset)]
    after = [s[1] for s in _scores(scorer, [b, a], vset)]
    assert twice == [alone, alone] and after[1] == alone and after[0] != alone
    # a trainer checkpoint and its export
    sd = synth.svc_state_dict(hp, 23)
    gen = torch.Generator().manual_seed(1)
    trainer = dict(sd, **{"enc_q.pre.weight": torch.randn(192, 513, 1, generator=gen),
                          "emb_g.weight": torch.randn(256, 256, generator=gen)})
    tr = tmp_path / "trainer.pt"
    torch.save({"model_g": trainer, "model_d": {"w": torch.randn(8, generator=gen)}, "optim_g": {}, "optim_d": {},
                "step": 1, "epoch": 1, "hp_str": ""}, tr)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "svc_export.py"), "-c", os.path.join(ROOT, "configs", "base.yaml"),
                        "-p", str(tr)], cwd=tmp_path, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    s_tr, s_ex = [s[1] for s in _scores(scorer, [str(tr), str(tmp_path / "sovits5.0.pth")], vset)]
    assert s_tr == s_ex


def test_memory_flat(hp, data, tmp_path):
    vset = validation.load_set(hp, data[0], 5, 2, "cuda")
    paths = [_exported(tmp_path / f"{i}.pth", hp, 30 + i) for i in range(5)]
    s = validation.Scorer(hp, "cuda")
    try:
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        _scores(s, paths[:1], vset)
        torch.cuda.synchronize()
        one = torch.cuda.max_memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        _scores(s, paths, vset)
        torch.cuda.synchronize()
        five = torch.cuda.max_memory_allocated()
    finally:
        s.close()
    print(f"peak device memory: {one} B after one checkpoint, {five} B after five")
    assert five == one


def test_cli(hp, data, tmp_path):
    files = data[0]
    with open(os.path.join(ROOT, "configs", "base.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg["data"]["validation_files"] = files
    cfg["train"]["batch_size"] = 2
    conf = tmp_path / "base.yaml"
    conf.write_text(yaml.safe_dump(cfg))
    a = _exported(tmp_path / "a.pth", hp, 41)
    b = _exported(tmp_path / "b.pth", hp, 42)
    bad = tmp_path / "bad.pt"
    bad.write_bytes(b"not a checkpoint")
    out = tmp_path / "audio"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "svc_validate.py"), "-c", str(conf), "-p", a, str(bad), b,
                        "--audio-dir", str(out)], cwd=tmp_path, capture_output=True, text=True)
    print(r.stdout, r.stderr)
    assert r.returncode == 1
    assert "bad.pt" in r.stderr
    lines = [ln for ln in r.stdout.splitlines() if "\t" in ln]
    assert [ln.split("\t")[0] for ln in lines[:2]] == [a, b]
    losses = [float(ln.split("\t")[1]) for ln in lines[:2]]
    assert lines[2] == f"best: {[a, b][int(np.argmin(losses))]}\t{min(losses)!r}"
    names = sorted(os.listdir(out))
    assert names == ["a.pth", "b.pth", "real_0.wav", "real_1.wav"]
    assert sorted(os.listdir(out / "a.pth")) == ["fake_0.wav", "fake_1.wav"]
