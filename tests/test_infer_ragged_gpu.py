"""svcb_infer_ragged on the device: each chunk of a ragged batch is bitwise what a lone call of its own length gives,
whatever its padding holds; the ragged BatchEngine converts utterances bitwise as the equal-length one does."""
import numpy as np
import pytest
import torch

from whisper_vits_svc_b200 import _lib

pytestmark = pytest.mark.gpu
HOP = 320


def _model(hp, sd, precision):
    from whisper_vits_svc_b200 import models
    m = models.SynthesizerInfer(513, 25, hp, precision=precision)
    m.load_state_dict(sd)
    return m.to("cuda")


@pytest.fixture(scope="module")
def model_tc(hp, sd):
    return _model(hp, sd, 3)


def _ragged_inputs(hp, lens, T, seed):
    """Padded inputs whose padding (past each item's length) is finite garbage of magnitude 1e3."""
    g = torch.Generator().manual_seed(seed)
    B = len(lens)
    d = {"ppg": torch.randn(B, T, hp.vits.ppg_dim, generator=g), "vec": torch.randn(B, T, hp.vits.vec_dim, generator=g),
         "pit": torch.randint(100, 501, (B, T), generator=g).float(), "spk": torch.randn(B, hp.vits.spk_dim, generator=g) * 0.05,
         "source": torch.randn(B, 1, T * HOP, generator=g) * 0.1, "eps": torch.randn(B, hp.vits.inter_channels, T, generator=g)}
    d["pit"][:, T // 3:T // 2] = 0
    for b, n in enumerate(lens):
        for k in ("ppg", "vec"):
            d[k][b, n:] = 1e3 * torch.randn(T - n, d[k].shape[2], generator=g)
        d["pit"][b, n:] = 1e3 * torch.randn(T - n, generator=g)
        d["eps"][b, :, n:] = 1e3 * torch.randn(d["eps"].shape[1], T - n, generator=g)
        d["source"][b, :, n * HOP:] = 1e3 * torch.randn(1, (T - n) * HOP, generator=g)
    return {k: v.cuda() for k, v in d.items()}


def _run(m, d, lens):
    return m.inference_ragged(d["ppg"], d["vec"], d["pit"], d["spk"], lens, d["source"], eps=d["eps"])


@pytest.mark.parametrize("lens,T", [([1, 2, 37, 64, 65, 301, 400], 400), ([2520, 2510, 1000, 110], 2520)])
def test_each_item_equals_its_lone_call(model_tc, hp, lens, T):
    d = _ragged_inputs(hp, lens, T, 11 + T)
    w = _run(model_tc, d, lens)
    torch.cuda.synchronize()
    assert w.shape == (len(lens), 1, T * HOP)
    for b, n in enumerate(lens):
        lone = model_tc.inference(d["ppg"][b:b + 1, :n], d["vec"][b:b + 1, :n], d["pit"][b:b + 1, :n], d["spk"][b:b + 1],
                                  torch.tensor([n]), d["source"][b:b + 1, :, :n * HOP], eps=d["eps"][b:b + 1, :, :n])
        assert torch.isfinite(lone).all()
        diff = (w[b, 0, :n * HOP] != lone[0, 0]).nonzero()
        assert diff.numel() == 0, (n, diff.numel(), int(diff[0]), float((w[b, :, :n * HOP] - lone[0]).abs().max()))
        assert not w[b, :, n * HOP:].any(), n


def test_permuted_items_and_reruns_are_bitwise(model_tc, hp):
    lens, T = [1, 2, 37, 64, 65, 301, 400], 400
    d = _ragged_inputs(hp, lens, T, 5)
    w = _run(model_tc, d, lens)
    assert torch.equal(_run(model_tc, d, lens), w)
    perm = [4, 6, 0, 3, 1, 5, 2]
    dp = {k: v[perm] for k, v in d.items()}
    assert torch.equal(_run(model_tc, dp, [lens[i] for i in perm]), w[perm])


def test_rejections_name_the_cause(model_tc, hp, sd):
    lens, T = [5, 8], 8
    d = _ragged_inputs(hp, lens, T, 3)
    for bad, why in (([5, 0], "item 1 has 0 frames"), ([9, 8], "item 0 has 9 frames")):
        with pytest.raises(_lib.SvcbError, match=why):
            _run(model_tc, d, bad)
    for precision in (0, 1):
        m = _model(hp, sd, precision)
        with pytest.raises(_lib.SvcbError, match="precision 3"):
            _run(m, d, lens)


def test_padded_source_prefix_equals_lone_source(model_tc):
    g = torch.Generator().manual_seed(9)
    lens, T = [700, 1, 333, 52], 700
    f0 = torch.randint(100, 501, (len(lens), T), generator=g).float()
    f0[:, 100:180] = 0
    rand_ini = torch.rand(len(lens), 11, generator=g)
    noise = torch.randn(len(lens), T * HOP, 11, generator=g)
    for b, n in enumerate(lens):
        f0[b, n:] = 0
    src = model_tc.pitch2source(f0, rand_ini=rand_ini, noise=noise)
    for b, n in enumerate(lens):
        lone = model_tc.pitch2source(f0[b:b + 1, :n], rand_ini=rand_ini[b:b + 1], noise=noise[b:b + 1, :n * HOP])
        assert torch.equal(src[b, :, :n * HOP], lone[0]), n


def test_ragged_engine_equals_equal_length_engine(model_tc, hp):
    from whisper_vits_svc_b200 import hostio
    C = hp.vits.inter_channels

    class Quiet:   # the random draws silenced, so that both engines are deterministic
        def __init__(self, m):
            self.m = m

        def pitch2source(self, f0, **kw):
            B, T = f0.shape
            return self.m.pitch2source(f0, rand_ini=torch.zeros(B, 11), noise=torch.zeros(B, T * HOP, 11))

        def inference(self, ppg, vec, pit, spk, ppg_l, source, eps=None):
            return self.m.inference(ppg, vec, pit, spk, ppg_l, source, eps=torch.zeros(ppg.shape[0], C, ppg.shape[1]))

        def inference_ragged(self, ppg, vec, pit, spk, n_frames, source, eps=None):
            return self.m.inference_ragged(ppg, vec, pit, spk, n_frames, source, eps=torch.zeros(ppg.shape[0], C, ppg.shape[1]))

    g = torch.Generator().manual_seed(29)
    lengths = [300, 300, 2600, 300, 41, 1, 2511, 999]
    jobs = []
    for i, n in enumerate(lengths):
        pit = torch.randint(100, 500, (n,), generator=g).float()
        pit[n // 3:n // 2] = 0
        jobs.append((f"u{i}", torch.randn(hp.vits.spk_dim, generator=g) * 0.05, pit,
                     torch.randn(n, hp.vits.ppg_dim, generator=g), torch.randn(n, hp.vits.vec_dim, generator=g)))
    q = Quiet(model_tc)
    dense = hostio.BatchEngine(q, hp, "cuda", max_batch=4, window=8)
    ragged = hostio.BatchEngine(q, hp, "cuda", max_batch=4, window=8, ragged=True)
    want, got = dict(dense.run(iter(jobs))), dict(ragged.run(iter(jobs)))
    chunks, _ = hostio.BatchEngine.plan(lengths, HOP, 4)
    assert len(chunks) == 10 and ragged.batches == 3 and dense.batches == 7
    assert ragged.samples == dense.samples == sum(n * HOP - 1 for n in lengths)
    for i, n in enumerate(lengths):
        assert got[f"u{i}"].shape == (n * HOP - 1,)
        assert np.array_equal(got[f"u{i}"], want[f"u{i}"]), (n, float(np.abs(got[f"u{i}"] - want[f"u{i}"]).max()))
