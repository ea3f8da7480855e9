"""GPU parity of the whole hot path (through the C ABI) against
  (1) the committed golden fixtures produced by the UNMODIFIED reference, and
  (2) the oracle on fresh seeded inputs, stage by stage (debug taps),
plus size-independent properties at BASELINE-size inputs.
Tolerance: waveform max-abs <= 1e-3 (north_star gate, fp32 mode); measured ~1e-5."""
import os

import numpy as np
import pytest
import torch

from oracle import svc_oracle as O
from tests.util import GOLDEN, make_inputs, max_abs, rel_l2
from whisper_vits_svc_b200 import hparams, synth

pytestmark = pytest.mark.gpu
WAVE_TOL = 1e-3      # the stated gate
TIGHT = 2e-4         # what fp32 kernels are expected to meet


def _model(hp, sd, precision=0):
    from whisper_vits_svc_b200 import models
    assert torch.cuda.is_available()
    m = models.SynthesizerInfer(hp.data.filter_length // 2 + 1, hp.data.segment_size // hp.data.hop_length, hp,
                                precision=precision)
    m.load_state_dict(sd)
    m.eval()
    return m.to("cuda")


@pytest.fixture(scope="module")
def model(hp, sd):
    """precision 0: every conv on the fp32 CUDA-core kernels (tightest parity, 1e-6)."""
    return _model(hp, sd, 0)


@pytest.mark.parametrize("name", ["infer_b2_t48", "infer_b3_t70_ragged"])
def test_golden_full(model, hp, name):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    d = make_inputs(int(g["seed"]), int(g["B"]), int(g["T"]), hp, ragged=bool(g["ragged"]))
    src = model.pitch2source(d["pit"], rand_ini=d["rand_ini"], noise=d["noise"])
    assert max_abs(src, g["source"]) <= 1e-5
    # integer work is bit-exact on identical input: the GOLDEN source through source2wav == the reference's pcm
    assert np.array_equal(model.source2wav(torch.from_numpy(g["source"][:1])), g["pcm"])
    # (the device's own source differs from the golden one by <= 1e-5, i.e. at most one int16 step)
    assert np.abs(model.source2wav(src[:1]).astype(np.int32) - g["pcm"].astype(np.int32)).max() <= 1
    wave = model.inference(d["ppg"], d["vec"], d["pit"], d["spk"], d["ppg_l"], torch.from_numpy(g["source"]),
                           eps=d["eps"])
    err = max_abs(wave, g["wave"])
    print(f"{name}: wave max-abs err {err:.3e}")
    assert err <= WAVE_TOL
    assert err <= TIGHT


@pytest.mark.parametrize("name,over", [("gen80_b2_t36", dict(gen__upsample_input=80, data__sampling_rate=24000)),
                                       ("gen192_b1_t64", {})])
def test_golden_generator(hp, name, over):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    hpx = hparams.override(hp, **over)
    sdx = synth.svc_state_dict(hpx, 1234)
    m = _model(hpx, sdx)
    d = make_inputs(int(g["seed"]), int(g["B"]), int(g["T"]), hpx, gen_only=True)
    src = m.pitch2source(d["pit"], rand_ini=d["rand_ini"], noise=d["noise"])
    assert max_abs(src, g["source"]) <= 1e-5
    wave = m.generator(d["spk"], d["z"], torch.from_numpy(g["source"]))
    err = max_abs(wave, g["wave"])
    print(f"{name}: wave max-abs err {err:.3e}")
    assert err <= TIGHT


def test_stage_taps_vs_oracle(model, hp, sd):
    """Every tapped intermediate against the oracle's: localises a broken kernel in one run."""
    B, T = 2, 90
    d = make_inputs(5, B, T, hp, ragged=True)
    src = O.pitch2source(sd, hp, d["pit"], d["rand_ini"], d["noise"])
    st = {}
    wave_o = O.synthesizer_infer(sd, hp, d["ppg"], d["vec"], d["pit"], d["spk"], d["ppg_l"], src, d["eps"], stages=st)
    taps = {k: torch.zeros(tuple(v.shape), device="cuda") for k, v in st.items() if k != "z"}
    wave = model.inference(d["ppg"], d["vec"], d["pit"], d["spk"], d["ppg_l"], src, eps=d["eps"], taps=taps)
    torch.cuda.synchronize()
    valid = O.sequence_mask(d["ppg_l"], T)[:, None, :]
    report, bad = [], []
    for k, v in st.items():
        if k == "z":
            continue
        got = taps[k].cpu()
        if k.startswith("enc_"):  # padded frames of encoder internals are don't-care (masked later)
            got, v = got * valid, v * valid
        e = max_abs(got, v)
        scale = float(v.abs().max())
        report.append(f"{k:12s} max-abs {e:.3e} (peak {scale:.2f})")
        if not e <= 1e-4 * max(1.0, scale):
            bad.append(k)
    report.append(f"wave         max-abs {max_abs(wave, wave_o):.3e}")
    print("\n".join(report))
    assert not bad, f"stages out of tolerance: {bad}\n" + "\n".join(report)
    assert max_abs(wave, wave_o) <= TIGHT


def test_stage_entry_points(model, hp, sd):
    d = make_inputs(6, 2, 50, hp, ragged=True)
    z_p_o, mask = O.prior_encoder(sd, d["ppg"], d["ppg_l"], d["vec"], d["pit"], d["eps"])
    z_o = O.flow_reverse(sd, z_p_o, mask, d["spk"])
    z_p = model.prior(d["ppg"], d["vec"], d["pit"], d["ppg_l"], d["eps"])
    assert max_abs(z_p, z_p_o) <= 1e-4
    z = model.flow_reverse(z_p_o, d["ppg_l"], d["spk"])
    assert max_abs(z, z_o) <= 1e-4


def test_batch_independence_and_determinism(model, hp):
    """Items do not interact: item 0 of a batch == the same item alone; reruns are bit-identical."""
    d = make_inputs(7, 3, 64, hp, ragged=True)
    src = model.pitch2source(d["pit"], rand_ini=d["rand_ini"], noise=d["noise"])
    full = model.inference(d["ppg"], d["vec"], d["pit"], d["spk"], d["ppg_l"], src, eps=d["eps"])
    again = model.inference(d["ppg"], d["vec"], d["pit"], d["spk"], d["ppg_l"], src, eps=d["eps"])
    assert torch.equal(full, again)
    one = model.inference(d["ppg"][1:2], d["vec"][1:2], d["pit"][1:2], d["spk"][1:2], d["ppg_l"][1:2],
                          src[1:2], eps=d["eps"][1:2])
    assert max_abs(full[1:2], one) <= 1e-6


def test_full_size_properties(model, hp, sd):
    """BASELINE config #4 geometry (10 s items), B reduced to 4 to keep the oracle leg bounded:
    finite output, |wave| <= 1, chunk-locality (a frame far from an edit is unaffected), and one
    item checked against the oracle end to end."""
    B, T = 4, 1000
    d = make_inputs(8, B, T, hp)
    src = model.pitch2source(d["pit"], rand_ini=d["rand_ini"], noise=d["noise"])
    wave = model.inference(d["ppg"], d["vec"], d["pit"], d["spk"], d["ppg_l"], src, eps=d["eps"])
    assert wave.shape == (B, 1, T * 320)
    assert torch.isfinite(wave).all() and float(wave.abs().max()) <= 1.0
    # source: closed-form scan vs oracle on the full 320k-sample utterance
    src_o = O.pitch2source(sd, hp, d["pit"][:1], d["rand_ini"][:1], d["noise"][:1])
    assert max_abs(src[:1], src_o) <= 1e-5
    wave_o = O.synthesizer_infer(sd, hp, d["ppg"][:1], d["vec"][:1], d["pit"][:1], d["spk"][:1], d["ppg_l"][:1],
                                 src_o, d["eps"][:1])
    err = max_abs(wave[:1], wave_o)
    print(f"10 s item: wave max-abs err {err:.3e}, rel-l2 {rel_l2(wave[:1], wave_o):.3e}")
    assert err <= WAVE_TOL


def test_empty_and_bad_inputs(model, hp):
    from whisper_vits_svc_b200 import _lib, models
    d = make_inputs(9, 1, 8, hp)
    src = model.pitch2source(d["pit"], rand_ini=d["rand_ini"], noise=d["noise"])
    with pytest.raises(AssertionError):
        model.inference(d["ppg"], d["vec"], d["pit"], d["spk"], d["ppg_l"], src[:, :, :-1], eps=d["eps"])
    # all-unvoiced, length-1 lengths: still finite
    pit0 = torch.zeros_like(d["pit"])
    src0 = model.pitch2source(pit0, rand_ini=d["rand_ini"], noise=d["noise"])
    w = model.inference(d["ppg"], d["vec"], pit0, d["spk"], torch.tensor([1]), src0, eps=d["eps"])
    assert torch.isfinite(w).all()
    # precision is 0, 1 or 3: any other value fails model creation on first use instead of running a hybrid
    bad = models.SynthesizerInfer(513, 25, hp, precision=2).to("cuda")
    with pytest.raises(_lib.SvcbError, match="precision"):
        bad.pitch2source(d["pit"], rand_ini=d["rand_ini"], noise=d["noise"])


@pytest.mark.parametrize("precision,tol", [(3, WAVE_TOL), (1, 5e-2)])
def test_tensor_core_generator_modes(hp, sd, precision, tol):
    """AMP-block convs on the tensor cores (wgmma): bf16x3 split meets the 1e-3 waveform gate; plain bf16 reports
    its own error (CPU emulation predicts ~1e-2)."""
    from whisper_vits_svc_b200 import models
    m = models.SynthesizerInfer(513, 25, hp, precision=precision)
    m.load_state_dict(sd)
    m.to("cuda")
    d = make_inputs(21, 2, 60, hp, ragged=True)
    src = O.pitch2source(sd, hp, d["pit"], d["rand_ini"], d["noise"])
    st = {}
    wave_o = O.synthesizer_infer(sd, hp, d["ppg"], d["vec"], d["pit"], d["spk"], d["ppg_l"], src, d["eps"], stages=st)
    names = [f"gen_stage{i}" for i in range(5)]
    taps = {k: torch.zeros(tuple(st[k].shape), device="cuda") for k in names}
    wave = m.inference(d["ppg"], d["vec"], d["pit"], d["spk"], d["ppg_l"], src, eps=d["eps"], taps=taps)
    for k in names:
        print(f"precision={precision} {k}: max-abs {max_abs(taps[k], st[k]):.3e}")
    err = max_abs(wave, wave_o)
    print(f"precision={precision}: wave max-abs {err:.3e}")
    assert err <= tol


@pytest.fixture(scope="module")
def model_tc(hp, sd):
    from whisper_vits_svc_b200 import models
    m = models.SynthesizerInfer(513, 25, hp, precision=3)
    m.load_state_dict(sd)
    return m.to("cuda")


@pytest.mark.parametrize("name", ["infer_b2_t48", "infer_b3_t70_ragged"])
def test_golden_full_tensor_core_mode(model_tc, hp, name):
    """The default (bf16x3 tensor-core + fused narrow-stage) mode against the reference's golden
    waveforms: the 1e-3 gate with margin."""
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    d = make_inputs(int(g["seed"]), int(g["B"]), int(g["T"]), hp, ragged=bool(g["ragged"]))
    wave = model_tc.inference(d["ppg"], d["vec"], d["pit"], d["spk"], d["ppg_l"], torch.from_numpy(g["source"]),
                              eps=d["eps"])
    err = max_abs(wave, g["wave"])
    print(f"{name} (precision 3): wave max-abs err {err:.3e}")
    assert err <= 2e-4


def test_full_size_tensor_core_mode(model_tc, hp, sd):
    """10 s items (tiles of every stage interior + both sequence edges) in the default mode."""
    B, T = 2, 1000
    d = make_inputs(31, B, T, hp)
    src = O.pitch2source(sd, hp, d["pit"], d["rand_ini"], d["noise"])
    wave = model_tc.inference(d["ppg"], d["vec"], d["pit"], d["spk"], d["ppg_l"], src, eps=d["eps"])
    wave_o = O.synthesizer_infer(sd, hp, d["ppg"][:1], d["vec"][:1], d["pit"][:1], d["spk"][:1], d["ppg_l"][:1],
                                 src[:1], d["eps"][:1])
    err = max_abs(wave[:1], wave_o)
    print(f"10 s item (precision 3): wave max-abs err {err:.3e}")
    assert torch.isfinite(wave).all() and err <= 2e-4


def test_svc_infer_chunk_loop_vs_oracle(model_tc, hp, sd, tmp_path):
    """SURVEY.md §8a row a17 / config #1 plumbing: the host loop of svc_inference.py:77-134 (2500-frame
    chunks, +-10-frame overlap discarded, last sample dropped) through hostio.svc_infer, against the
    same loop restated over the oracle chunk by chunk, with the reference's random draws injected."""
    from whisper_vits_svc_b200 import hostio
    n = 2600  # -> chunks (0,2510) and (2490,2600)
    g = torch.Generator().manual_seed(17)
    ppg = torch.randn(n, hp.vits.ppg_dim, generator=g)
    vec = torch.randn(n + 3, hp.vits.vec_dim, generator=g)  # ragged feature lengths are trimmed to the min
    pit = torch.randint(100, 500, (n + 1,), generator=g).float()
    pit[700:900] = 0
    spk = torch.randn(hp.vits.spk_dim, generator=g) * 0.05
    rand_ini = torch.rand(1, 11, generator=g)
    noise = torch.randn(1, n * 320, 11, generator=g)
    plan = hostio.chunk_plan(n, 320)
    assert [(c[0], c[1]) for c in plan] == [(0, 2510), (2490, 2600)]
    eps = {i: torch.randn(1, hp.vits.inter_channels, ce - cs, generator=g) for i, (cs, ce, _, _) in enumerate(plan)}
    out = hostio.svc_infer(model_tc, spk, pit, ppg, vec, hp, "cuda", write_pit_wav=None, rand_ini=rand_ini,
                           noise=noise, eps_fn=lambda i, b, t: eps[i])
    assert out.dtype == np.float32 and out.shape == (n * 320 - 1,)
    src = O.pitch2source(sd, hp, pit[:n][None], rand_ini, noise)
    ref = []
    for i, (cs, ce, so, eo) in enumerate(plan):
        w = O.synthesizer_infer(sd, hp, ppg[None, cs:ce], vec[None, cs:ce], pit[None, cs:ce], spk[None],
                                torch.tensor([ce - cs]), src[:, :, cs * 320:ce * 320], eps[i])
        ref.append(w[0, 0].numpy()[so:eo])
    ref = np.concatenate(ref)
    err = float(np.abs(out - ref).max())
    print(f"svc_infer 26 s utterance, 2 chunks: max-abs {err:.3e}")
    assert err <= 2e-4


@pytest.mark.parametrize("B,T", [(1, 1), (2, 3), (1, 37)])
def test_tiny_lengths_tensor_core_mode(model_tc, hp, sd, B, T):
    """Sequences shorter than one tile in every stage (single CTA holds both sequence edges)."""
    d = make_inputs(40 + T, B, T, hp)
    src = O.pitch2source(sd, hp, d["pit"], d["rand_ini"], d["noise"])
    wave = model_tc.inference(d["ppg"], d["vec"], d["pit"], d["spk"], d["ppg_l"], src, eps=d["eps"])
    wave_o = O.synthesizer_infer(sd, hp, d["ppg"], d["vec"], d["pit"], d["spk"], d["ppg_l"], src, d["eps"])
    err = max_abs(wave, wave_o)
    print(f"B={B} T={T} (precision 3): wave max-abs err {err:.3e}")
    assert err <= 2e-4


@pytest.mark.parametrize("stage", [0, 2, 3, 4, 5])
def test_large_snake_alpha_tensor_core_mode(hp, sd, stage):
    """Trained BigVGAN checkpoints reach e^alpha ~ 10-50 (arguments of sin in the hundreds), far outside
    the synthetic N(0, 0.4^2) log-alphas: Snake's sin must stay accurate there (csrc/common.cuh:snake_sin
    reduces to [-pi, pi] before the hardware approximation; a bare `__sinf` loses |x| * 2^-24).
    One stage at a time gets log-alpha ~ U(2, 3.5) (e^alpha 7..33) in the FIRST activation of each of its
    three AMP blocks (stage 5 = activation_post) — every Snake large at once makes the generator chaotic
    (d/du of sin^2(e^a u)/e^b ~ e^a per activation, six deep), where not even two fp32 summation orders
    agree.  Covers snake_pack + amp_conv_tc (stages 0-2) and the narrow-stage kernels (3-4)."""
    from whisper_vits_svc_b200 import models
    g = torch.Generator().manual_seed(404 + stage)
    sd2 = dict(sd)
    keys = ([f"dec.resblocks.{3 * stage + j}.activations.0.act" for j in range(3)] if stage < 5 else ["dec.activation_post.act"])
    for k in keys:
        sd2[k + ".alpha"] = torch.rand(sd[k + ".alpha"].shape, generator=g) * 1.5 + 2.0
        sd2[k + ".beta"] = torch.rand(sd[k + ".beta"].shape, generator=g) * 1.0 + 0.5
    m = models.SynthesizerInfer(513, 25, hp, precision=3)
    m.load_state_dict(sd2)
    m.to("cuda")
    d = make_inputs(52, 2, 40, hp, ragged=True)
    src = O.pitch2source(sd2, hp, d["pit"], d["rand_ini"], d["noise"])
    st = {}
    wave_o = O.synthesizer_infer(sd2, hp, d["ppg"], d["vec"], d["pit"], d["spk"], d["ppg_l"], src, d["eps"], stages=st)
    names = [f"gen_stage{i}" for i in range(5)]
    taps = {k: torch.zeros(tuple(st[k].shape), device="cuda") for k in names}
    wave = m.inference(d["ppg"], d["vec"], d["pit"], d["spk"], d["ppg_l"], src, eps=d["eps"], taps=taps)
    errs = " ".join(f"{max_abs(taps[k], st[k]):.1e}" for k in names)
    err = max_abs(wave, wave_o)
    print(f"large alpha in stage {stage}: stage max-abs [{errs}], wave max-abs {err:.3e}")
    assert err <= WAVE_TOL


def test_batch_engine_matches_svc_infer(model_tc, hp):
    """hostio.BatchEngine (chunks of many utterances bucketed into equal-length device batches, copies on side
    streams) against the per-utterance host loop hostio.svc_infer: shapes / bookkeeping with the default
    random draws, then — with the draws silenced (zero source noise, eps = 0) so both paths are
    deterministic — the same waveform utterance by utterance."""
    from whisper_vits_svc_b200 import hostio
    g = torch.Generator().manual_seed(23)
    lens = [300, 300, 2600, 300, 41]
    jobs = []
    for i, n in enumerate(lens):
        ppg = torch.randn(n, hp.vits.ppg_dim, generator=g)
        vec = torch.randn(n, hp.vits.vec_dim, generator=g)
        pit = torch.randint(100, 500, (n,), generator=g).float()
        pit[n // 3:n // 2] = 0
        spk = torch.randn(hp.vits.spk_dim, generator=g) * 0.05
        jobs.append((f"u{i}", spk, pit, ppg, vec))
    eng = hostio.BatchEngine(model_tc, hp, "cuda", max_batch=2, window=4)
    got = dict(eng.run(iter(jobs)))
    assert set(got) == {f"u{i}" for i in range(len(lens))}
    for i, n in enumerate(lens):
        w = got[f"u{i}"]
        assert w.dtype == np.float32 and w.shape == (n * 320 - 1,) and np.isfinite(w).all()
    assert eng.samples == sum(n * 320 - 1 for n in lens) and eng.device_seconds > 0
    # the deterministic part (everything but the random draws) is identical: with eps = 0 and a noise-free
    # source the engine's batches equal the per-utterance host loop
    class Quiet:
        def __init__(self, m):
            self.m = m
        def pitch2source(self, f0, **kw):
            B, T = f0.shape
            return self.m.pitch2source(f0, rand_ini=torch.zeros(B, 11), noise=torch.zeros(B, T * 320, 11))
        def inference(self, ppg, vec, pit, spk, ppg_l, source, eps=None):
            return self.m.inference(ppg, vec, pit, spk, ppg_l, source, eps=torch.zeros(ppg.shape[0], hp.vits.inter_channels, ppg.shape[1]))
        def source2wav(self, s):
            return self.m.source2wav(s)
    q = Quiet(model_tc)
    eng2 = hostio.BatchEngine(q, hp, "cuda", max_batch=3, window=8)
    got2 = dict(eng2.run(iter(jobs)))
    for i, (key, spk, pit, ppg, vec) in enumerate(jobs):
        ref = hostio.svc_infer(q, spk, pit, ppg, vec, hp, "cuda", write_pit_wav=None)
        assert float(np.abs(got2[key] - ref).max()) <= 1e-6, key
