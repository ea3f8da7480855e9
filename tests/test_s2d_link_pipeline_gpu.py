"""The space-to-depth AMP link (csrc/amp_s2d.cu) where each persistent CTA walks many tiles: the next tile's A
panel loads while the current tile's epilogue still reads the accumulator staged over the weight ring, and
the next tile's weights wait for that epilogue.  Covers every space-to-depth factor, the 3- and 15-tap
extremes, links with and without the Snake output, and (through the generator) accumulating / dividing
links and ragged batches whose consecutive tiles on one CTA belong to different items.  Results are checked
against the oracle at the gates of test_ops_gpu.py and must be bitwise identical across reruns."""
import pytest
import torch
import torch.nn.functional as F

from oracle import svc_oracle as O
from tests.util import make_inputs, max_abs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    from whisper_vits_svc_b200 import ops as o
    return o


# C (r = 160 / C), K, dilation, Snake output
LINKS = [(40, 3, 1, True), (20, 3, 1, True), (10, 3, 1, True), (40, 11, 5, True), (20, 7, 3, False)]


@pytest.mark.parametrize("C,K,dil,snake", LINKS)
def test_link_many_tiles_per_cta(ops, sd, C, K, dil, snake):
    r = 160 // C
    S = 128 - 2 * (1 if r >= 8 else 2)                       # useful rows per tile
    B = 2
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    tpi = 2 * n_sm + 3                                       # tiles per item: > 4 tiles per CTA, uneven last wave
    L = r * S * tpi - 8 * r                                  # last tile of each item partly empty; L % 8 == 0
    g = torch.Generator().manual_seed(C * 7 + K + dil)
    x = torch.randn(B, C, L, generator=g) * 1.5
    w = torch.randn(C, C, K, generator=g) / (C * K) ** 0.5
    b = torch.randn(C, generator=g) * 0.1
    res = torch.randn(B, C, L, generator=g)
    filt = {"upsample.filter": sd["dec.activation_post.upsample.filter"],
            "downsample.lowpass.filter": sd["dec.activation_post.downsample.lowpass.filter"]}
    fa = {"a.act.alpha": torch.randn(C, generator=g) * 0.4, "a.act.beta": torch.randn(C, generator=g) * 0.4,
          **{"a." + k: v for k, v in filt.items()}}
    fb = {"b.act.alpha": torch.randn(C, generator=g) * 0.4, "b.act.beta": torch.randn(C, generator=g) * 0.4,
          **{"b." + k: v for k, v in filt.items()}}

    def run():
        return ops.amp_s2d_link(x.cuda(), fa["a.act.alpha"], fa["a.act.beta"], filt["upsample.filter"],
                                filt["downsample.lowpass.filter"], w, b.cuda(), dilation=dil, res=res.cuda(),
                                alpha_out=fb["b.act.alpha"] if snake else None, beta_out=fb["b.act.beta"] if snake else None)

    got, got_act = run()
    again, again_act = run()
    torch.cuda.synchronize()
    assert torch.equal(got, again)
    assert (got_act is None) == (not snake)
    if snake:
        assert torch.equal(got_act, again_act)
    ref = F.conv1d(O.snake_alias(fa, "a", x), w, b, dilation=dil, padding=dil * (K - 1) // 2) + res
    e1 = max_abs(got, ref)
    e2 = max_abs(got_act, O.snake_alias(fb, "b", ref)) if snake else 0.0
    print(f"C={C} K={K} d={dil} {B * tpi} tiles on {n_sm} SMs: conv max-abs {e1:.3e}, next-snake image max-abs {e2:.3e}")
    assert e1 <= 2e-4 and e2 <= 3e-4


def test_generator_stages_ragged_many_tiles(hp, sd):
    """Stages 2-4 in the default precision: their last links accumulate the AMP blocks' mean into the stage
    output and divide by the block count.  A ragged batch of 3 x 7 s items gives every CTA 2-3 tiles of
    stage 4, each from a different item."""
    from whisper_vits_svc_b200 import models
    m = models.SynthesizerInfer(513, 25, hp, precision=3)
    m.load_state_dict(sd)
    m.to("cuda")
    B, T = 3, 700
    d = make_inputs(61, B, T, hp, ragged=True)
    assert int(d["ppg_l"].min()) < T
    src = O.pitch2source(sd, hp, d["pit"], d["rand_ini"], d["noise"])
    st = {}
    wave_o = O.synthesizer_infer(sd, hp, d["ppg"], d["vec"], d["pit"], d["spk"], d["ppg_l"], src, d["eps"], stages=st)
    names = [f"gen_stage{i}" for i in (2, 3, 4)]
    runs = []
    for _ in range(2):
        taps = {k: torch.zeros(tuple(st[k].shape), device="cuda") for k in names}
        wave = m.inference(d["ppg"], d["vec"], d["pit"], d["spk"], d["ppg_l"], src, eps=d["eps"], taps=taps)
        torch.cuda.synchronize()
        runs.append((wave, taps))
    (wave, taps), (wave2, taps2) = runs
    assert torch.equal(wave, wave2) and all(torch.equal(taps[k], taps2[k]) for k in names)
    errs = {k: max_abs(taps[k], st[k]) for k in names}
    err = max_abs(wave, wave_o)
    print(f"stage max-abs {errs}, wave max-abs {err:.3e}")
    assert all(e <= 2e-4 * max(1.0, float(st[k].abs().max())) for k, e in errs.items())
    assert err <= 2e-4
