"""Every generator, prior and flow stage of precisions 3, 1 and 0 against float64, one stage at a time.

Each stage's reference is the float64 oracle of that one stage fed the device's own previous tap (cast to
double) and the same source, so no error carries over from earlier stages: a stage computed in exact fp32
is held to fp32 accuracy even where the stages before it ran in plain bf16, and a failing gate names the
kernel that broke.  The gates and the form each stage computes in live in tests/test_gen_stages_cpu.py
(GATES, FORMS), which also shows that defects at sequence and tile edges exceed them.
"""
import math

import pytest
import torch

from oracle import svc_oracle as O
from tests.test_gen_stages_cpu import FORMS, GEN_STAGES, gate, gen_prev, gen_stage_ref, stage_error
from tests.util import make_inputs

pytestmark = pytest.mark.gpu

# ------------------------------------------------------------------------------------------- lengths
# Tile sizes of the narrow-stage fp32 kernels, as their sources define them:
#   amp_block_fused (csrc/amp_block_fused.cu, AbCfg): a CTA's buffer is W = 768 samples for C = 20 (384
#   threads x 2) and 1536 for C = 10 (512 x 3); it writes TOUT = W - 2H of them, H = ab_halo(K, dil) =
#   sum_d (6 + d(K-1)/2 + 6 + (K-1)/2).
#   ups_fused (csrc/ups_fused.cu): 256 input positions per CTA (stage 3 reads 80 T of them, stage 4 160 T).
#   post_fused (csrc/snake.cu): PF_OUT_RUNS = 254 runs of 8 samples = 2032 waveform samples per CTA.
AB_W = {20: 768, 10: 1536}
UPS_FUSED_TILE = 256
POST_FUSED_TILE = 254 * 8


def _ab_tout(C, K, dil):
    return AB_W[C] - 2 * sum(12 + d * (K - 1) // 2 + (K - 1) // 2 for d in dil)


def narrow_tiles(hp):
    """[(what, samples per frame, samples per CTA)] of every narrow-stage fp32 kernel in the base config."""
    rates = list(hp.gen.upsample_rates)
    n, tiles, ch, per = len(rates), [], hp.gen.upsample_initial_channel, 1
    for i, r in enumerate(rates):
        ch //= 2
        if i >= n - 2:   # the two narrow stages (C = 20, 10): ups_fused and amp_block_fused
            tiles.append((f"ups_fused stage {i}", per, UPS_FUSED_TILE))
            for K, dil in zip(hp.gen.resblock_kernel_sizes, hp.gen.resblock_dilation_sizes):
                tiles.append((f"amp_block_fused stage {i} K={K}", per * r, _ab_tout(ch, K, dil)))
        per *= r
    tiles.append(("post_fused", per, POST_FUSED_TILE))
    return tiles


def full_tile_lengths(hp):
    """The least T at which each kernel's last tile is exactly full: samples-per-frame * T % tile == 0.
    Base config: amp_block_fused 21 (C20 K3, C10 K11), 39 (C20 K7), 18 (C20 K11), 9 (C10 K3), 87 (C10 K7);
    ups_fused 16 (stage 3), 8 (stage 4); post_fused 127."""
    return sorted({tile // math.gcd(tile, per) for _, per, tile in narrow_tiles(hp)})


BASE_LENGTHS = [1, 3, 37, 64, 65, 129, 1000]
FULL_TILE_LENGTHS = [8, 9, 16, 18, 21, 39, 87, 127]   # full_tile_lengths(hp) of the base config
LENGTHS = sorted(set(BASE_LENGTHS) | set(FULL_TILE_LENGTHS))
LONG_CHUNK = 2520   # svc_inference's longest chunk: 2500 frames + 10 frames of overlap on each side


def test_lengths_cover_every_tile_edge(hp):
    """FULL_TILE_LENGTHS are the kernels' own full-tile lengths, and each narrow-stage kernel meets both a
    partial last tile and an exactly full one among the lengths."""
    assert FULL_TILE_LENGTHS == full_tile_lengths(hp)
    for what, per, tile in narrow_tiles(hp):
        assert any(per * T % tile == 0 for T in LENGTHS), what
        assert any(per * T % tile != 0 and per * T > tile for T in LENGTHS), what


# --------------------------------------------------------------------------------------------- models
@pytest.fixture(scope="module")
def models(hp, sd):
    from whisper_vits_svc_b200 import models as M
    cache = {}

    def get(precision):
        if precision not in cache:
            m = M.SynthesizerInfer(513, 25, hp, precision=precision)
            m.load_state_dict(sd)
            cache[precision] = m.to("cuda")
        return cache[precision]
    yield get
    cache.clear()


@pytest.fixture(scope="module")
def sd64(sd):
    return O.to_float64(sd)


def _gen_tap_shapes(hp, B, T):
    shapes = {"gen_pre": (B, hp.gen.upsample_initial_channel, T)}
    ch, L = hp.gen.upsample_initial_channel, T
    for i, r in enumerate(hp.gen.upsample_rates):
        ch, L = ch // 2, L * r
        shapes[f"gen_up{i}"] = shapes[f"gen_stage{i}"] = (B, ch, L)
    return shapes


def _check(rows, precision, T, what):
    """Print every stage's error; fail naming each stage over its gate with its form, T and the precision."""
    lines, bad = [], []
    for stage, form, e, scale, g in rows:
        line = f"precision {precision} T={T:5d} {stage:11s} {form:6s} max-abs {e:.3e} rel {e / scale:.2e} gate {g:.0e}"
        lines.append(line)
        if not e <= g * scale:
            bad.append(line)
    print("\n" + "\n".join(lines))
    assert not bad, f"{what}: stages over their gates:\n" + "\n".join(bad)


def _gen_inputs(m, hp, B, T, seed):
    d = make_inputs(seed, B, T, hp, gen_only=True)
    src = m.pitch2source(d["pit"], rand_ini=d["rand_ini"], noise=d["noise"])
    return d, src


GEN_CASES = [(p, T) for p in (3, 1) for T in LENGTHS] + [(3, LONG_CHUNK)] + [(0, T) for T in (1, 37, 129)]


@pytest.mark.parametrize("precision,T", GEN_CASES)
def test_generator_stages_vs_float64(models, hp, sd64, precision, T):
    """gen_pre, gen_up0..4, gen_stage0..4 and the post_fused tail, B = 2 (the 2520-frame chunk: B = 1)."""
    m = models(precision)
    B = 1 if T == LONG_CHUNK else 2
    d, src = _gen_inputs(m, hp, B, T, seed=1000 + T)
    taps = {k: torch.zeros(s, device="cuda") for k, s in _gen_tap_shapes(hp, B, T).items()}
    wave = m.generator(d["spk"], d["z"], src, taps=taps)
    torch.cuda.synchronize()
    dev = {k: v.cpu().double() for k, v in taps.items()}
    dev["wave"] = wave.cpu().double()
    src64, spk64, z64 = src.cpu().double(), d["spk"].double(), d["z"].double()
    rows = []
    with torch.no_grad():
        for stage in GEN_STAGES:
            p = gen_prev(stage)
            ref = gen_stage_ref(sd64, hp, stage, z64 if p is None else dev[p], src64, spk=spk64)
            e, scale = stage_error(dev[stage], ref)
            rows.append((stage, FORMS[precision][stage], e, scale, gate(precision, stage)))
    _check(rows, precision, T, f"generator, precision {precision}, B={B}, T={T}")


@pytest.mark.parametrize("precision", [3, 1, 0])
@pytest.mark.parametrize("T", [1, 37])
def test_fallback_tail_vs_float64(models, hp, sd64, precision, T):
    """The tail the generator runs when the waveform is not 16-byte aligned (snake_alias, then conv1d + tanh):
    the wave pointer is one float into a larger buffer, whose other floats must stay untouched."""
    m = models(precision)
    m._ensure()
    B = 2
    d, src = _gen_inputs(m, hp, B, T, seed=3000 + T)
    L = T * m.hop
    sentinel = 7.0
    buf = torch.full((B * L + 8,), sentinel, device="cuda")
    wave = buf[1:1 + B * L]
    assert wave.data_ptr() % 16 == 4
    stage4 = torch.zeros(_gen_tap_shapes(hp, B, T)["gen_stage4"], device="cuda")
    spk, z, src = (t.to("cuda", torch.float32).contiguous() for t in (d["spk"], d["z"], src))
    ws = m._workspace(B, T)
    m._handle.call("generator", spk.data_ptr(), z.data_ptr(), src.data_ptr(), wave.data_ptr(), B, T,
                   ws.data_ptr(), ws.numel(), m._taps({"gen_stage4": stage4}))
    torch.cuda.synchronize()
    assert float(buf[0]) == sentinel and bool((buf[1 + B * L:] == sentinel).all()), "the tail wrote outside the waveform"
    with torch.no_grad():
        ref = O.gen_tail(sd64, stage4.cpu().double())
    e, scale = stage_error(wave.view(B, 1, L).cpu(), ref)
    _check([("wave", "fp32", e, scale, gate(precision, "wave"))], precision, T, "fallback tail (unaligned wave)")


@pytest.mark.parametrize("T", [65, 129, 1000])
def test_prior_and_flow_stages_vs_float64(models, hp, sd64, T):
    """Precision 3's prior encoder (front, six layers, proj + reparam) and reverse flow, ragged lengths
    (1, 64, 65, T), each stage fed the device's previous tap; padded frames are don't-care."""
    m = models(3)
    d = make_inputs(2000 + T, 4, T, hp)
    d["ppg_l"] = torch.tensor([1, 64, 65, T], dtype=torch.long)
    H, C = hp.vits.hidden_channels, hp.vits.inter_channels
    taps = {k: torch.zeros(4, H, T, device="cuda") for k in ["enc_front"] + [f"enc_layer{i}" for i in range(6)]}
    taps["z_p"] = torch.zeros(4, C, T, device="cuda")
    z_p = m.prior(d["ppg"], d["vec"], d["pit"], d["ppg_l"], d["eps"], taps=taps)
    ftaps = {f"flow{i}": torch.zeros(4, C, T, device="cuda") for i in range(4)}
    m.flow_reverse(z_p, d["ppg_l"], d["spk"], taps=ftaps)
    torch.cuda.synchronize()
    dev = {k: v.cpu().double() for k, v in {**taps, **ftaps}.items()}
    z_p = z_p.cpu().double()
    d64 = O.to_float64(d)
    rows = []
    with torch.no_grad():
        # pit stays fp32: the coarse pitch bin is an fp32 computation on the device and in the reference
        x, mask = O.prior_front(sd64, d64["ppg"], d["ppg_l"], d64["vec"], d["pit"])
        refs = {"enc_front": x}
        for i in range(6):
            prev = dev["enc_front"] if i == 0 else dev[f"enc_layer{i - 1}"]
            refs[f"enc_layer{i}"] = O.encoder_layer(sd64, i, prev * mask, mask)
        refs["z_p"] = O.prior_proj(sd64, dev["enc_layer5"], mask, d64["eps"])
        for i in reversed(range(4)):
            prev = z_p if i == 3 else dev[f"flow{i + 1}"]
            refs[f"flow{i}"] = O.coupling_reverse(sd64, f"flow.flows.{2 * i}", torch.flip(prev, [1]), mask, d64["spk"])
    for k, ref in refs.items():
        e, scale = stage_error(dev[k], ref, valid=mask)
        rows.append((k, FORMS[3][k], e, scale, gate(3, k)))
    _check(rows, 3, T, "prior and flow, ragged lengths (1, 64, 65, T)")
