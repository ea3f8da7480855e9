"""The per-stage float64 references the generator, prior and flow stages are gated against
(tests/test_gen_stages_gpu.py), and proof that those gates can see edge-sized defects.

A stage is gated in isolation: its reference is the float64 oracle function of that one stage, fed the
device's own previous tap, so no error carries over from earlier stages and each gate can sit close to what
the stage's kernels compute.  The gate is `GATES[form] * max(1, peak)`, where `form` is how the stage's
kernels do their arithmetic (FORMS below) and `peak` is the stage reference's max |value|.

This file holds the one table of gates both test files use, checks that the split oracle is the oracle
(bitwise), derives the plain-bf16 gate from a CPU emulation of bf16 operand rounding, and checks that each
planted defect at a sequence or tile edge moves its stage by more than 3x that stage's gate.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import svc_oracle as O
from tests.util import make_inputs

# ----------------------------------------------------------------------------------------- the gates
# Relative to max(1, peak) of the stage reference.
GATES = {
    # Exact fp32 kernels (CUDA-core convolutions, ups_finalize, ups_fused, amp_block_fused, post_fused, the
    # snake_alias + conv1d tail).  The fp32 oracle against the same oracle in float64, one stage fed its exact
    # input, differs by <= 6e-7 relative at T = 37 (test_fp32_floor_below_gate); measured on an H100 (700 W)
    # the fp32 kernels reach 1.4e-6 over every length.
    "fp32": 1e-5,
    # bf16x3 tensor-core kernels (conv_tc, amp_conv_tc, the S2D links, noise_tc, the comb upsampler,
    # rel_attn_tc): each fp32 operand is split into bf16 hi + lo, the three significant products are summed
    # in fp32, so an operand keeps ~16 of its 24 bits and a product is good to ~2^-16 ~ 1.5e-5 relative.
    # Measured on an H100 (700 W) over every length: generator stages <= 7.6e-6, flow <= 1.4e-6, encoder
    # layers <= 1.7e-5, enc_front (pre + hub, 6400-term sums) 2.0e-5 relative: the gate is 3x that.
    "bf16x3": 6e-5,
    # Plain bf16 tensor-core kernels (precision 1's conv_pre and stages 0-2): operands rounded to bf16 (8
    # significant bits, 2^-9 relative), fp32 accumulation.  test_bf16_gate_covers_emulation replays the
    # rounding on the CPU: the worst emulated stage is 2.6e-3 relative at T = 37; measured on an H100 (700 W)
    # the worst stage is 3.2e-3 over every length.  The gate sits 3x above both.
    "bf16": 1e-2,
}

GEN_STAGES = ["gen_pre"] + [f"{k}{i}" for i in range(5) for k in ("gen_up", "gen_stage")] + ["wave"]
PRIOR_STAGES = ["enc_front"] + [f"enc_layer{i}" for i in range(6)] + ["z_p"] + [f"flow{i}" for i in range(4)]

# How each stage computes at each precision (csrc/api.cu:resolve for the base config).
_F, _X, _B = "fp32", "bf16x3", "bf16"
FORMS = {
    # conv_pre + Mish: conv_tc; stage 0: conv_tc phases + ups_finalize + noise_tc, amp_conv_tc; stages 1-2: the
    # comb upsampler; stage 1: amp_conv_tc; stages 2-4: S2D links; stages 3-4: ups_fused; tail: post_fused
    3: dict(gen_pre=_X, gen_up0=_X, gen_stage0=_X, gen_up1=_X, gen_stage1=_X, gen_up2=_X, gen_stage2=_X,
            gen_up3=_F, gen_stage3=_X, gen_up4=_F, gen_stage4=_X, wave=_F,
            # pre/hub/qkv/o/ffn/proj and the flow convolutions on conv_tc, attention on rel_attn_tc
            enc_front=_X, z_p=_X, **{f"enc_layer{i}": _X for i in range(6)}, **{f"flow{i}": _X for i in range(4)}),
    # as precision 3 with plain bf16 operands in conv_pre and stages 0-2; stages 3-4: ups_fused, amp_block_fused
    1: dict(gen_pre=_B, gen_up0=_B, gen_stage0=_B, gen_up1=_B, gen_stage1=_B, gen_up2=_B, gen_stage2=_B,
            gen_up3=_F, gen_stage3=_F, gen_up4=_F, gen_stage4=_F, wave=_F),
    # every convolution on the fp32 CUDA-core kernels: conv1d phases + ups_finalize, noise by conv1d
    0: {k: _F for k in GEN_STAGES},
}


def gate(precision: int, stage: str) -> float:
    return GATES[FORMS[precision][stage]]


# --------------------------------------------------------------------------------- stage references
def gen_stage_ref(sd, hp, stage, prev, source, spk=None):
    """The oracle of one generator stage on the stage's input `prev` (z for gen_pre, else the previous tap)."""
    if stage == "gen_pre":
        return O.gen_pre(sd, spk, prev)
    if stage == "wave":
        return O.gen_tail(sd, prev)
    i = int(stage[-1])
    if stage.startswith("gen_up"):
        return O.gen_upsample(sd, hp, i, prev, source)
    return O.gen_amp_stage(sd, hp, i, prev)


def gen_prev(stage):
    """The tap a generator stage reads (None: the generator's input z)."""
    if stage == "gen_pre":
        return None
    if stage == "wave":
        return "gen_stage4"
    i = int(stage[-1])
    if stage.startswith("gen_up"):
        return "gen_pre" if i == 0 else f"gen_stage{i - 1}"
    return f"gen_up{i}"


def stage_error(got, ref, valid=None):
    """(max |got - ref| in float64, max(1, peak of ref)), over the valid frames only when a mask is given."""
    got, ref = torch.as_tensor(got).double().cpu(), torch.as_tensor(ref).double().cpu()
    if valid is not None:
        got, ref = got * valid, ref * valid
    return float((got - ref).abs().max()), max(1.0, float(ref.abs().max()))


# ------------------------------------------------------------------------------------ shared fixtures
T_CPU = 37


@pytest.fixture(scope="module")
def sd64(sd):
    return O.to_float64(sd)


@pytest.fixture(scope="module")
def gen_case(hp, sd):
    """B = 2, T = 37: generator inputs, the fp32 source and every float64 stage of the chained oracle."""
    d = make_inputs(11, 2, T_CPU, hp, gen_only=True)
    src = O.pitch2source(sd, hp, d["pit"], d["rand_ini"], d["noise"])
    return d, src


@pytest.fixture(scope="module")
def gen64(hp, sd64, gen_case):
    d, src = gen_case
    st = {}
    with torch.no_grad():
        st["wave"] = O.generator(sd64, hp, d["spk"].double(), d["z"].double(), src.double(), stages=st)
    return st


# ------------------------------------------------------------------------ (a) the split is the oracle
def test_split_generator_is_the_oracle(hp, sd, gen_case):
    """Chaining gen_pre, gen_upsample, gen_amp_stage and gen_tail reproduces O.generator bitwise in fp32,
    with each stage fed the previous stage's output exactly as the GPU test feeds it."""
    d, src = gen_case
    st = {}
    with torch.no_grad():
        wave = O.generator(sd, hp, d["spk"], d["z"], src, stages=st)
        st["wave"] = wave
        for stage in GEN_STAGES:
            p = gen_prev(stage)
            got = gen_stage_ref(sd, hp, stage, d["z"] if p is None else st[p], src, spk=d["spk"])
            assert torch.equal(got, st[stage]), stage


def test_split_prior_and_flow_are_the_oracle(hp, sd):
    """prior_front, encoder_layer, prior_proj and coupling_reverse, chained tap to tap as the GPU test does,
    reproduce O.synthesizer_infer's taps and waveform bitwise in fp32 (ragged lengths)."""
    d = make_inputs(12, 3, 29, hp, ragged=True)
    src = O.pitch2source(sd, hp, d["pit"], d["rand_ini"], d["noise"])
    st = {}
    with torch.no_grad():
        wave = O.synthesizer_infer(sd, hp, d["ppg"], d["vec"], d["pit"], d["spk"], d["ppg_l"], src, d["eps"], stages=st)
        x, mask = O.prior_front(sd, d["ppg"], d["ppg_l"], d["vec"], d["pit"])
        assert torch.equal(x, st["enc_front"])
        x = x * mask
        for i in range(6):
            x = O.encoder_layer(sd, i, x, mask)
            assert torch.equal(x, st[f"enc_layer{i}"]), i
        z_p = O.prior_proj(sd, x, mask, d["eps"])
        assert torch.equal(z_p, st["z_p"])
        y = z_p
        for i in reversed(range(4)):
            y = O.coupling_reverse(sd, f"flow.flows.{2 * i}", torch.flip(y, [1]), mask, d["spk"])
            assert torch.equal(y, st[f"flow{i}"]), i
        assert torch.equal(O.generator(sd, hp, d["spk"], y * mask, src), wave)


# ------------------------------------------------------------------------ the gates against the floors
@pytest.mark.slow
def test_fp32_floor_below_gate(hp, sd, gen_case, gen64):
    """Each stage of the fp32 oracle fed the exact (float64) stage input, against float64: the fp32 floor.
    The fp32 gate is at least 3x above it."""
    d, src = gen_case
    rows = []
    with torch.no_grad():
        for stage in GEN_STAGES:
            p = gen_prev(stage)
            x = d["z"] if p is None else gen64[p].float()
            got = gen_stage_ref(sd, hp, stage, x, src, spk=d["spk"])
            e, scale = stage_error(got, gen64[stage])
            rows.append((stage, e / scale))
    print("\n".join(f"fp32 floor {s:11s} {r:.2e}" for s, r in rows))
    worst = max(r for _, r in rows)
    assert 3 * worst <= GATES["fp32"], rows


class _Bf16Convs:
    """torch.nn.functional for the oracle with the operands of every dense convolution rounded to bf16 (the
    depthwise alias filters, which the kernels apply in fp32, and the biases stay exact)."""

    @staticmethod
    def _r(t):
        return t.to(torch.bfloat16).to(t.dtype)

    def __getattr__(self, name):
        return getattr(F, name)

    def conv1d(self, x, w, b=None, stride=1, padding=0, dilation=1, groups=1):
        if groups == 1:
            x, w = self._r(x), self._r(w)
        return F.conv1d(x, w, b, stride=stride, padding=padding, dilation=dilation, groups=groups)

    def conv_transpose1d(self, x, w, b=None, stride=1, padding=0, groups=1):
        if groups == 1:
            x, w = self._r(x), self._r(w)
        return F.conv_transpose1d(x, w, b, stride=stride, padding=padding, groups=groups)


@pytest.mark.slow
def test_bf16_gate_covers_emulation(hp, sd64, gen_case, gen64, monkeypatch):
    """Precision 1's bf16 stages replayed in float64 with bf16-rounded conv operands, each fed its exact input:
    the plain-bf16 gate is at least 3x above the worst stage."""
    d, src = gen_case
    src = src.double()
    monkeypatch.setattr(O, "F", _Bf16Convs())
    rows = []
    with torch.no_grad():
        for stage in [s for s in GEN_STAGES if FORMS[1][s] == "bf16"]:
            p = gen_prev(stage)
            x = d["z"].double() if p is None else gen64[p]
            got = gen_stage_ref(sd64, hp, stage, x, src, spk=d["spk"].double())
            e, scale = stage_error(got, gen64[stage])
            rows.append((stage, e / scale))
    print("\n".join(f"bf16 emulation {s:11s} {r:.2e}" for s, r in rows))
    worst = max(r for _, r in rows)
    assert worst > 1e-4, "the emulation rounded nothing"
    assert 3 * worst <= GATES["bf16"], rows


# ---------------------------------------------------------------------- (b) planted defects at the edges
def _snake_alias_zero_right(sd, p, x):
    """O.snake_alias with zero padding instead of replicate padding at the sequence's end (both its pads)."""
    c = x.shape[1]
    fu, fd = sd[p + ".upsample.filter"], sd[p + ".downsample.lowpass.filter"]
    ku, kd, ratio = fu.shape[-1], fd.shape[-1], 2
    pad = ku // ratio - 1
    pl, pr = pad * ratio + (ku - ratio) // 2, pad * ratio + (ku - ratio + 1) // 2
    u = F.pad(F.pad(x, (pad, 0), mode="replicate"), (0, pad))
    u = ratio * F.conv_transpose1d(u, fu.expand(c, -1, -1), stride=ratio, groups=c)[..., pl:-pr]
    alpha = torch.exp(sd[p + ".act.alpha"])[None, :, None]
    beta = torch.exp(sd[p + ".act.beta"])[None, :, None]
    u = u + (1.0 / (beta + 1e-9)) * torch.sin(u * alpha) ** 2
    u = F.pad(F.pad(u, (kd // 2 - (1 - kd % 2), 0), mode="replicate"), (0, kd // 2))
    return F.conv1d(u, fd.expand(c, -1, -1), stride=ratio, groups=c)


def _defect_noise0_last_window(sd, hp, st, src):
    """noise_convs[0] drops the source window of the last stage-0 sample."""
    s = int(np.prod(list(hp.gen.upsample_rates)[1:]))
    b = sd["dec.noise_convs.0.bias"]
    nc = F.conv1d(src, sd["dec.noise_convs.0.weight"], b, stride=s, padding=s // 2)
    bad = st["gen_up0"].clone()
    bad[..., -1] -= nc[..., -1] - b
    return "gen_up0", bad


def _defect_rate2_last_phase(sd, hp, st, src):
    """ups[3] (rate 2) leaves its last output phase at the sequence end unwritten (zero)."""
    i = 3
    assert list(hp.gen.upsample_rates)[i] == 2
    u, k = 2, list(hp.gen.upsample_kernel_sizes)[i]
    ct = F.conv_transpose1d(st["gen_stage2"], O.fold_weight_norm(sd, f"dec.ups.{i}"), sd[f"dec.ups.{i}.bias"],
                            stride=u, padding=(k - u) // 2)
    bad = st["gen_up3"].clone()
    bad[..., -1] -= ct[..., -1]
    return "gen_up3", bad


def _defect_snake_zero_pad(sd, hp, st, src, monkeypatch):
    """The first SnakeAlias of one AMP unit of stage 4 zero-pads the sequence end instead of replicating it."""
    target = "dec.resblocks.12.activations.0"
    plain = O.snake_alias
    monkeypatch.setattr(O, "snake_alias", lambda sd_, p, x: _snake_alias_zero_right(sd_, p, x) if p == target else plain(sd_, p, x))
    try:
        bad = O.gen_amp_stage(sd, hp, 4, st["gen_up4"])
    finally:
        monkeypatch.setattr(O, "snake_alias", plain)
    return "gen_stage4", bad


def _defect_conv_post_shift(sd, hp, st, src):
    """conv_post pads 2 | 4 instead of 3 | 3."""
    x = O.snake_alias(sd, "dec.activation_post", st["gen_stage4"])
    return "wave", torch.tanh(F.conv1d(F.pad(x, (2, 4)), sd["dec.conv_post.weight"]))


GEN_DEFECTS = [_defect_noise0_last_window, _defect_rate2_last_phase, _defect_snake_zero_pad, _defect_conv_post_shift]


@pytest.mark.slow
@pytest.mark.parametrize("defect", GEN_DEFECTS, ids=lambda f: f.__name__[len("_defect_"):])
def test_generator_defect_exceeds_gates(hp, sd64, gen_case, gen64, defect, monkeypatch):
    """Each defect moves its stage by more than 3x the stage's gate at every precision."""
    d, src = gen_case
    kw = {"monkeypatch": monkeypatch} if defect is _defect_snake_zero_pad else {}
    with torch.no_grad():
        stage, bad = defect(sd64, hp, gen64, src.double(), **kw)
    e, scale = stage_error(bad, gen64[stage])
    for p in FORMS:
        g = gate(p, stage)
        print(f"{defect.__name__}: {stage} moves {e / scale:.2e} relative; precision {p} gate {g:.0e} ({FORMS[p][stage]})")
        assert e > 3 * g * scale, (stage, p, e, g * scale)


@pytest.mark.slow
def test_rel_position_defect_exceeds_gate(hp, sd64):
    """Attention layer 2 without its relative-position terms (both tables zero) moves enc_layer2 by more than 3x
    its gate, over the valid frames of a ragged batch."""
    d = O.to_float64(make_inputs(13, 2, T_CPU, hp, ragged=True))
    i = 2
    with torch.no_grad():
        x, mask = O.prior_front(sd64, d["ppg"], d["ppg_l"], d["vec"], d["pit"].float())
        x = x * mask
        for j in range(i):
            x = O.encoder_layer(sd64, j, x, mask)
        good = O.encoder_layer(sd64, i, x, mask)
        sd2 = dict(sd64)
        for t in ("emb_rel_k", "emb_rel_v"):
            sd2[f"enc_p.enc.attn_layers.{i}.{t}"] = torch.zeros_like(sd64[f"enc_p.enc.attn_layers.{i}.{t}"])
        bad = O.encoder_layer(sd2, i, x, mask)
    e, scale = stage_error(bad, good, valid=mask)
    g = gate(3, f"enc_layer{i}")
    print(f"rel-position drop: enc_layer{i} moves {e / scale:.2e} relative; precision 3 gate {g:.0e}")
    assert e > 3 * g * scale


def test_gate_table_is_complete():
    assert set(FORMS[3]) == set(GEN_STAGES) | set(PRIOR_STAGES)
    assert set(FORMS[1]) == set(FORMS[0]) == set(GEN_STAGES)
    assert all(f in GATES for p in FORMS for f in FORMS[p].values())
    assert GATES["fp32"] < GATES["bf16x3"] < GATES["bf16"] and all(0 < g < 1 for g in GATES.values())
