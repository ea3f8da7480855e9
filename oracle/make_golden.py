"""Generate tests/golden/*.npz by running the UNMODIFIED reference (TEST INFRASTRUCTURE).

Run in the build container only (needs /root/reference):  python oracle/make_golden.py
The reference's internal RNG calls are answered with the seeded tensors of tests/util.make_inputs
(in the order the reference draws them: torch.rand -> rand_ini, torch.randn_like -> noise, then
torch.randn_like -> eps), so the fixtures pin the reference's arithmetic, not its RNG stream.
Also asserts that oracle/svc_oracle.py reproduces every fixture.

`whisper_case` does the same for the PPG extractor: the reference's `Whisper` module is built from a
synthetic checkpoint through the loader surgery of whisper/inference.py:11-20 (decoder deleted, last
quarter of the encoder blocks deleted, strict=False load) and `model.encoder(mel)` is stored next to
the mel; oracle/whisper_oracle.py must reproduce it.
"""
import contextlib
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_import, svc_oracle as O  # noqa: E402
from tests.util import GOLDEN, make_inputs  # noqa: E402
from whisper_vits_svc_b200 import hparams, synth  # noqa: E402


class FeedRNG:
    """Answer torch.rand / torch.randn_like with queued tensors."""

    def __init__(self, rand_q, randn_q):
        self.rand_q, self.randn_q = list(rand_q), list(randn_q)

    def __enter__(self):
        self.o = (torch.rand, torch.randn_like)

        def rand(*shape, **kw):
            t = self.rand_q.pop(0)
            assert tuple(t.shape) == tuple(shape), (t.shape, shape)
            return t.clone()

        def randn_like(x, **kw):
            t = self.randn_q.pop(0)
            assert t.shape == x.shape, (t.shape, x.shape)
            return t.clone()

        torch.rand, torch.randn_like = rand, randn_like
        return self

    def __exit__(self, *a):
        torch.rand, torch.randn_like = self.o


def ref_model(hp, sd):
    Syn = ref_import.import_synthesizer()
    m = Syn(hp.data.filter_length // 2 + 1, hp.data.segment_size // hp.data.hop_length,
            ref_import.to_attr(hp)).eval()
    m.load_state_dict(sd)
    return m


def full_case(name, hp, seed, B, T, ragged):
    sd = synth.svc_state_dict(hp, 1234)
    m = ref_model(hp, sd)
    d = make_inputs(seed, B, T, hp, ragged=ragged)
    with torch.no_grad(), FeedRNG([d["rand_ini"]], [d["noise"], d["eps"]]):
        src = m.pitch2source(d["pit"])
        wave = m.inference(d["ppg"], d["vec"], d["pit"], d["spk"], d["ppg_l"], src)
    st = {}
    src_o = O.pitch2source(sd, hp, d["pit"], d["rand_ini"], d["noise"])
    wave_o = O.synthesizer_infer(sd, hp, d["ppg"], d["vec"], d["pit"], d["spk"], d["ppg_l"], src_o, d["eps"], stages=st)
    assert torch.equal(src, src_o) or (src - src_o).abs().max() < 1e-6, "oracle source != reference"
    err = (wave - wave_o).abs().max().item()
    assert err < 1e-5, f"oracle wave != reference ({err})"
    np.savez_compressed(os.path.join(GOLDEN, name + ".npz"), seed=seed, B=B, T=T, ragged=int(ragged),
                        source=src.numpy(), wave=wave.numpy(), z_p=st["z_p"].numpy(), z=st["z"].numpy(),
                        pcm=m.source2wav(src[:1]))
    print(name, "wave peak %.3f" % wave.abs().max().item(), "oracle-vs-reference max abs", err)


def gen_case(name, hp, seed, B, T):
    """BASELINE config #2 shape family: Generator.inference on a random latent."""
    sd = synth.svc_state_dict(hp, 1234)
    ref_import._ensure_path()
    from vits_decoder.generator import Generator
    g = Generator(ref_import.to_attr(hp))
    torch.nn.Module.eval(g)
    g.load_state_dict({k[4:]: v for k, v in sd.items() if k.startswith("dec.")})
    d = make_inputs(seed, B, T, hp, gen_only=True)
    with torch.no_grad(), FeedRNG([d["rand_ini"]], [d["noise"]]):
        src = g.pitch2source(d["pit"])
        wave = g.inference(d["spk"], d["z"], src)
    wave_o = O.generator(sd, hp, d["spk"], d["z"], O.pitch2source(sd, hp, d["pit"], d["rand_ini"], d["noise"]))
    err = (wave - wave_o).abs().max().item()
    assert err < 1e-5, err
    np.savez_compressed(os.path.join(GOLDEN, name + ".npz"), seed=seed, B=B, T=T, source=src.numpy(), wave=wave.numpy())
    print(name, "wave peak %.3f" % wave.abs().max().item(), "oracle-vs-reference max abs", err)


WHISPER_CASES = {
    # name: (dims overrides, checkpoint seed, B, n_frames, input seed)
    "whisper_d256_l8_b2_n200": (dict(n_audio_state=256, n_audio_head=4, n_audio_layer=8), 21, 2, 200, 31),
    "whisper_d512_l4_b1_n301": (dict(n_audio_state=512, n_audio_head=8, n_audio_layer=4), 22, 1, 301, 32),
}
_SMALL_TEXT = dict(n_vocab=64, n_text_ctx=8, n_text_state=64, n_text_head=1, n_text_layer=1)


def whisper_dims(over):
    return dict(synth.WHISPER_LARGE_V2_DIMS, **_SMALL_TEXT, **over)


def whisper_mel(seed, B, n):
    """SURVEY.md §8d config 3 input recipe: N(0,1) clipped to the log-mel range [-1, 1.5]."""
    return torch.randn(B, 80, n, generator=torch.Generator().manual_seed(seed)).clamp(-1, 1.5)


def ref_whisper(ck):
    """whisper/inference.py:11-20 verbatim in effect (the checkpoint is passed in, not read from disk)."""
    wm = ref_import.import_whisper_model()
    model = wm.Whisper(wm.ModelDimensions(**ck["dims"]))
    del model.decoder
    cut = len(model.encoder.blocks) // 4
    cut = -1 * cut
    del model.encoder.blocks[cut:]
    model.load_state_dict(ck["model_state_dict"], strict=False)
    model.eval()
    return model


def whisper_case(name):
    from oracle import whisper_oracle as WO
    over, ck_seed, B, n, in_seed = WHISPER_CASES[name]
    ck = synth.whisper_checkpoint(whisper_dims(over), seed=ck_seed)
    mel = whisper_mel(in_seed, B, n)
    with torch.no_grad():
        ppg = ref_whisper(ck).encoder(mel)
    ppg_o = WO.audio_encoder(ck, mel)
    err = (ppg - ppg_o).abs().max().item()
    assert err < 1e-5, f"whisper oracle != reference ({err})"
    np.savez_compressed(os.path.join(GOLDEN, name + ".npz"), mel=mel.numpy(), ppg=ppg.numpy())
    print(name, "ppg rms %.3f" % ppg.pow(2).mean().sqrt().item(), "oracle-vs-reference max abs", err)


HUBERT_CASES = {  # name: (checkpoint seed, B, n_samples, input seed)
    "hubert_soft_b2_n8000": (31, 2, 8000, 32),
    "hubert_soft_b1_n16123": (33, 1, 16123, 34),
}


def hubert_wav(seed, B, n):
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(n) / 16000.0
    tone = 0.3 * torch.sin(2 * math.pi * 220.0 * t)[None, :] * (1.0 + 0.5 * torch.sin(2 * math.pi * 3.0 * t))[None, :]
    return (tone + 0.1 * torch.randn(B, n, generator=g)).float().unsqueeze(1)


def ref_hubert(sd):
    """hubert/hubert_model.py:212-222 in effect (the state dict is passed in, not read from disk)."""
    hm = ref_import.import_hubert_model()
    model = hm.HubertSoft()
    model.load_state_dict(sd)
    return model.eval()


def hubert_case(name):
    from oracle import hubert_oracle as HO
    ck_seed, B, n, in_seed = HUBERT_CASES[name]
    sd = synth.hubert_checkpoint(ck_seed)
    wav = hubert_wav(in_seed, B, n)
    units = ref_hubert(sd).units(wav)
    units_o = HO.units(sd, wav)
    err = (units - units_o).abs().max().item()
    assert err < 2e-5, f"hubert oracle != reference ({err})"
    assert units.shape[1] == HO.frames(n)
    np.savez_compressed(os.path.join(GOLDEN, name + ".npz"), wav=wav.numpy(), units=units.numpy())
    print(name, tuple(units.shape), "units rms %.3f" % units.pow(2).mean().sqrt().item(), "oracle-vs-reference max abs", err)


# (dims override, B, n_frames) of the Whisper encoder pins; stored in reference_pins.npz as whisper<index>_*
WHISPER_PIN_CASES = [(dict(n_audio_state=256, n_audio_head=4, n_audio_layer=8), 2, 120),
                     (dict(n_audio_state=384, n_audio_head=6, n_audio_layer=4), 1, 77)]


to_float64 = O.to_float64


@contextlib.contextmanager
def float64_default():
    """The reference allocates some buffers with the default dtype (vits_decoder/nsf.py:292): float64 inside."""
    torch.set_default_dtype(torch.float64)
    try:
        yield
    finally:
        torch.set_default_dtype(torch.float32)


def reference_pins(hp):
    """tests/golden/reference_pins.npz: what the pins of tests/test_oracle_cpu.py compare the oracle with — the
    unmodified reference's outputs on the same seeded inputs, its state-dict keys / shapes and alias-filter taps.
    The SVC and Whisper outputs are computed in float64 (model.double(), float64 inputs): fp32 CPU results move by
    ~1e-6 with the host's thread count and instruction set, float64 ones by ~1e-15, so a stored float64 result pins
    the restatement as tightly on any host as a live comparison on one."""
    out = {}
    sd = synth.svc_state_dict(hp, 1234)
    d = to_float64(make_inputs(77, 2, 33, hp, ragged=True))
    with torch.no_grad(), float64_default():
        m = ref_model(hp, sd).double()
        with FeedRNG([d["rand_ini"]], [d["noise"], d["eps"]]):
            src = m.pitch2source(d["pit"])
            wave = m.inference(d["ppg"], d["vec"], d["pit"], d["spk"], d["ppg_l"], src)
    out["svc_source"], out["svc_wave"] = src.numpy(), wave.numpy()
    Syn = ref_import.import_synthesizer()
    ref_sd = Syn(513, 25, ref_import.to_attr(hp)).state_dict()
    out["sd_keys"] = np.array(sorted(ref_sd))
    out["sd_shapes"] = np.array([",".join(map(str, ref_sd[k].shape)) for k in sorted(ref_sd)])
    out["up_filter"] = ref_sd["dec.activation_post.upsample.filter"].numpy()
    for i, (over, B, n) in enumerate(WHISPER_PIN_CASES):
        ck = synth.whisper_checkpoint(whisper_dims(over), seed=5)
        model = ref_whisper(ck).double()   # built in fp32 exactly as whisper/inference.py loads it, then widened
        with torch.no_grad():
            out[f"whisper{i}_ppg"] = model.encoder(whisper_mel(6, B, n).double()).numpy()
        out[f"whisper{i}_kept_layers"] = np.array(len(model.encoder.blocks))
    with torch.no_grad():
        out["hubert_units"] = ref_hubert(synth.hubert_checkpoint(7)).units(hubert_wav(8, 1, 5003)).numpy()
    np.savez_compressed(os.path.join(GOLDEN, "reference_pins.npz"), **out)


if __name__ == "__main__":
    os.makedirs(GOLDEN, exist_ok=True)
    hp = hparams.load_hparams(os.path.join(ROOT, "configs", "base.yaml"))
    full_case("infer_b2_t48", hp, seed=11, B=2, T=48, ragged=False)
    full_case("infer_b3_t70_ragged", hp, seed=12, B=3, T=70, ragged=True)
    hp24 = hparams.override(hp, gen__upsample_input=80, data__sampling_rate=24000)
    gen_case("gen80_b2_t36", hp24, seed=13, B=2, T=36)
    gen_case("gen192_b1_t64", hp, seed=14, B=1, T=64)
    for name in WHISPER_CASES:
        whisper_case(name)
    for name in HUBERT_CASES:
        hubert_case(name)
    reference_pins(hp)
