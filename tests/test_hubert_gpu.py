"""GPU parity of the HuBERT-Soft content encoder (SURVEY.md §8f-2) through the C ABI (svcb_hubert_*).

The reference runs this model in fp16 on GPU (hubert/inference.py:20-21, 35-36); here the stem is fp32 and the
transformer uses bf16 tensor-core GEMMs with fp32 accumulation and an fp32 residual stream, so the gate is relative,
as for the PPG extractor: rel-L2 <= 2e-2 and cosine >= 0.999 against the reference's fp32 output."""
import numpy as np
import pytest
import torch

from tests.util import GOLDEN, max_abs, rel_l2
from whisper_vits_svc_b200 import synth

pytestmark = pytest.mark.gpu


def _cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm()))


@pytest.fixture(scope="module")
def models():
    from whisper_vits_svc_b200 import hubert_infer
    cache = {}

    def get(seed):
        if seed not in cache:
            sd = synth.hubert_checkpoint(seed)
            cache[seed] = (sd, hubert_infer.HubertSoftB200(sd, "cuda"))
        return cache[seed]
    return get


@pytest.mark.parametrize("name", ["hubert_soft_b2_n8000", "hubert_soft_b1_n16123"])
def test_units_vs_reference_golden(models, name):
    """tests/golden/hubert_*.npz = `HubertSoft.units` of the unmodified reference (oracle/make_golden.py:hubert_case)."""
    from oracle import make_golden as mg
    ck_seed, B, n, in_seed = mg.HUBERT_CASES[name]
    g = np.load(f"{GOLDEN}/{name}.npz")
    sd, model = models(ck_seed)
    wav = torch.from_numpy(g["wav"])
    got = model.units(wav).cpu()
    ref = torch.from_numpy(g["units"])
    assert got.shape == ref.shape
    r, c = rel_l2(got, ref), _cos(got, ref)
    print(f"{name}: rel-l2 {r:.3e}, cosine {c:.6f}, max-abs {max_abs(got, ref):.3e}")
    assert r <= 2e-2 and c >= 0.999


def test_units_stages_vs_oracle(models):
    """3 s x 2 items against the CPU oracle, stage by stage (the fp32 stem must agree to fp32 accuracy, the bf16
    transformer within the relative gate), plus item independence and the frame count of the reference's conv stack."""
    from oracle import hubert_oracle as ho, make_golden as mg
    sd, model = models(31)
    wav = mg.hubert_wav(77, 2, 48000)
    taps_o, taps, taps32 = {}, {}, {}
    ref = ho.units(sd, wav, taps_o)
    got = model.units(wav, taps).cpu()
    T = ho.frames(48000)
    assert got.shape == ref.shape == (2, T, 256) and model.frames(48000) == T
    feats_o = taps_o["features"].transpose(1, 2)                      # time-major here, channel-major in the oracle
    got32 = model.units(wav, taps32, fp32_stem=True).cpu()            # flags bit 0: the stride-2 convs in fp32
    e = max_abs(taps32["features"].cpu(), feats_o)
    print(f"features (fp32 stem) max-abs {e:.3e} (rms {feats_o.pow(2).mean().sqrt():.3f})")
    assert e <= 2e-4
    r = rel_l2(taps["features"].cpu(), feats_o)
    print(f"features (tensor-core stem, bf16) rel-l2 {r:.3e}; units fp32-stem vs tensor-core-stem rel-l2 {rel_l2(got, got32):.3e}")
    assert r <= 1e-2 and rel_l2(got32, ref) <= 2e-2
    for nm in ("projected", "embedded", "layer0", "encoded"):
        r = rel_l2(taps[nm].cpu(), taps_o[nm])
        print(f"{nm}: rel-l2 {r:.3e}")
        assert r <= 2e-2, nm
    r, c = rel_l2(got, ref), _cos(got, ref)
    print(f"units 2 x 3 s: rel-l2 {r:.3e}, cosine {c:.6f}")
    assert r <= 2e-2 and c >= 0.999
    one = model.units(wav[1:2]).cpu()
    assert max_abs(one, got[1:2]) <= 1e-5                              # items do not interact


def test_pred_vec_matches_reference_chunking(models, tmp_path):
    """hubert/inference.py:25-50: 20 s chunks + remainder, rows concatenated; 41.3 s of audio -> 2 full chunks + 1.3 s."""
    from scipy.io import wavfile
    from oracle import hubert_oracle as ho, make_golden as mg
    from whisper_vits_svc_b200 import hubert_infer
    sd, model = models(31)
    n = 41 * 16000 + 4800
    wav = mg.hubert_wav(5, 1, n)[0, 0].clamp(-0.99, 0.99)
    pcm = (wav * 32768.0).round().clamp(-32768, 32767).to(torch.int16)
    path = tmp_path / "a.wav"
    wavfile.write(path, 16000, pcm.numpy())
    hubert_infer.pred_vec(model, str(path), str(tmp_path / "a.vec.npy"))
    got = np.load(tmp_path / "a.vec.npy")
    x = pcm.float() / 32768.0
    rows = sum(ho.frames(e - s) for s, e in hubert_infer.chunk_plan(n))
    assert got.shape == (rows, 256) and got.dtype == np.float32
    tail = ho.units(sd, x[40 * 16000:][None, None])[0]                 # the last (short) chunk against the oracle
    r = rel_l2(torch.from_numpy(got[-tail.shape[0]:]), tail)
    print(f"pred_vec: rows {rows}, tail rel-l2 {r:.3e}")
    assert r <= 2e-2
