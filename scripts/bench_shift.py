#!/usr/bin/env python
"""The pitch-shift sweep of svc_inference_shift.py: one synthetic 180 s utterance (18,000 frames, seeded features) at
all 25 shifts from -12 to +12, on a seeded synthetic checkpoint at precision 3, two ways:
  sweep  every shift one job of hostio.BatchEngine(ragged=True), as the CLI runs them;
  loop   25 sequential hostio.svc_infer calls, the reference's loop (svc_inference_shift.py:61-69).
Neither arm writes files.  After one warm-up run of each, the arms alternate --repeats times.  Per arm: device seconds
(CUDA events around every pitch2source and model call), wall seconds (host clock around the arm, ending in a device
synchronise), device calls (model calls) and audio seconds converted per wall second (median over the repeats; min and
max beside).  Then, with the draws silenced (eps = 0, zero source noise), both arms convert every shift once more and
the waveforms are compared with np.array_equal.  Prints one JSON line with the card and its power limit, read in the
same run.

    python scripts/bench_shift.py [--repeats 3]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

HOP, SR, FRAMES = 320, 32000, 18000
SHIFTS = list(range(-12, 13))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits",
                        "-i", str(torch.cuda.current_device())], capture_output=True, text=True, check=True).stdout
    name, pl = [s.strip() for s in q.strip().splitlines()[0].split(",")]
    return name, float(pl)


class Timed:
    """The model with CUDA events around each pitch2source and model call on the current stream."""

    def __init__(self, m):
        self.m, self.events, self.calls = m, [], 0

    def _timed(self, fn, *a, **kw):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn(*a, **kw)
        e1.record()
        self.events.append((e0, e1))
        return out

    def pitch2source(self, *a, **kw):
        return self._timed(self.m.pitch2source, *a, **kw)

    def inference(self, *a, **kw):
        self.calls += 1
        return self._timed(self.m.inference, *a, **kw)

    def inference_ragged(self, *a, **kw):
        self.calls += 1
        return self._timed(self.m.inference_ragged, *a, **kw)

    def device_seconds(self):
        return sum(e0.elapsed_time(e1) for e0, e1 in self.events) * 1e-3


class Quiet:
    """The model with its random draws silenced, so that both arms are deterministic."""

    def __init__(self, m, C):
        self.m, self.C = m, C

    def pitch2source(self, f0, **kw):
        B, T = f0.shape
        return self.m.pitch2source(f0, rand_ini=torch.zeros(B, 11), noise=torch.zeros(B, T * HOP, 11))

    def inference(self, ppg, vec, pit, spk, ppg_l, source, eps=None):
        return self.m.inference(ppg, vec, pit, spk, ppg_l, source, eps=torch.zeros(ppg.shape[0], self.C, ppg.shape[1]))

    def inference_ragged(self, ppg, vec, pit, spk, n_frames, source, eps=None):
        return self.m.inference_ragged(ppg, vec, pit, spk, n_frames, source,
                                       eps=torch.zeros(ppg.shape[0], self.C, ppg.shape[1]))


def utterance(hp, seed):
    """spk, integer CSV-style pitch with unvoiced runs, and the repeated 20 ms feature rows of one 180 s recording."""
    rs = np.random.RandomState(seed)
    pit = [int(v) for v in rs.randint(100, 501, size=FRAMES)]
    for s in range(0, FRAMES, 997):
        pit[s:s + 60] = [0] * len(pit[s:s + 60])
    ppg = torch.from_numpy(np.repeat(rs.randn(FRAMES // 2, hp.vits.ppg_dim).astype(np.float32), 2, 0))
    vec = torch.from_numpy(np.repeat(rs.randn(FRAMES // 2, hp.vits.vec_dim).astype(np.float32), 2, 0))
    spk = torch.from_numpy((rs.randn(hp.vits.spk_dim) * 0.05).astype(np.float32))
    return spk, pit, ppg, vec


def sweep(model, hp, jobs):
    from whisper_vits_svc_b200 import hostio
    eng = hostio.BatchEngine(model, hp, "cuda", ragged=True)
    return dict(eng.run(iter(jobs)))


def loop(model, hp, jobs):
    from whisper_vits_svc_b200 import hostio
    return {s: hostio.svc_infer(model, spk, pit, ppg, vec, hp, "cuda", write_pit_wav=None) for s, spk, pit, ppg, vec in jobs}


def timed_run(arm, model, hp, jobs):
    t = Timed(model)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = arm(t, hp, jobs)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    return t.device_seconds(), wall, t.calls, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    from whisper_vits_svc_b200 import hostio, hparams, models, synth
    assert torch.cuda.is_available(), "bench_shift needs a CUDA device"
    name, power = gpu_info()
    hp = hparams.load_hparams(os.path.join(ROOT, "configs", "base.yaml"))
    model = models.SynthesizerInfer(513, 25, hp, precision=3)
    model.load_state_dict(synth.svc_state_dict(hp, 1234))
    model.eval()
    model.to("cuda")
    spk, pit, ppg, vec = utterance(hp, 7)
    jobs = [(s, spk, hostio.shift_pitch(pit, s), ppg, vec) for s in SHIFTS]
    audio_s = len(SHIFTS) * (FRAMES * HOP - 1) / SR
    arms = {"sweep": sweep, "loop": loop}
    for arm in arms.values():          # warm-up: kernels, allocator, workspaces, pinned staging
        timed_run(arm, model, hp, jobs)
    samples = {k: {"device_s": [], "wall_s": []} for k in arms}
    res = {"metric": "pitch_shift_sweep", "gpu": name, "power_limit_w": power, "precision": 3, "repeats": args.repeats,
           "frames": FRAMES, "shifts": len(SHIFTS), "chunks": len(SHIFTS) * len(hostio.chunk_plan(FRAMES, HOP)),
           "audio_seconds": round(audio_s, 1)}
    for _ in range(args.repeats):
        for k, arm in arms.items():
            dev, wall, calls, out = timed_run(arm, model, hp, jobs)
            assert sorted(out) == SHIFTS and all(w.shape == (FRAMES * HOP - 1,) for w in out.values())
            samples[k]["device_s"].append(dev)
            samples[k]["wall_s"].append(wall)
            res[k] = {"device_calls": calls}
    for k in arms:
        dev, wall = sorted(samples[k]["device_s"]), sorted(samples[k]["wall_s"])
        res[k].update(device_s_median=round(float(np.median(dev)), 3), device_s_min=round(dev[0], 3),
                      device_s_max=round(dev[-1], 3), wall_s_median=round(float(np.median(wall)), 3),
                      wall_s_min=round(wall[0], 3), wall_s_max=round(wall[-1], 3),
                      audio_s_per_wall_s=round(audio_s / float(np.median(wall)), 1))
    res["wall_speedup"] = round(res["loop"]["wall_s_median"] / res["sweep"]["wall_s_median"], 3)
    res["device_speedup"] = round(res["loop"]["device_s_median"] / res["sweep"]["device_s_median"], 3)
    q = Quiet(model, hp.vits.inter_channels)
    a, b = sweep(q, hp, jobs), loop(q, hp, jobs)
    res["silenced_waveforms_equal"] = bool(sorted(a) == sorted(b) == SHIFTS and all(np.array_equal(a[s], b[s]) for s in SHIFTS))
    print(json.dumps(res), flush=True)
    assert res["silenced_waveforms_equal"], "the two arms' waveforms differ"


if __name__ == "__main__":
    main()
