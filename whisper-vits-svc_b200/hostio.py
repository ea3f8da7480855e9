"""Host loop and wire formats of the inference CLIs (svc_inference.py of the reference).

Arithmetic-free glue, restated from the reference so the drop-in produces byte-compatible
outputs: checkpoint loading (svc_inference.py:61-74), feature preparation (:172-199), the
2500-frame chunk loop with +-10-frame overlap discard (:77-134), the pitch CSV format
(pitch/inference.py:102-119).  The only structural change: chunks of equal length are run as
batch items of ONE device call instead of a Python loop of batch-1 calls (chunks are
independent: the overlap is discarded, not blended).
"""
from __future__ import annotations

import os
from typing import List, Sequence, Tuple

import numpy as np
import torch


def load_svc_model(checkpoint_path: str, model):
    """svc_inference.py:61-74: key-by-key copy; missing keys are printed and keep their default."""
    assert os.path.isfile(checkpoint_path), checkpoint_path
    ckpt = torch.load(checkpoint_path, map_location="cpu", weights_only=False)
    saved = ckpt["model_g"]
    state = model.state_dict()
    new = {}
    for k, v in state.items():
        if k in saved:
            new[k] = saved[k]
        else:
            print("%s is not in the checkpoint" % k)
            new[k] = v
    model.load_state_dict(new)
    return model


def save_svc_model(model, checkpoint_path: str):
    """svc_export.py:40-45: {'model_g': state_dict}."""
    torch.save({"model_g": {k: v.detach().cpu() for k, v in model.state_dict().items()}}, checkpoint_path)


def load_csv_pitch(path: str) -> List[int]:
    """pitch/inference.py:113-119: last comma-separated field of every line, as int."""
    pitch = []
    with open(path, "r", encoding="utf-8") as f:
        for line in f.readlines():
            pitch.append(int(line.strip().split(",")[-1]))
    return pitch


def save_csv_pitch(pitch: Sequence[float], path: str):
    """pitch/inference.py:102-110: '{m}m {s}s {ms:3d},{int Hz}' every 10 ms."""
    with open(path, "w", encoding="utf-8") as f:
        for i in range(len(pitch)):
            t = i * 10
            minute = t // 60000
            seconds = (t - minute * 60000) // 1000
            millisecond = t % 1000
            print(f"{minute}m {seconds}s {millisecond:3d},{int(pitch[i])}", file=f)


def shift_pitch(pit: Sequence[int], shift: int) -> torch.Tensor:
    """svc_inference.py:187-200 and svc_inference_shift.py:63-65: the CSV pitch times 2^(shift/12) in float64, then
    rounded once to float32.  (At shift 0 the factor is exactly 1, so the integer pitch passes unchanged.)"""
    return torch.FloatTensor(np.array(pit) * (2 ** (shift / 12)))


def prepare_features(ppg_path: str, vec_path: str, pit_path: str, shift: int = 0):
    """svc_inference.py:172-199: 20 ms rows repeated x2, CSV pitch, optional 2^(k/12) shift."""
    # (torch.from_numpy on the repeated float32 array: the same values as the reference's torch.FloatTensor(...)
    #  without a second 5 MB copy per utterance)
    ppg = torch.from_numpy(np.ascontiguousarray(np.repeat(np.load(ppg_path), 2, 0), dtype=np.float32))
    vec = torch.from_numpy(np.ascontiguousarray(np.repeat(np.load(vec_path), 2, 0), dtype=np.float32))
    return ppg, vec, shift_pitch(load_csv_pitch(pit_path), shift)


def extract_missing_features(wave: str, ppg: str | None, vec: str | None) -> Tuple[str, str]:
    """svc_inference.py:138-148, in process: a missing `vec` / `ppg` path is extracted from `wave` by the device
    HuBERT-Soft / Whisper encoders into svc_tmp.vec.npy / svc_tmp.ppg.npy, with the checkpoints
    hubert_pretrain/hubert-soft-0d54a1f4.pt and whisper_pretrain/large-v2.pt of the working directory.
    Returns the (ppg, vec) paths."""
    if vec is None:
        from . import hubert_infer
        vec = "svc_tmp.vec.npy"
        print(f"Auto run : H100 hubert-soft encoder -w {wave} -v {vec}")
        hm = hubert_infer.load_model(os.path.join("hubert_pretrain", "hubert-soft-0d54a1f4.pt"), "cuda")
        hubert_infer.pred_vec(hm, wave, vec)
        del hm                      # (its device weights are freed before Whisper large-v2 loads)
    if ppg is None:
        from . import whisper_infer
        ppg = "svc_tmp.ppg.npy"
        print(f"Auto run : H100 whisper encoder -w {wave} -p {ppg}")
        wm = whisper_infer.load_model(os.path.join("whisper_pretrain", "large-v2.pt"), "cuda")
        whisper_infer.pred_ppg(wm, wave, ppg, "cuda")
    return ppg, vec


def extract_missing_pitch(wave: str, pit: str | None, crepe_path: str) -> str:
    """svc_inference.py:150-154, in process: a missing `pit` path is extracted from `wave` by the device CREPE-full
    model (`crepe_path`, the checkpoint pitch_inference.py reads) into svc_tmp.pit.csv, as pitch_inference.py writes
    it.  The model is freed before returning.  Returns the pit path."""
    if pit is None:
        from . import crepe_infer
        pit = "svc_tmp.pit.csv"
        print(f"Auto run : H100 CREPE pitch extractor -w {wave} -p {pit}")
        cm = crepe_infer.load_model(crepe_path, "cuda")
        crepe_infer.pred_pit(cm, wave, pit)
        del cm
    return pit


def chunk_plan(all_frame: int, hop_size: int, out_chunk: int = 2500, hop_frame: int = 10
               ) -> List[Tuple[int, int, int, int]]:
    """The reference's chunk arithmetic (svc_inference.py:94-115,129-131) as data:
    [(cut_s, cut_e, cut_s_out, cut_e_out)] in frames / samples; cut_e_out is the (negative) end
    index of the slice applied to the chunk's output (-1 on the last chunk, which drops one sample)."""
    plan = []
    out_index = 0
    while out_index < all_frame:
        if out_index == 0:
            cut_s, cut_s_out = 0, 0
        else:
            cut_s, cut_s_out = out_index - hop_frame, hop_frame * hop_size
        if out_index + out_chunk + hop_frame > all_frame:
            cut_e, cut_e_out = all_frame, -1
        else:
            cut_e, cut_e_out = out_index + out_chunk + hop_frame, -1 * hop_frame * hop_size
        plan.append((cut_s, cut_e, cut_s_out, cut_e_out))
        out_index += out_chunk
    return plan


def svc_infer(model, spk, pit, ppg, vec, hp, device, write_pit_wav: str | None = "svc_out_pit.wav",
              rand_ini=None, noise=None, eps_fn=None, max_batch: int = 16, retrieval=None):
    """svc_inference.py:77-134.  Returns the float32 waveform as a numpy array of length
    n_frames*hop - 1 (the reference's last-chunk slice).  `rand_ini`/`noise` and
    `eps_fn(chunk_idx, 1, n_frames) -> [1, inter_channels, n_frames]` (one call per chunk) inject the
    reference's random draws for parity tests.  `retrieval`: an object with `retriv_whisper` / `retriv_hubert`
    (retrieval.py) or None.  The reference applies it per chunk (svc_inference.py:117-118); retrieval is row-wise,
    so applying it once to the whole utterance gives the same rows."""
    len_min = min(pit.size(0), vec.size(0), ppg.size(0))
    pit, vec, ppg = pit[:len_min], vec[:len_min, :], ppg[:len_min, :]
    if retrieval is not None:
        ppg, vec = retrieval.retriv_whisper(ppg), retrieval.retriv_hubert(vec)
    hop = int(hp.data.hop_length)
    with torch.no_grad():
        spk = spk.unsqueeze(0).to(device)
        source = model.pitch2source(pit.unsqueeze(0).to(device), rand_ini=rand_ini, noise=noise)
        if write_pit_wav:
            from scipy.io.wavfile import write
            write(write_pit_wav, hp.data.sampling_rate, model.source2wav(source))
        plan = chunk_plan(len_min, hop)
        outs: List[np.ndarray | None] = [None] * len(plan)
        # group chunk indices by length; equal-length chunks become one batch
        by_len = {}
        for i, (cs, ce, _, _) in enumerate(plan):
            by_len.setdefault(ce - cs, []).append(i)
        for n, idxs in by_len.items():
            for g0 in range(0, len(idxs), max_batch):
                grp = idxs[g0:g0 + max_batch]
                B = len(grp)
                sub_ppg = torch.stack([ppg[plan[i][0]:plan[i][1]] for i in grp]).to(device)
                sub_vec = torch.stack([vec[plan[i][0]:plan[i][1]] for i in grp]).to(device)
                sub_pit = torch.stack([pit[plan[i][0]:plan[i][1]] for i in grp]).to(device)
                sub_len = torch.LongTensor([n] * B).to(device)
                sub_har = torch.cat([source[:, :, plan[i][0] * hop:plan[i][1] * hop] for i in grp], 0)
                eps = None
                if eps_fn is not None:
                    eps = torch.cat([eps_fn(i, 1, n) for i in grp], 0)
                out = model.inference(sub_ppg, sub_vec, sub_pit, spk.expand(B, -1), sub_len, sub_har, eps=eps)
                out = out[:, 0].cpu().numpy()
                for b, i in enumerate(grp):
                    outs[i] = out[b][plan[i][2]:plan[i][3]]
        return np.concatenate(outs).astype(np.float32)


# ------------------------------------------------------------------------------------------------ batched engine
class BatchEngine:
    """Many utterances through ONE model with full device batches (SURVEY.md §8e: "bucket into batches per
    rank"; the reference runs one subprocess and batch-1 device calls per file, svc_inference_batch.py:39-43).

    Every utterance is cut by the reference's own chunk plan (svc_inference.py:101-131: 2500-frame chunks, +-10
    frames of discarded overlap) and the chunks of ALL queued utterances run up to `max_batch` at a time.
    Host->device copies of the next batch and the device->host copy of the previous result run on side streams and
    overlap the current batch's kernels.

    ragged=False (plan): only equal-length chunks share a batch.  The model's `inference` pads by replication and
    convolves with zero padding at the end of the batch, so a chunk padded to a longer neighbour would differ from
    the reference's batch-1 result in its last few hundred samples.  On real data almost every chunk has its own
    length, so this runs about one chunk per call.
    ragged=True (plan_ragged): chunks sorted by length, longest first, fill every batch, through the model's
    `inference_ragged` (precision 3), which gives each chunk bitwise what a lone call of its own length gives.
    The NSF sources of whole utterances come from padded `pitch2source` calls over groups of utterances sorted by
    length; the source scan is causal, so each utterance's prefix is its lone source.

        eng = BatchEngine(model, hp, device, ragged=True)
        for key, wave in eng.run(jobs):      # jobs: iterable of (key, spk, pit, ppg, vec) CPU tensors
            ...                              # wave: float32 numpy array of n_frames*hop - 1 samples
    """

    # padded frames per padded pitch2source call: its [B, T*hop, n_harmonics] noise draw is 3.5 KB per frame
    SOURCE_FRAMES = 32 * 2520

    def __init__(self, model, hp, device, max_batch: int = 32, window: int = 128, ragged: bool = False):
        self.model, self.hp, self.device = model, hp, torch.device(device)
        self.max_batch, self.window = int(max_batch), int(window)
        self.ragged = bool(ragged)
        self.hop = int(hp.data.hop_length)
        self.device_seconds = 0.0          # time spent inside device batches (CUDA events)
        self.batches = 0                   # device batches (model inference calls)
        self.samples = 0
        self._events = []
        self._pinned = {}

    # -- planning (pure host logic, unit-tested on CPU)
    @staticmethod
    def plan(lengths: Sequence[int], hop: int, max_batch: int):
        """lengths[i] = frames of utterance i -> (chunks, batches): chunks[j] = (utt, cs, ce, out_start, out_end)
        exactly as chunk_plan() gives them per utterance; batches = lists of chunk indices of equal length,
        longest first, each at most max_batch long."""
        chunks = []
        for u, n in enumerate(lengths):
            for (cs, ce, so, eo) in chunk_plan(int(n), hop):
                chunks.append((u, cs, ce, so, eo))
        by_len = {}
        for j, (u, cs, ce, _, _) in enumerate(chunks):
            by_len.setdefault(ce - cs, []).append(j)
        batches = []
        for n in sorted(by_len, reverse=True):
            idx = by_len[n]
            for g0 in range(0, len(idx), max_batch):
                batches.append(idx[g0:g0 + max_batch])
        return chunks, batches

    @staticmethod
    def plan_ragged(lengths: Sequence[int], hop: int, max_batch: int):
        """The chunks of plan(); batches = runs of up to max_batch chunks of any length, longest first (so a
        batch pads its chunks to its first one's length, and lengths never increase from one batch to the next)."""
        chunks, _ = BatchEngine.plan(lengths, hop, max_batch)
        order = sorted(range(len(chunks)), key=lambda j: chunks[j][1] - chunks[j][2])   # stable: by length, descending
        return chunks, [order[g0:g0 + max_batch] for g0 in range(0, len(order), max_batch)]

    @staticmethod
    def source_groups(lengths: Sequence[int], max_batch: int, max_frames: int):
        """Utterance indices in groups for padded pitch2source calls: sorted by length, longest first, at most
        max_batch per group and at most max_frames padded frames (a longer utterance gets a group of its own)."""
        order = sorted(range(len(lengths)), key=lambda u: -int(lengths[u]))
        groups = []
        for u in order:
            g = groups[-1] if groups else None
            if g is None or len(g) == max_batch or (len(g) + 1) * int(lengths[g[0]]) > max_frames:
                groups.append([u])
            else:
                g.append(u)
        return groups

    def run(self, jobs):
        win = []
        for job in jobs:
            win.append(job)
            if len(win) == self.window:
                yield from self._run_window(win)
                win = []
        if win:
            yield from self._run_window(win)

    @torch.no_grad()
    def _run_window(self, win):
        dev, hop, model = self.device, self.hop, self.model
        cur = torch.cuda.current_stream(dev)
        copy_s, out_s = torch.cuda.Stream(dev), torch.cuda.Stream(dev)
        feats = []
        for (key, spk, pit, ppg, vec) in win:
            n = min(pit.size(0), vec.size(0), ppg.size(0))       # svc_inference.py:78-81
            feats.append((key, spk, pit[:n], ppg[:n], vec[:n], n))
        lengths = [f[5] for f in feats]
        chunks, batches = (self.plan_ragged if self.ragged else self.plan)(lengths, hop, self.max_batch)
        # NSF source of whole utterances (svc_inference.py:89-91): equal-length utterances in one call, or (ragged)
        # groups of any length padded with unvoiced frames, each utterance keeping its own prefix
        source = [None] * len(feats)
        if self.ragged:
            groups = self.source_groups(lengths, self.max_batch, self.SOURCE_FRAMES)
        else:
            by_n = {}
            for u, n in enumerate(lengths):
                by_n.setdefault(n, []).append(u)
            groups = [us[g0:g0 + self.max_batch] for us in by_n.values() for g0 in range(0, len(us), self.max_batch)]
        for grp in groups:
            f0 = torch.zeros(len(grp), lengths[grp[0]])
            for k, u in enumerate(grp):
                f0[k, :lengths[u]] = feats[u][2]
            src = model.pitch2source(f0.to(dev, non_blocking=True))
            for k, u in enumerate(grp):
                source[u] = src[k:k + 1, :, :lengths[u] * hop]
        pieces = {u: [] for u in range(len(feats))}

        def pinned(name, slot, shape, dtype=torch.float32):
            """Reused pinned staging buffers (cudaHostAlloc per batch was most of the host time)."""
            key = (name, slot)
            numel = int(np.prod(shape))
            buf = self._pinned.get(key)
            if buf is None or buf.numel() < numel or buf.dtype != dtype:
                buf = torch.empty(numel, dtype=dtype).pin_memory()
                self._pinned[key] = buf
            return buf[:numel].view(*shape)

        h2d_done = [None, None]

        def stage(bi):   # features of batch bi -> pinned set (bi & 1) -> device tensors on the copy stream
            idx = batches[bi]
            slot = bi & 1
            if h2d_done[slot] is not None:
                h2d_done[slot].synchronize()          # the copy that last read this pinned set has finished
            n = chunks[idx[0]][2] - chunks[idx[0]][1]    # (ragged: the longest; rows past a chunk's end are don't-care)
            B = len(idx)
            host = {"ppg": pinned("ppg", slot, (B, n, feats[0][3].shape[1])), "vec": pinned("vec", slot, (B, n, feats[0][4].shape[1])),
                    "pit": pinned("pit", slot, (B, n)), "spk": pinned("spk", slot, (B, feats[0][1].shape[0]))}
            for b, j in enumerate(idx):
                u, cs, ce = chunks[j][0], chunks[j][1], chunks[j][2]
                host["ppg"][b, :ce - cs].copy_(feats[u][3][cs:ce]); host["vec"][b, :ce - cs].copy_(feats[u][4][cs:ce])
                host["pit"][b, :ce - cs].copy_(feats[u][2][cs:ce]); host["spk"][b].copy_(feats[u][1])
            with torch.cuda.stream(copy_s):
                d = {k: v.to(dev, non_blocking=True) for k, v in host.items()}
                d["len"] = torch.full((B,), n, dtype=torch.int64, device=dev)
                ev = torch.cuda.Event()
                ev.record(copy_s)
            h2d_done[slot] = ev
            return d, ev

        def collect(bi, res, done):   # device -> host copy of batch bi has landed: cut the reference's slices out
            done.synchronize()
            arr = res.numpy()
            for b, j in enumerate(batches[bi]):
                u, cs, ce, so, eo = chunks[j]
                pieces[u].append((cs, arr[b][:(ce - cs) * hop][so:eo].copy()))

        prev = None    # (batch index, pinned result, event) still in flight
        nxt = stage(0) if batches else None
        for bi in range(len(batches)):
            d, ev = nxt
            cur.wait_event(ev)
            if bi + 1 < len(batches):
                nxt = stage(bi + 1)
            idx = batches[bi]
            if self.ragged:
                n_frames = [chunks[j][2] - chunks[j][1] for j in idx]
                har = torch.zeros(len(idx), 1, n_frames[0] * hop, device=dev)
                for b, j in enumerate(idx):
                    har[b, :, :n_frames[b] * hop] = source[chunks[j][0]][0, :, chunks[j][1] * hop:chunks[j][2] * hop]
            else:
                har = torch.cat([source[chunks[j][0]][:, :, chunks[j][1] * hop:chunks[j][2] * hop] for j in idx], 0)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(cur)
            for t in d.values():
                t.record_stream(cur)
            if self.ragged:
                w = model.inference_ragged(d["ppg"], d["vec"], d["pit"], d["spk"], n_frames, har)
            else:
                w = model.inference(d["ppg"], d["vec"], d["pit"], d["spk"], d["len"], har)
            e1.record(cur)
            self.batches += 1
            self._events.append((e0, e1))
            if prev is not None:
                collect(*prev)                        # (its result buffer is the other slot)
            res = pinned("wave", bi & 1, (w.shape[0], w.shape[2]))
            with torch.cuda.stream(out_s):
                out_s.wait_event(e1)
                res.copy_(w[:, 0], non_blocking=True)
                done = torch.cuda.Event()
                done.record(out_s)
            w.record_stream(out_s)
            prev = (bi, res, done)
        if prev is not None:
            collect(*prev)
        for e0, e1 in self._events:
            self.device_seconds += e0.elapsed_time(e1) * 1e-3
        self._events = []
        for u, f in enumerate(feats):
            ps = [p for _, p in sorted(pieces[u], key=lambda t: t[0])]
            wave = ps[0] if len(ps) == 1 else np.concatenate(ps)     # (pieces are float32 copies already)
            self.samples += wave.shape[0]
            yield f[0], wave
