"""Dataset preparation on the device: the loader, batch plan and retry loop the preprocess_*.py CLIs share.

Files are read by host threads while the device works on earlier ones.  `run_batched` groups them into device
batches, saves each result, reports and skips a file that fails to load, and retries a failing device batch file by
file so that only the culprit is lost.  Ragged batches are padded to their longest item, so with a `size` function
the plan sorts a bounded look-ahead window of loaded files by size before cutting it into batches: neighbours in
length share a batch, and the padding stays small."""
from __future__ import annotations

import collections
import os
import sys
from concurrent.futures import ThreadPoolExecutor
from typing import Callable, List, Optional, Sequence, Tuple


def speaker_wavs(wav_dir: str, out_dir: str, ext: str) -> List[Tuple[str, str]]:
    """The walk of prepare/preprocess_ppg.py and preprocess_hubert.py: every `<wav_dir>/<speaker>/<file>.wav` ->
    (wav path, `<out_dir>/<speaker>/<file><ext>`; np.save appends .npy).  Creates the speaker output directories as
    the reference does; files outside speaker directories are not taken.  Speakers and files in sorted order."""
    jobs = []
    os.makedirs(out_dir, exist_ok=True)
    for spk in sorted(os.listdir(wav_dir)):
        if os.path.isdir(f"./{wav_dir}/{spk}"):
            os.makedirs(f"./{out_dir}/{spk}", exist_ok=True)
            for f in sorted(os.listdir(f"./{wav_dir}/{spk}")):
                if f.endswith(".wav"):
                    jobs.append((f"{wav_dir}/{spk}/{f}", f"{out_dir}/{spk}/{f[:-4]}{ext}"))
    return jobs


def plan_window(sizes: Sequence[int], max_items: int, max_padded: int) -> List[List[int]]:
    """Cut one look-ahead window into device batches: indices sorted by size (ties keep their order), each batch at
    most `max_items` items and at most `max_padded` padded samples (items x its longest size).  An item larger than
    `max_padded` on its own forms a batch alone."""
    batches: List[List[int]] = []
    cur: List[int] = []
    for i in sorted(range(len(sizes)), key=lambda i: sizes[i]):
        if cur and (len(cur) == max_items or (len(cur) + 1) * sizes[i] > max_padded):
            batches.append(cur)
            cur = []
        cur.append(i)
    if cur:
        batches.append(cur)
    return batches


def run_batched(keys: Sequence, load: Callable, run: Callable, save: Callable, threads: int, batch: int,
                size: Optional[Callable] = None, max_padded: int = 0, window: int = 0) -> dict:
    """Process every key: `load(key)` on `threads` host threads -> payload; `run([payload, ...])` on the device ->
    one result per payload; `save(key, result)`.  At most `window` files are loaded ahead of the ones being
    processed (default: 2 x batch in order, 8 x batch with a size plan, whose padding falls as the window
    grows), so host memory stays bounded.

    size None: batches of up to `batch` files in the order given.  Otherwise each window of loaded files is planned
    by `plan_window(size(payload), batch, max_padded)`.  A file that fails to load or, retried alone, fails on the
    device is reported on stderr and skipped.  Returns {"failed", "samples", "padded"}: the failures, and the sizes
    of the items run against the padded size of their batches (both 0 without `size`)."""
    window = window or (2 if size is None else 8) * batch
    stats = {"failed": 0, "samples": 0, "padded": 0}

    def safe_load(k):
        try:
            return k, load(k), None
        except Exception as e:
            return k, None, e

    def skip(k, e):
        stats["failed"] += 1
        print(f"[!] skipped {k}: {e}", file=sys.stderr)

    def process(items):
        for k, r in zip([k for k, _ in items], run([p for _, p in items])):
            save(k, r)

    pending = collections.deque()
    it = iter(keys)
    done = 0
    with ThreadPoolExecutor(max(1, threads)) as pool:
        def refill():
            while len(pending) < window:
                k = next(it, None)
                if k is None:
                    return
                pending.append(pool.submit(safe_load, k))

        refill()
        while pending:
            chunk = [pending.popleft().result() for _ in range(min(batch if size is None else window, len(pending)))]
            refill()
            done += len(chunk)
            good = []
            for k, p, err in chunk:
                if err is None:
                    good.append((k, p))
                else:
                    skip(k, err)
            if size is None:
                groups = [good] if good else []
            else:
                sizes = [size(p) for _, p in good]
                plan = plan_window(sizes, batch, max_padded)
                groups = [[good[i] for i in g] for g in plan]
                for g in plan:
                    stats["samples"] += sum(sizes[i] for i in g)
                    stats["padded"] += len(g) * max(sizes[i] for i in g)
            for g in groups:
                try:
                    process(g)
                except Exception:
                    for item in g:   # find the file the batch failed on; the others are still written
                        try:
                            process([item])
                        except Exception as e:
                            skip(item[0], e)
            print(f"{done}/{len(keys)}")
    return stats
