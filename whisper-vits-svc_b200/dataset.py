"""Dataset preparation on the device: the loader, batch plan and retry loop the preprocess_*.py CLIs share.

Files are read by host threads while the device works on earlier ones.  `run_batched` groups them into device
batches, saves each result, reports and skips a file that fails to load, and retries a failing device batch file by
file so that only the culprit is lost.  Ragged batches are padded to their longest item, so with a `size` function
the plan sorts a bounded look-ahead window of loaded files by size before cutting it into batches: neighbours in
length share a batch, and the padding stays small.

Under `torchrun` every rank walks the same tree and takes its share of the files (`rank_share`): the same
longest-first deal on every rank, so no list is exchanged.  A CLI's `main` wrapped in `rank_main` then sums its
failures and agrees on its exit status over gloo, the only collectives; rank 0 prints the summed failure line."""
from __future__ import annotations

import collections
import contextlib
import datetime
import functools
import os
import sys
import traceback
from concurrent.futures import ThreadPoolExecutor
from typing import Callable, List, Optional, Sequence, Tuple

# How long a rank waits in a collective for the others: a rank may wait out the host steps of svc_preprocessing.py
# on rank 0, or a slower rank's share, so it is hours rather than gloo's default 30 minutes.  If a rank dies, torchrun
# stops the others without waiting for it.
GROUP_TIMEOUT = datetime.timedelta(hours=12)


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


def share(jobs: Sequence, sizes: Sequence[int], rank: int, world: int) -> list:
    """Rank `rank`'s part of `jobs` out of `world`: `shard.assign`'s deal of `sizes` (longest first, boustrophedon,
    ties by position), kept in the order given.  Every rank deals the same full list the same way, so the parts are
    disjoint and cover it with nothing exchanged, and the ranks' totals differ by at most one largest size.  World 1:
    `jobs` itself."""
    if world <= 1:
        return jobs
    from . import shard
    mine = set(shard.assign(sizes, world)[rank])
    return [j for i, j in enumerate(jobs) if i in mine]


def file_size(path: str) -> int:
    """Bytes of `path`; 0 for one that cannot be stat'ed, which still goes to a rank that reports it as failed."""
    try:
        return os.path.getsize(path)
    except OSError:
        return 0


def rank_share(jobs: Sequence, path: Callable = lambda job: job[0]) -> list:
    """This process's share of the full job list of a walk, by the sizes of the files `path(job)` names, for the
    rank and world size torchrun sets (RANK, WORLD_SIZE).  The deal runs over the jobs sorted by path, so it does not
    depend on the order a rank listed the directories in; the share keeps the order of `jobs`.  Share the full walk,
    before any filter on outputs that already exist: other ranks write theirs meanwhile, and a filtered list would
    differ from rank to rank.  Without torchrun (WORLD_SIZE unset or 1), `jobs` itself, in order."""
    from . import shard
    rank, _, world = shard.env_world()
    if world <= 1:
        return jobs
    order = sorted(range(len(jobs)), key=lambda i: path(jobs[i]))
    mine = set(share(order, [file_size(path(jobs[i])) for i in order], rank, world))
    return [j for i, j in enumerate(jobs) if i in mine]


@contextlib.contextmanager
def process_group():
    """The gloo group of a torchrun launch (WORLD_SIZE > 1), with this rank's device, cuda:(LOCAL_RANK % device
    count), made current.  A group that already exists is reused and left to its owner: svc_preprocessing.py holds
    one over all its steps, while a CLI run on its own makes one and destroys it before its `main` returns.  Does
    nothing without torchrun."""
    from . import shard
    _, local, world = shard.env_world()
    if world <= 1:
        yield
        return
    import torch
    import torch.distributed as dist
    if torch.cuda.is_available():
        torch.cuda.set_device(local % torch.cuda.device_count())
    own = not dist.is_initialized()
    if own:
        dist.init_process_group("gloo", timeout=GROUP_TIMEOUT)
    try:
        yield
    finally:
        if own:
            dist.destroy_process_group()


def sum_over_ranks(values: Sequence[int]) -> List[int]:
    """Element-wise sums of host integers over the ranks (one gloo all-reduce); `values` itself without torchrun."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()):
        return list(values)
    import torch
    t = torch.tensor(list(values), dtype=torch.int64)
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return [int(v) for v in t]


_tally = [0, 0]   # files failed, files taken: this rank's, for the running rank_main


def report_failed(failed: int, total: int) -> None:
    """The `N of M files failed` line on stderr, when N > 0.  Under `rank_main` with torchrun the counts are summed
    over the ranks first and rank 0 prints the line for all of them."""
    from . import shard
    if shard.env_world()[2] > 1:
        _tally[0] += failed
        _tally[1] += total
    elif failed:
        print(f"{failed} of {total} files failed", file=sys.stderr)


def rank_main(main: Callable) -> Callable:
    """Run a data-preparation CLI's `main(argv)` as one rank of a torchrun launch.  Each rank runs `main` on its
    share; a rank that raises (a bad argument, a missing model file) prints its traceback instead.  Then one gloo
    all-reduce sums the failed and taken files of `report_failed` and the count of ranks whose status is non-zero,
    which every rank joins, an empty share included.  Rank 0 prints the summed failure line, and every rank returns
    1 if any rank failed, else 0.  Without torchrun, `main` runs as it is."""
    @functools.wraps(main)
    def run(argv=None):
        from . import shard
        rank, _, world = shard.env_world()
        if world <= 1:
            return main(argv)
        with process_group():
            _tally[:] = [0, 0]
            try:
                status = main(argv)
            except SystemExit as e:
                if isinstance(e.code, str):
                    print(e.code, file=sys.stderr)
                status = 0 if e.code is None else e.code
            except Exception:
                traceback.print_exc()
                status = 1
            sys.stderr.flush()
            failed, total, bad = sum_over_ranks([_tally[0], _tally[1], int(bool(status))])
            if rank == 0 and failed:
                print(f"{failed} of {total} files failed", file=sys.stderr)
            return 1 if bad else 0
    return run


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
