"""Data preparation under torchrun, on the host: the share of the files each rank takes (disjoint, covering,
balanced, the same on every rank, the list itself without torchrun) and, in 2-rank gloo runs of
svc_preprocessing.py's step loop with stub steps, the agreed exit status and the host steps that run on rank 0 only."""
import os

import numpy as np
import pytest

from tests.ranks import RANK_PID_LINES, alive, rank_pids, torchrun
from tests.util import ROOT
from whisper_vits_svc_b200 import dataset

TIMEOUT = 300


@pytest.mark.parametrize("seed", range(40))
def test_shares_are_disjoint_cover_and_balance(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(0, 60))
    sizes = [int(s) for s in rng.integers(0, 1 << 20, n)]
    if n and seed % 4 == 0:
        sizes[: n // 2] = [sizes[0]] * (n // 2)           # ties: dealt by position
    jobs = [f"wav/{i:03d}.wav" for i in range(n)]
    for world in range(1, 9):
        parts = [dataset.share(jobs, sizes, r, world) for r in range(world)]
        assert sorted(j for p in parts for j in p) == jobs, world
        for p in parts:
            assert p == sorted(p)                           # each share keeps the walk's order
        tot = [sum(sizes[jobs.index(j)] for j in p) for p in parts]
        assert max(tot) - min(tot) <= max(sizes, default=0), (world, tot)
        again = [dataset.share(list(jobs), list(sizes), r, world) for r in range(world)]
        assert again == parts


def test_world_one_returns_the_list_itself(monkeypatch):
    jobs = [("b.wav", "x"), ("a.wav", "y")]
    assert dataset.share(jobs, [1, 2], 0, 1) is jobs
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    assert dataset.rank_share(jobs) is jobs
    monkeypatch.setenv("WORLD_SIZE", "1")
    assert dataset.rank_share(jobs) is jobs


def test_share_does_not_depend_on_listing_order(tmp_path, monkeypatch):
    """Ranks that list the same files in different orders (os.listdir gives no order) still take disjoint shares that
    cover the list, each in its own listing order."""
    sizes = _tree(tmp_path, np.random.default_rng(5), 23)
    monkeypatch.chdir(tmp_path)
    monkeypatch.setenv("WORLD_SIZE", "3")
    walk = sorted(sizes)
    parts = []
    for r in range(3):
        listing = [walk[i] for i in np.random.default_rng(r).permutation(len(walk))]
        monkeypatch.setenv("RANK", str(r))
        mine = dataset.rank_share(listing, path=lambda w: w)
        assert mine == [w for w in listing if w in set(mine)]
        parts.append(mine)
    assert sorted(w for p in parts for w in p) == walk


def _tree(root, rng, n):
    sizes = {}
    for i in range(n):
        rel = f"spk{i % 3}/{i:03d}.wav"
        p = root / "wav" / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_bytes(b"\0" * int(rng.integers(100, 50000)))
        sizes[f"wav/{rel}"] = p.stat().st_size
    return sizes


def test_every_rank_walks_the_same_tree_into_its_own_share(tmp_path, monkeypatch):
    """Each rank walks the tree itself; the shares partition the walk and balance the bytes to within one file."""
    sizes = _tree(tmp_path, np.random.default_rng(7), 37)
    monkeypatch.chdir(tmp_path)
    for world in (2, 3, 8):
        monkeypatch.setenv("WORLD_SIZE", str(world))
        parts = []
        for r in range(world):
            monkeypatch.setenv("RANK", str(r))
            parts.append(dataset.rank_share(dataset.speaker_wavs("wav", "out", ".pit")))
        walk = dataset.speaker_wavs("wav", "out", ".pit")
        assert sorted(j for p in parts for j in p) == sorted(walk)
        tot = [sum(sizes[w] for w, _ in p) for p in parts]
        assert max(tot) - min(tot) <= max(sizes.values())


def test_ppg_share_is_taken_before_done_files_are_dropped(tmp_path, monkeypatch):
    """Rank 1's outputs appearing while rank 0 walks do not change rank 0's share; its own done files are dropped."""
    import preprocess_ppg
    _tree(tmp_path, np.random.default_rng(3), 12)
    monkeypatch.chdir(tmp_path)
    monkeypatch.setenv("WORLD_SIZE", "2")
    monkeypatch.setenv("RANK", "0")
    mine = preprocess_ppg.ppg_jobs("wav", "ppg")
    monkeypatch.setenv("RANK", "1")
    theirs = preprocess_ppg.ppg_jobs("wav", "ppg")
    for _, p in theirs:
        open(f"{p}.npy", "wb").close()
    monkeypatch.setenv("RANK", "0")
    assert preprocess_ppg.ppg_jobs("wav", "ppg") == mine
    open(f"{mine[0][1]}.npy", "wb").close()
    assert preprocess_ppg.ppg_jobs("wav", "ppg") == mine[1:]


WORKER = r"""
import os, sys
sys.path.insert(0, os.environ["SVCB_ROOT"])
import svc_preprocessing as P
from whisper_vits_svc_b200 import dataset

out, case = os.environ["SVCB_OUT"], os.environ["SVCB_CASE"]
rank = int(os.environ["RANK"])


def record(name):
    with open(os.path.join(out, f"{name}.{rank}"), "a") as f:
        f.write("ran\n")


def stub(step):
    script = step.split()[0]
    if case == "import_rank0" and script == "preprocess_train.py" and rank == 0:
        raise ImportError("stub import failure on rank 0")

    @dataset.rank_main
    def device_step(argv):
        record(script)
        jobs = dataset.rank_share([("only.wav", "only.out")], path=lambda j: j[0])   # rank 1's share is empty
        if case == "raise_rank1" and script == "preprocess_crepe.py" and rank == 1:
            raise RuntimeError("stub failure on rank 1")
        if case == "nonzero_rank0" and script == "preprocess_ppg.py" and rank == 0:
            return 2
        dataset.report_failed(len(jobs), len(jobs))   # the one file fails, on whichever rank takes it
        return 0

    def host_step(argv):
        record(script)
        return 0

    return (host_step if script in P.HOST_STEPS else device_step), step.split()[1:]


status = P.run_steps(P.STEPS, stub)
with open(os.path.join(out, f"status.{rank}"), "w") as f:
    f.write(str(status))
"""


def _launch(tmp_path, case):
    """Two ranks of the worker under torchrun, stopped if they outlive TIMEOUT (tests/ranks.py)."""
    script = tmp_path / "worker.py"
    script.write_text(RANK_PID_LINES + WORKER)
    env = dict(os.environ, SVCB_ROOT=ROOT, SVCB_OUT=str(tmp_path), SVCB_CASE=case)
    code, out, err = torchrun([str(script)], 2, tmp_path, env, TIMEOUT, tmp_path)
    if code is None:
        pytest.fail(f"{case}: the ranks did not finish in {TIMEOUT} s")
    assert code == 0, out[-3000:] + err[-3000:]
    status = [int((tmp_path / f"status.{r}").read_text()) for r in (0, 1)]
    ran = {f.name: f.read_text().count("ran") for f in tmp_path.iterdir() if f.name.startswith("preprocess_")}
    return status, ran, out, err


def _ran_through(ran, last):
    """The device steps run on both ranks and the host steps on rank 0 alone, each once, up to step `last`."""
    import svc_preprocessing as P
    want = {}
    for step in P.STEPS[:last]:
        script = step.split()[0]
        for r in ((0,) if script in P.HOST_STEPS else (0, 1)):
            want[f"{script}.{r}"] = want.get(f"{script}.{r}", 0) + 1
    assert ran == want


@pytest.mark.slow
def test_step_loop_every_rank_succeeds_with_an_empty_share(tmp_path):
    status, ran, out, err = _launch(tmp_path, "ok")
    assert status == [0, 0], err[-3000:]
    _ran_through(ran, 10)
    assert out.count("Command: python ") == 10                     # rank 0 prints the step lines
    assert err.count("1 of 1 files failed") == 7                   # one summed line per device step, by rank 0


@pytest.mark.slow
def test_step_loop_raise_on_rank1_stops_every_rank(tmp_path):
    status, ran, _, err = _launch(tmp_path, "raise_rank1")
    assert status == [1, 1]
    assert "stub failure on rank 1" in err
    _ran_through(ran, 3)


@pytest.mark.slow
def test_step_loop_nonzero_on_rank0_stops_every_rank(tmp_path):
    status, ran, _, _ = _launch(tmp_path, "nonzero_rank0")
    assert status == [1, 1]
    _ran_through(ran, 4)


SLEEPER = """
import time
time.sleep(3600)
"""


@pytest.mark.slow
def test_timed_out_ranks_are_stopped(tmp_path):
    """Ranks that outlive the launch's timeout are all stopped: torchrun runs each in a session of its own, out of
    reach of its launcher's process group."""
    script = tmp_path / "sleeper.py"
    script.write_text(RANK_PID_LINES + SLEEPER)
    code, _, _ = torchrun([str(script)], 2, tmp_path, dict(os.environ), 45, tmp_path)
    pids = rank_pids(tmp_path)
    assert code is None and len(pids) == 2
    assert not any(alive(pid) for pid in pids)


@pytest.mark.slow
def test_step_loop_import_failure_on_rank0_stops_every_rank(tmp_path):
    status, ran, _, err = _launch(tmp_path, "import_rank0")
    assert status == [1, 1]
    assert "stub import failure on rank 0" in err
    _ran_through(ran, 8)
