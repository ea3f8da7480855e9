"""Host logic of the ragged conversion batches (no GPU): BatchEngine.plan_ragged and the source groups."""
import math

import numpy as np

from whisper_vits_svc_b200 import hostio

HOP = 320


def _check_ragged_plan(lengths, mb):
    chunks, batches = hostio.BatchEngine.plan_ragged(lengths, HOP, mb)
    assert chunks == hostio.BatchEngine.plan(lengths, HOP, mb)[0]
    assert sorted(j for b in batches for j in b) == list(range(len(chunks)))   # every chunk exactly once
    last = None
    for b in batches:
        assert 1 <= len(b) <= mb
        ns = [chunks[j][2] - chunks[j][1] for j in b]
        assert ns == sorted(ns, reverse=True)               # the first chunk is the batch's padded length
        assert last is None or ns[0] <= last                # lengths never increase from one batch to the next
        last = ns[-1]
    for u, n in enumerate(lengths):
        mine = sorted((c for c in chunks if c[0] == u), key=lambda c: c[1])
        assert [(c[1], c[2], c[3], c[4]) for c in mine] == hostio.chunk_plan(n, HOP)
        assert sum(len(range((c[2] - c[1]) * HOP)[c[3]:c[4]]) for c in mine) == n * HOP - 1
    return chunks, batches


def test_plan_ragged_covers_sorts_and_reassembles():
    lengths = [1000, 1000, 2600, 37, 1000, 5050, 1, 2500, 2511, 1000, 300, 2490]
    for mb in (1, 3, 4, 32):
        chunks, batches = _check_ragged_plan(lengths, mb)
        assert len(batches) == math.ceil(len(chunks) / mb)   # every batch but the last is full


def test_plan_ragged_distinct_lengths_fill_batches():
    rs = np.random.RandomState(5)
    lengths = [int(v) for v in rs.randint(200, 2801, size=512)]
    chunks, batches = _check_ragged_plan(lengths, 32)
    assert len(batches) == math.ceil(len(chunks) / 32)
    # the equal-length plan of the same utterances needs one call per distinct chunk length or more
    assert len(hostio.BatchEngine.plan(lengths, HOP, 32)[1]) >= len({c[2] - c[1] for c in chunks}) > len(batches)


def test_plan_ragged_all_distinct_chunk_lengths():
    lengths = list(range(1, 101))
    chunks, batches = _check_ragged_plan(lengths, 7)
    assert len(chunks) == 100 and len(batches) == math.ceil(100 / 7)


def test_source_groups_cap_batch_and_padded_frames():
    lengths = [2600, 10, 5000, 300, 300, 2600, 90000, 41]
    groups = hostio.BatchEngine.source_groups(lengths, 3, 6000)
    assert sorted(u for g in groups for u in g) == list(range(len(lengths)))
    for g in groups:
        n = [lengths[u] for u in g]
        assert n == sorted(n, reverse=True) and len(g) <= 3
        assert len(g) == 1 or len(g) * n[0] <= 6000        # an utterance longer than the cap goes alone
    assert [lengths[g[0]] for g in groups] == sorted((lengths[g[0]] for g in groups), reverse=True)
    assert [6] in groups and [2] in groups
