"""Host logic of filtered and subset lookups on the peer exchange, on CPU over ``gloo`` with a recording engine.

The engine stands in for ``CudaShardEngine``: ``group_search`` records what ``ShardedVectorBase`` asks the peer
exchange for (ties, mask kind, subset share, deferral) and returns empty results; ``upload_mask`` can be made to fail
on one rank.  The process group is wrapped to count collectives.  Checked: with ``exchange="peer"`` row masks,
per-query masks, predicates, ties, subsets and per-query subsets go to ``group_search`` and the process-group
exchange is not used; with ``exchange="nccl"`` nothing goes to it; errors from replicated arguments are raised
with no collective; a new mask costs one all-reduce and a mask already agreed on none; a failed upload on one
rank raises on every rank before anything is published; a deferred subset lookup is decoded at ``finish()``;
``close()`` drops what deferred lookups and agreed masks left behind.
The device side is covered by tests/test_gpu_peer_filtered.py.
"""

from __future__ import annotations

import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.test_sharded_gloo import _free_port  # noqa: E402

N, D = 37, 8


class RecordingEngine:
    def __init__(self):
        self.calls, self.rows, self.fail_upload = [], 0, False

    def load_rows(self, rows):
        self.rows = 0 if rows is None else len(rows)

    def n_local(self):
        return self.rows

    def group_search(self, dist_, pg, rank, world, q, k, floor, lo, defer, ties_low_first=False, mask=None,
                     subset=None):
        kind = None if mask is None else ("query" if np.ndim(mask[0]) == 2 else "row")
        share = None if subset is None else (len(subset[0]), subset[1] is not None, list(subset[2]))
        self.calls.append(("group", k, bool(defer), bool(ties_low_first), kind, share))
        b = len(q)
        return (torch.full((b, k), -1, dtype=torch.int64), torch.zeros((b, k)), torch.zeros(b, dtype=torch.int32))

    def upload_mask(self, mask, n_queries):
        self.calls.append(("upload",))
        if self.fail_upload:
            raise MemoryError("mask upload failed")

    def group_finish(self):
        self.calls.append(("group_finish",))
        return 0

    def finish(self):
        return 0

    def map_items(self, items, table):
        self.calls.append(("map", len(table)))
        return items

    def search_rows_packed(self, *a, **kw):
        raise AssertionError("the process-group path was taken")

    search_subset_packed = search_subsets_packed = search_rows_packed


class CountingDist:
    """torch.distributed with a count of the collectives ShardedVectorBase runs."""

    def __init__(self):
        self.n = 0

    def __getattr__(self, name):
        fn = getattr(dist, name)
        if name in ("all_reduce", "all_gather", "all_gather_into_tensor", "all_gather_object", "barrier"):
            def counted(*a, **kw):
                self.n += 1
                return fn(*a, **kw)
            return counted
        return fn


def _worker(rank: int, world: int, port: int):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from types import SimpleNamespace

        from oracle import vectorbase_oracle as O
        from typeagent_py_b200.sharded import ShardedVectorBase

        settings = SimpleNamespace(embedding_model=O.FakeEmbeddingModel(), min_score=0.85, max_matches=None)
        rng = np.random.default_rng(1)
        v = rng.standard_normal((N, D)).astype(np.float32)
        q = rng.standard_normal((3, D)).astype(np.float32)
        eng = RecordingEngine()
        sh = ShardedVectorBase(settings, engine=eng, exchange="peer")
        sh.deserialize(v)
        counting = CountingDist()
        sh._dist = counting
        allowed = rng.random(N) < 0.5

        # a new row mask: one all-reduce (the upload agreement), then the peer exchange; the same mask again: none
        sh.search_arrays(q, 4, allowed=allowed)
        assert counting.n == 1 and eng.calls == [("upload",), ("group", 4, False, False, "row", None)], eng.calls
        eng.calls.clear()
        sh.search_arrays(q, 4, allowed=allowed, ties_low_first=True)
        assert counting.n == 1 and eng.calls == [("group", 4, False, True, "row", None)], eng.calls
        eng.calls.clear()
        masks = rng.random((3, N)) < 0.5
        sh.search_arrays(q, 5, allowed=masks)
        assert counting.n == 2 and eng.calls == [("upload",), ("group", 5, False, False, "query", None)], eng.calls
        eng.calls.clear()
        sh.search_arrays(q, 4, ties_low_first=True)
        assert eng.calls == [("group", 4, False, True, None, None)], eng.calls
        eng.calls.clear()

        # a subset: this rank's share and its positions, merged positions decoded through the caller's list
        lo, hi = sh.local_range
        sub = np.array([0, N - 1, -1, 18, 19, 18, -N], np.int64)
        rows = np.where(sub < 0, sub + N, sub)
        mine = [i for i, r in enumerate(rows) if lo <= r < hi]
        sh.search_arrays(q, 3, subset=sub)
        assert eng.calls == [("group", 3, False, False, None, (len(mine), False, mine)), ("map", len(sub))], eng.calls
        eng.calls.clear()
        subsets = [[0, 1, N - 1], [], [-1, 20, 20]]
        sh.search_arrays(q, 2, subsets=subsets)
        assert eng.calls[0][0] == "group" and eng.calls[0][5][1] and eng.calls[1] == ("map", 6), eng.calls
        eng.calls.clear()

        # deferred on the device: decoded at finish(), after the library finished the searches
        sh.search_tensors(q, 3, subset=sub, defer_check=True)
        assert eng.calls == [("group", 3, True, False, None, (len(mine), False, mine))], eng.calls
        sh.finish()
        assert eng.calls[1:] == [("group_finish",), ("map", len(sub))], eng.calls
        eng.calls.clear()

        # errors from replicated arguments: on every rank, before any collective or device work
        n0 = counting.n
        for kw, err in ((dict(subset=[N]), IndexError), (dict(subset=[0], allowed=allowed), ValueError),
                        (dict(allowed=allowed[:-1]), ValueError), (dict(allowed=masks[:2]), ValueError),
                        (dict(subsets=[[0]] * 2), ValueError)):
            with pytest.raises(err):
                sh.search_arrays(q, 3, **kw)
        assert counting.n == n0 and eng.calls == [], eng.calls

        # a mask upload that fails on one rank raises on every rank, before anything is published
        eng.fail_upload = rank == world - 1
        with pytest.raises(MemoryError if eng.fail_upload else RuntimeError):
            sh.search_arrays(q, 3, allowed=rng.random(N) < 0.5)
        assert ("group" not in [c[0] for c in eng.calls]), eng.calls
        eng.fail_upload = False
        eng.calls.clear()

        # close() drops deferred decodes and the agreed masks with the pending lookups
        sh.search_tensors(q, 3, subset=sub, defer_check=True)
        assert sh._decode and sh._peer_masks
        sh.close()
        assert sh._decode == [] and sh._peer_masks == {} and sh._pending == []

        # exchange="nccl": the process-group path, never the peer exchange
        sh2 = ShardedVectorBase(settings, engine=RecordingEngine(), exchange="nccl")
        sh2.deserialize(v)
        with pytest.raises(AssertionError, match="process-group"):
            sh2.search_arrays(q, 3, subset=sub)
        assert sh2._engine.calls == []
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_peer_filter_routing_over_gloo(world):
    mp.spawn(_worker, args=(world, _free_port()), nprocs=world, join=True)
