"""Host logic of threshold searches on the peer exchange, on CPU over ``gloo``.

The engine stands in for ``CudaShardEngine``: besides the numpy threshold search of tests/test_sharded_range_gloo.py
(``range_local``, ``merge_range``: the process-group route) it has ``group_range``, which records the local arguments
it is given and returns the exact merged result (the ranks' lists exchanged with ``all_gather_object``).  Checked,
at worlds 1, 2 and 3: with ``exchange="peer"`` and more than one rank, ``search_range``, ``max_hits=0`` lookups and
filtered threshold searches go to ``group_range`` and never to the process-group exchange; one rank and
``exchange="nccl"`` keep the process-group route; errors from replicated arguments are raised on every rank before
any collective; the capacity plan of the range inbox as a pure function of (totals, capacity); and the grow
agreement (``reserve_everywhere``) when one rank's reservation fails.  The device side is covered by
tests/test_gpu_peer_range.py.
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

from tests.exact import dyadic_corpus, preset  # noqa: E402
from tests.test_gpu_range import expected_range  # noqa: E402
from tests.test_sharded_gloo import _free_port  # noqa: E402
from tests.test_sharded_range_gloo import CountingDist, RangeEngine, assert_same, exact_dots, make  # noqa: E402


class PeerRangeEngine(RangeEngine):
    """RangeEngine with the peer route: ``group_range`` records its local arguments and returns the exact merge."""

    def __init__(self):
        super().__init__()
        self.group_calls = []

    def group_search(self, *a, **kw):
        raise AssertionError("no top-k lookup runs in this test")

    def upload_mask(self, mask, n_queries):
        pass

    def group_range(self, dist_, pg, rank, world, q, floor, lo, ties_low_first, **local):
        self.group_calls.append(sorted(local))
        b = len(q)
        mine = (np.zeros(b + 1, np.int64), np.empty(0, np.int64), np.empty(0, np.float32))
        if len(self.rows) and not local:
            mine = expected_range(exact_dots(q, self.rows), floor, ties_low=ties_low_first, item_offset=lo)
        got = [None] * world
        dist.all_gather_object(got, mine, group=pg)
        out_o, out_i, out_s = [0], [], []
        for qi in range(b):
            it = np.concatenate([g[1][g[0][qi]:g[0][qi + 1]] for g in got])
            sc = np.concatenate([g[2][g[0][qi]:g[0][qi + 1]] for g in got])
            order = np.lexsort((it if ties_low_first else -it, -sc.view(np.uint32).astype(np.int64)))
            out_i.append(it[order])
            out_s.append(sc[order])
            out_o.append(out_o[-1] + len(order))
        return (torch.from_numpy(np.array(out_o, np.int64)), torch.from_numpy(np.concatenate(out_i)),
                torch.from_numpy(np.concatenate(out_s)))

    def map_items(self, items, table):
        items.copy_(torch.from_numpy(np.asarray(table, np.int64)[items.numpy()]))
        return items


def test_capacity_plan():
    from typeagent_py_b200.sharded import RANGE_MIN_HITS, range_capacity_plan, range_retain_hits

    # the retention: the largest power of two of hits whose bytes from every rank fit
    assert range_retain_hits(2, 64 << 20) == 1 << 21
    assert range_retain_hits(8, 64 << 20) == 1 << 19
    assert range_retain_hits(3, 12 * 3 * 32768) == 32768
    assert range_retain_hits(8, 1) == RANGE_MIN_HITS
    retain = 1 << 15
    # every rank's hits fit: one round, nothing given back
    assert range_capacity_plan([10, 4096, 0], 4096, retain) == (None, None)
    # one rank's do not: grow to the next power of two of the largest total, kept when within the retention
    assert range_capacity_plan([4097, 3], 4096, retain) == (8192, None)
    assert range_capacity_plan([20000, 18000], 4096, retain) == (32768, None)
    assert range_capacity_plan([20000, 18000], 32768, retain) == (None, None)  # the repeated call: one round
    # past the retention: grow, then give the excess back
    assert range_capacity_plan([5, 100000], 32768, retain) == (131072, 32768)
    # a small total never grows below the smallest inbox
    assert range_capacity_plan([1], 0, retain) == (RANGE_MIN_HITS, None)
    # the plan is a function of the replicated totals only: every rank computes the same
    assert len({range_capacity_plan(t, 4096, retain) for t in ([9000, 1],) * 3}) == 1


def _worker(rank, world, port):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        amp, exp = preset("coarse", 16)
        n = 301
        v, _, _ = dyadic_corpus(n, 16, 1, amp, exp, seed=7, dup=[(n - 1 - j, j) for j in range(0, 40, 3)])
        rng = np.random.default_rng(3)
        q = (rng.integers(-amp, amp + 1, size=(5, 16)) * 2.0 ** -exp).astype(np.float32)
        whole = lambda ms, ties=False: expected_range(exact_dots(q, v), ms, ties_low=ties)  # noqa: E731

        # exchange="peer": the peer route for more than one rank, the process group for one
        eng = PeerRangeEngine()
        sh = make(world, eng)
        sh.deserialize(v)
        peer = world > 1
        for ms, ties in ((0.5, False), (0.5, True), (0.0, False), (1.5, False)):
            assert_same(sh.search_range(q, ms, ties_low_first=ties), whole(ms, ties), f"W={world} ms={ms}")
        assert (len(eng.group_calls), eng.range_calls) == ((4, 0) if peer else (0, 4)), (eng.group_calls,
                                                                                          eng.range_calls)
        hits = sh.fuzzy_lookup_embedding(q[0], max_hits=0, min_score=0.5)
        o, i, s = whole(0.5)
        assert [(h.item, h.score) for h in hits] == list(zip(i[: o[1]].tolist(), s[: o[1]].tolist()))
        assert (len(eng.group_calls), eng.range_calls) == ((5, 0) if peer else (0, 5))

        # filtered threshold searches take the peer route with their local arguments
        if peer:
            eng.group_calls.clear()
            sh.search_range(q, 0.5, allowed=rng.random(n) < 0.5)
            sh.search_range(q, 0.5, subset=[0, n - 1, -1, 150, 150])
            sh.search_range(q, 0.5, subsets=[[0, 1], [], [n - 1], [150, 151, -3], [2]])
            assert eng.group_calls == [["mask", "mask_key", "mask_owner"], ["positions", "subset"],
                                       ["positions", "subsets"]], eng.group_calls

        # errors from replicated arguments: on every rank, before any collective and any engine call
        counting = CountingDist(dist)
        sh._dist = counting
        before = (len(eng.group_calls), eng.range_calls)
        for kw, err in ((dict(subset=[n]), IndexError), (dict(subset=[0], allowed=np.ones(n, bool)), ValueError),
                        (dict(allowed=np.ones(n - 1, bool)), ValueError),
                        (dict(allowed=np.ones((4, n), bool)), ValueError), (dict(subsets=[[0]] * 2), ValueError),
                        (dict(subsets=[[n]] * 5), IndexError)):
            with pytest.raises(err):
                sh.search_range(q, 0.5, **kw)
        with pytest.raises(ValueError):
            sh.search_range(q[:, :8], 0.5)
        assert counting.calls == 0 and (len(eng.group_calls), eng.range_calls) == before
        sh._dist = dist

        # exchange="nccl": the process-group route whatever the world
        eng2 = PeerRangeEngine()
        sh2 = make(world, eng2)
        sh2.exchange = "nccl"
        sh2.deserialize(v)
        assert_same(sh2.search_range(q, 0.5), whole(0.5), f"W={world} nccl")
        assert eng2.group_calls == [] and eng2.range_calls == 1
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [1, 2, 3])
def test_peer_range_routing_over_gloo(world):
    mp.spawn(_worker, args=(world, _free_port()), nprocs=world, join=True)


def _reserve_worker(rank, world, port):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from typeagent_py_b200.sharded import reserve_everywhere

        released = []

        def reserve(fail=None):
            def go():
                if fail is not None:
                    raise fail
                return bytes([rank]) * 4
            return go

        # every rank reserves: the handles in rank order, nothing released
        assert reserve_everywhere(dist, None, world, reserve(), lambda: released.append(1)) == \
            [bytes([r]) * 4 for r in range(world)]
        assert released == []
        # the last rank runs out of memory: MemoryError on every rank, and every rank releases its inbox
        last = rank == world - 1
        with pytest.raises(MemoryError):
            reserve_everywhere(dist, None, world, reserve(MemoryError("no room") if last else None),
                               lambda: released.append(1))
        assert released == [1]
        # another failure on one rank: its own error there, RuntimeError on the others
        with pytest.raises(ValueError if last else RuntimeError):
            reserve_everywhere(dist, None, world, reserve(ValueError("bad") if last else None),
                               lambda: released.append(2))
        assert released == [1, 2]
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [1, 2, 3])
def test_grow_agreement_over_gloo(world):
    mp.spawn(_reserve_worker, args=(world, _free_port()), nprocs=world, join=True)
