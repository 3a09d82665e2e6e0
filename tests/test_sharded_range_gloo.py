"""Host logic of the row-sharded threshold search on CPU: ``ShardedVectorBase.search_range`` and what is
routed to it, world sizes 1, 2 and 3 over the ``gloo`` backend, every result exact.

The engine is a numpy stand-in with ``CudaShardEngine``'s interface: ``range_local`` is the threshold search
of the rank's rows (``expected_range`` of their exact dots), ``merge_range`` a numpy merge that decodes the
product's packed all-gather layout (offsets and a status word per rank; items then scores, padded to the
largest rank's total).  What is under test is the product code around them (typeagent-py_b200/sharded.py):
the two exchanges, the padding, the SPMD early returns and failure handling, and the routing of
``max_hits=0`` lookups and of ``search_arrays`` with ``k >= rows > 8192``.  The CUDA engine
(``tav_range_search`` + ``tav_merge_range``) is covered by tests/test_gpu_sharded_range.py.
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

from tests.exact import dyadic_corpus, expected_topk, preset  # noqa: E402
from tests.test_gpu_range import expected_range  # noqa: E402
from tests.test_sharded_gloo import OracleShardEngine, _free_port  # noqa: E402


def exact_dots(q, v):
    """float32 dots of dyadic rows: exact in float64, so exact after the cast."""
    return (np.asarray(q, np.float64) @ np.asarray(v, np.float64).T).astype(np.float32)


class RangeEngine(OracleShardEngine):
    """CPU stand-in for CudaShardEngine's threshold search and merge (test infrastructure)."""

    def __init__(self, fail=False, fail_fetch=False):
        super().__init__()
        self.fail, self.fail_fetch = fail, fail_fetch
        self.range_calls = 0

    def comm_device(self):
        return torch.device("cpu")

    def search_packed(self, queries, k, min_score, item_offset):
        raise AssertionError("this lookup must be served by the threshold search")

    def range_local(self, queries, min_score, item_offset, ties_low_first):
        from typeagent_py_b200.sharded import LocalRange

        self.range_calls += 1
        if self.fail:
            raise RuntimeError("threshold search failed on this rank")
        b = len(queries)
        if len(self.rows) == 0:
            return LocalRange(np.zeros(b + 1, np.int64), None)
        offsets, items, scores = expected_range(exact_dots(queries, self.rows), min_score, ties_low=ties_low_first,
                                                item_offset=item_offset)

        def fetch(out_items, out_scores):
            if self.fail_fetch:
                raise MemoryError("staging the hits failed on this rank")
            np.asarray(out_items)[:] = items
            np.asarray(out_scores)[:] = scores

        return LocalRange(offsets, fetch)

    def merge_range(self, offsets_all, payload, world, n_queries, t_pad, total, ties_low_first):
        offs = offsets_all.numpy()
        pay = payload.numpy()
        out_o, out_i, out_s = [0], [], []
        for q in range(n_queries):
            its, scs = [], []
            for g in range(world):
                lo, hi = offs[g, q], offs[g, q + 1]
                its.append(pay[g, : 8 * t_pad].view(np.int64)[lo:hi])
                scs.append(pay[g, 8 * t_pad:].view(np.float32)[lo:hi])
            it, sc = np.concatenate(its), np.concatenate(scs)
            order = np.lexsort((it if ties_low_first else -it, -sc.view(np.uint32).astype(np.int64)))
            out_i.append(it[order])
            out_s.append(sc[order])
            out_o.append(out_o[-1] + len(order))
        assert out_o[-1] == total
        return (torch.from_numpy(np.array(out_o, np.int64)), torch.from_numpy(np.concatenate(out_i)),
                torch.from_numpy(np.concatenate(out_s)))


class CountingDist:
    """``torch.distributed`` as the object sees it, counting the collectives it enters."""

    def __init__(self, inner):
        self.inner, self.calls = inner, 0

    def __getattr__(self, name):
        fn = getattr(self.inner, name)
        if not callable(fn) or name.startswith("get_"):
            return fn

        def counted(*a, **k):
            self.calls += 1
            return fn(*a, **k)

        return counted


def assert_same(got, want, what):
    go, gi, gs = got
    wo, wi, ws = want
    np.testing.assert_array_equal(go, wo, err_msg=f"{what}: offsets")
    np.testing.assert_array_equal(gi, wi, err_msg=f"{what}: items")
    np.testing.assert_array_equal(gs.view(np.uint32), ws.view(np.uint32), err_msg=f"{what}: score bits")


def as_lists(csr):
    o, i, s = csr
    return [list(zip(i[o[b]:o[b + 1]].tolist(), s[o[b]:o[b + 1]].tolist())) for b in range(len(o) - 1)]


def make(world, engine=None):
    from types import SimpleNamespace

    from oracle import vectorbase_oracle as O
    from typeagent_py_b200.sharded import ShardedVectorBase

    settings = SimpleNamespace(embedding_model=O.FakeEmbeddingModel(), min_score=0.85, max_matches=None)
    return ShardedVectorBase(settings, engine=engine or RangeEngine())


def _worker(rank, world, port):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        # whole corpus, both tie orders, max_hits=0 lookups; heavy ties and duplicate rows in every block
        amp, exp = preset("coarse", 16)
        n = 301
        dup = [(n - 1 - j, j) for j in range(0, 40, 3)]  # copies of early rows near the end: equal scores across blocks
        v, q, _ = dyadic_corpus(n, 16, 5, amp, exp, seed=11, dup=dup)
        dots = exact_dots(q, v)
        sh = make(world)
        sh.deserialize(v)
        for ms in (0.0, 0.5, 0.75):
            for tl in (False, True):
                assert_same(sh.search_range(q, ms, ties_low_first=tl), expected_range(dots, ms, ties_low=tl),
                            f"rank {rank} ms {ms} ties_low {tl}")
            want = as_lists(expected_range(dots, ms))
            got = sh.fuzzy_lookup_embeddings(q, max_hits=0, min_score=ms)
            assert [[(h.item, h.score) for h in hits] for hits in got] == want
            assert [(h.item, h.score) for h in sh.fuzzy_lookup_embedding(q[2], max_hits=0, min_score=ms)] == want[2]

        # early returns on replicated state: no collective entered
        counting = CountingDist(sh._dist)
        sh._dist = counting
        o, i, s = sh.search_range(q, float("nan"))
        assert o.tolist() == [0] * 6 and len(i) == 0 and len(s) == 0
        o, i, s = sh.search_range(q[:0], 0.0)
        assert o.tolist() == [0] and len(i) == 0
        assert sh.fuzzy_lookup_embeddings(q, max_hits=0, min_score=float("nan")) == [[]] * 5
        empty = make(world)
        empty._dist = counting
        o, i, s = empty.search_range(q, 0.0)
        assert o.tolist() == [0] * 6 and len(i) == 0
        assert empty.fuzzy_lookup_embeddings(q, max_hits=0) == [[]] * 5
        # more ranks than one merge takes: ValueError on every rank, before any exchange
        sh.world = 33
        with pytest.raises(ValueError, match="at most 32"):
            sh.search_range(q, 0.0)
        sh.world = world
        assert counting.calls == 0, counting.calls
        sh._dist = counting.inner

        # appended rows live on the last rank and join the result
        extra = dyadic_corpus(23, 16, 1, amp, exp, seed=12)[0]
        sh.add_embeddings(None, extra)
        both = np.concatenate([v, extra])
        assert_same(sh.search_range(q, 0.25), expected_range(exact_dots(q, both), 0.25), f"rank {rank} appended")

        # fewer rows than ranks: the last rank(s) hold nothing but still join both exchanges
        tiny = make(world)
        tiny.deserialize(v[: world - 1] if world > 1 else v[:1])
        assert_same(tiny.search_range(q, 0.0), expected_range(exact_dots(q, v[: max(world - 1, 1)]), 0.0),
                    f"rank {rank} empty block")
        # load_local_shard with an empty block on the last rank
        from typeagent_py_b200.sharded import shard_bounds

        n2 = 2 if world == 3 else 1
        lo, hi = shard_bounds(n2, world)[rank]
        part = make(world)
        part.load_local_shard(v[lo:hi], n2)
        assert_same(part.search_range(q, 0.0), expected_range(exact_dots(q, v[:n2]), 0.0), f"rank {rank} local empty")

        # skew: rank 0's block holds nearly every hit, the others one row each: padding must not leak
        per = -(-n // world)
        sk = v.copy()
        d0 = exact_dots(q[:1], sk)[0]
        flip = np.where(np.arange(n) < per, d0 < 0, d0 > 0)
        sk[flip] = -sk[flip]
        for g in range(1, world):
            r = g * per
            if r < n and exact_dots(q[:1], sk[r:r + 1])[0, 0] < 0:
                sk[r] = -sk[r]
        sh2 = make(world)
        sh2.deserialize(sk)
        skd = exact_dots(q, sk)
        for ms in (0.5, 0.5000001):
            assert_same(sh2.search_range(q, ms), expected_range(skd, ms), f"rank {rank} skewed {ms}")

        # a failure on one rank raises on every rank, and nobody is left in a collective
        bad = make(world, RangeEngine(fail=(rank == world - 1)))
        bad.deserialize(v)
        with pytest.raises(RuntimeError):
            bad.search_range(q, 0.0)
        bad._engine.fail = False
        assert_same(bad.search_range(q, 0.5), expected_range(dots, 0.5), f"rank {rank} after a failure")
        # ... and so does a failure to stage the hits after the first exchange (an allocation or the fetch)
        if world > 1:
            bad._engine.fail_fetch = rank == 0
            with pytest.raises((MemoryError, RuntimeError)):
                bad.search_range(q, 0.0)
            bad._engine.fail_fetch = False
            assert_same(bad.search_range(q, 0.5), expected_range(dots, 0.5), f"rank {rank} after a staging failure")
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [1, 2, 3])
def test_sharded_search_range_over_gloo(world):
    mp.spawn(_worker, args=(world, _free_port()), nprocs=world, join=True)


def _routing_worker(rank, world, port):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        # search_arrays with k >= rows > 8192 is one threshold search laid out [B, rows] (search_packed raises)
        amp, exp = preset("fine", 8)
        n = 8200
        v, q, dots = dyadic_corpus(n, 8, 3, amp, exp, seed=5)
        sh = make(world)
        sh.deserialize(v)
        for k, ms in ((n, 0.5), (n + 7, 0.0)):
            items, scores, counts = sh.search_arrays(q, k, ms)
            wi, ws, wc = expected_topk(dots, n, ms)
            np.testing.assert_array_equal(counts, wc)
            np.testing.assert_array_equal(items, wi)
            np.testing.assert_array_equal(scores.view(np.uint32), ws.view(np.uint32))
        got = sh.fuzzy_lookup_embeddings(q, max_hits=n, min_score=0.5)
        assert [[(h.item, h.score) for h in hits] for hits in got] == as_lists(expected_range(dots, 0.5))
        assert sh._engine.range_calls >= 2
        # at or below 8192 rows the top-k exchange keeps serving k >= rows
        small = make(world)
        small.deserialize(v[:8192])
        with pytest.raises(AssertionError, match="threshold search"):
            small.search_arrays(q, 8192, 0.0)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_search_arrays_routing_over_gloo(world):
    mp.spawn(_routing_worker, args=(world, _free_port()), nprocs=world, join=True)
