"""Host logic of ``ShardedVectorBase.rebalance`` on CPU, world sizes 1, 2 and 3 over ``gloo``.

The engine is the numpy stand-in of the sharded lookup tests (tests/test_sharded_filter_gloo.py and the per-query
mask and subsets variants, exact on dyadic corpora) plus ``CudaShardEngine``'s rebalance steps: a rank's exported
record carries its rows (standing in for the IPC mapping of its allocation), staging lays the plan's pieces out in
order, and commit swaps them in.  Under test is the product code around them (typeagent-py_b200/sharded.py): the
target blocks, the plan, the protocol's collectives and their agreement on failure, the float32 mirror exchange
over the process group, the row generation, and ``rebalance_at``.

Appends skew the last block and removals empty one; after ``rebalance()`` the blocks equal ``shard_bounds``, and
every lookup kind equals a numpy statement of one ``VectorBase`` over the whole corpus before and after: plain,
predicate, 1-D and 2-D ``allowed=``, ``subset=``, ``subsets=``, ``search_range``, both tie orders.
"""

from __future__ import annotations

import os
import sys

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.exact import dyadic_corpus, preset  # noqa: E402
from tests.test_sharded_filter_gloo import CountingDist, _pack, make, oracle_arrays, oracle_csr, oracle_lists  # noqa: E402
from tests.test_sharded_filter_gloo import same_arrays, same_csr  # noqa: E402
from tests.test_sharded_gloo import DeferringOracleEngine, _free_port  # noqa: E402
from tests.test_sharded_query_masks_gloo import QueryMaskEngine, as_arrays, per_query  # noqa: E402
from tests.test_sharded_range_gloo import exact_dots  # noqa: E402
from tests.test_sharded_subsets_gloo import SubsetsEngine, oracle_batch_arrays  # noqa: E402

D = 16


class RebalanceSteps:
    """CudaShardEngine's rebalance steps on numpy rows (test infrastructure).  ``rows`` is the host mirror and
    ``device_rows`` what the device would hold; ``readback``: the mirror is read back from the staged rows (float32
    storage) instead of exchanged; ``fail_stage``: staging raises MemoryError on this rank."""

    adopted = False
    readback = False
    fail_stage = False

    def rows_adopted(self):
        return self.adopted

    def rows_export(self):
        self.exports = getattr(self, "exports", 0) + 1
        return np.array(self.rows, np.float32)  # the peers' "mapping" of this rank's rows

    def mirror_from_rows(self):
        return self.readback

    def local_rows(self):
        return self.rows

    def rows_stage(self, records, pieces, rank, dim):
        if self.fail_stage:
            raise MemoryError("cannot allocate the new block on this rank")
        parts = [(self.rows if src == rank else records[src])[first: first + n] for src, first, n in pieces]
        self.staged = np.concatenate(parts) if parts else np.zeros((0, dim), np.float32)
        return self.staged.copy() if self.readback else None

    def rows_commit(self, commit, mirror=None):
        staged, self.staged = getattr(self, "staged", None), None
        self.commits = getattr(self, "commits", []) + [bool(commit)]
        if commit:
            self.device_rows = staged
            self.rows = mirror


class RebalanceEngine(RebalanceSteps, SubsetsEngine, QueryMaskEngine):
    def search_packed(self, queries, k, min_score, item_offset):
        lists = oracle_lists(exact_dots(queries, self.rows), min_score) if len(self.rows) else [[]] * len(queries)
        return _pack(len(queries), k, [[(it + item_offset, sc) for it, sc in h] for h in lists])


class DeferringRebalanceEngine(RebalanceSteps, DeferringOracleEngine):
    pass


# ---------------------------------------------------------------- every lookup kind, and its oracle
def lookups(sh, q, k, ms, masks1, masks2, sub, subs, pred):
    out = {
        "plain": sh.search_arrays(q, k, ms),
        "ties_low": sh.search_arrays(q, k, ms, ties_low_first=True),
        "allowed": sh.search_arrays(q, k, ms, allowed=masks1),
        "allowed_2d": sh.search_arrays(q, k, ms, allowed=masks2, ties_low_first=True),
        "subset": sh.search_arrays(q, k, ms, subset=sub),
        "subsets": sh.search_arrays(q, k, ms, subsets=subs),
        "range": sh.search_range(q, ms),
        "range_low": sh.search_range(q, ms, ties_low_first=True),
        "range_subset": sh.search_range(q, ms, subset=sub),
    }
    out["predicate"] = [[(h.item, h.score) for h in sh.fuzzy_lookup_embedding(qq, k, ms, predicate=pred)] for qq in q]
    return out


def oracle(v, q, k, ms, masks1, masks2, sub, subs, pred):
    dots = exact_dots(q, v)
    n = len(v)
    kk = max(1, min(k, n))
    pmask = np.array([bool(pred(i)) for i in range(n)])
    return {
        "plain": oracle_arrays(dots, kk, ms),
        "ties_low": oracle_arrays(dots, kk, ms, ties_low=True),
        "allowed": oracle_arrays(dots, kk, ms, allowed=masks1),
        "allowed_2d": as_arrays(per_query(dots, ms, masks2, ties_low=True), kk),
        "subset": oracle_arrays(dots, max(1, min(k, len(sub))), ms, subset=sub),
        "subsets": oracle_batch_arrays(dots, k, ms, subs),
        "range": oracle_csr(dots, ms),
        "range_low": oracle_csr(dots, ms, ties_low=True),
        "range_subset": oracle_csr(dots, ms, subset=sub),
        "predicate": [oracle_lists(dots[b:b + 1], ms, allowed=pmask, ties_low=True)[0][:k] for b in range(len(q))],
    }


def check_all(sh, engine, v, q, rng, what):
    """Every lookup kind against the oracle over ``v``; each rank's rows (host mirror and device copy) are its
    block of ``v``."""
    lo, hi = sh.local_range
    np.testing.assert_array_equal(np.asarray(engine.rows).reshape(-1, D), v[lo:hi], err_msg=what)
    if getattr(engine, "device_rows", None) is not None:
        np.testing.assert_array_equal(engine.device_rows.reshape(-1, D), v[lo:hi], err_msg=what)
    n = len(v)
    masks1 = rng.random(n) < 0.5
    masks2 = rng.random((len(q), n)) < 0.6
    sub = np.concatenate([rng.permutation(n)[: n // 3], [0, n - 1, -1, 0]]).astype(np.int64)
    subs = [rng.permutation(n)[: 30], np.array([n - 1, 0, -2, n - 1]), np.arange(n)[::-3]][: len(q)]
    pred = lambda i: i % 3 != 1  # noqa: E731
    for k, ms in ((7, 0.0), (40, 0.45)):
        got = lookups(sh, q, k, ms, masks1, masks2, sub, subs, pred)
        want = oracle(v, q, k, ms, masks1, masks2, sub, subs, pred)
        for name in got:
            tag = f"{what}: {name} k {k} ms {ms}"
            if name.startswith("range"):
                same_csr(got[name], want[name], tag)
            elif name == "predicate":
                assert got[name] == want[name], tag
            else:
                same_arrays(got[name], want[name], tag)


def _worker(rank, world, port, readback):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from typeagent_py_b200.sharded import shard_bounds

        amp, exp = preset("coarse", D)
        n0 = 90
        # equal rows on both sides of every later block boundary
        v, q, _ = dyadic_corpus(n0 + 150, D, 3, amp, exp, seed=31, dup=[(n0 + 140 - j, j) for j in range(0, 30, 3)])
        engine = RebalanceEngine()
        engine.readback = readback
        sh = make(engine)
        sh._dist = CountingDist(dist)
        rng = np.random.default_rng(7)
        sh.deserialize(v[:n0])
        cur = v[:n0]
        assert sh.rebalance() == 0 and sh._dist.calls == 0  # already even: no collective
        # skew the last block with appends, empty the first block with a removal
        for lo, hi in ((n0, n0 + 60), (n0 + 60, n0 + 150)):
            sh.add_embeddings(None, v[lo:hi])
            cur = v[:hi]
        gone = np.arange(*sh.blocks[0]) if world > 1 else np.arange(30)
        sh.remove_embeddings(gone)
        cur = np.delete(cur, gone, axis=0)
        if world > 1:
            assert sh.blocks[0] == (0, 0) and sh.blocks[-1][1] - sh.blocks[-1][0] > len(cur) // 2
        check_all(sh, engine, cur, q, rng, f"rank {rank} skewed")
        gen = sh._generation
        calls = sh._dist.calls
        want_moved = sum(a != b for a, b in zip(
            np.searchsorted([s for s, _ in sh.blocks][1:], np.arange(len(cur)), side="right"),
            np.searchsorted([s for s, _ in shard_bounds(len(cur), world)][1:], np.arange(len(cur)), side="right")))
        moved = sh.rebalance()
        assert moved == want_moved, (moved, want_moved)
        assert sh.blocks == shard_bounds(len(cur), world)
        assert sh._generation == gen + (world > 1)
        if world > 1:
            # one all_gather_object of the records, then one status word (a second before the mirror exchange,
            # and the exchange itself, when the mirror is not read back)
            assert sh._dist.calls - calls == (2 if readback else 4), sh._dist.calls - calls
        check_all(sh, engine, cur, q, rng, f"rank {rank} rebalanced")
        assert sh.rebalance() == 0

        # sizes=: everything on the middle (or only) rank, then one row each and the rest on the last
        sizes = [0] * world
        sizes[world // 2] = len(cur)
        sh.rebalance(sizes)
        assert [hi - lo for lo, hi in sh.blocks] == sizes
        check_all(sh, engine, cur, q, rng, f"rank {rank} sizes {sizes}")
        sizes = [1] * (world - 1) + [len(cur) - (world - 1)]
        sh.rebalance(np.array(sizes))
        assert [hi - lo for lo, hi in sh.blocks] == sizes
        check_all(sh, engine, cur, q, rng, f"rank {rank} sizes {sizes}")

        # invalid sizes: ValueError on every rank, no collective, nothing changed
        calls, blocks = sh._dist.calls, sh.blocks
        for bad in ([len(cur) + 1] * world, [1] * (world + 1), [-1] + [0] * (world - 2) + [len(cur) + 1], [0.5] * world):
            with pytest.raises(ValueError):
                sh.rebalance(bad)
        assert sh._dist.calls == calls and sh.blocks == blocks

        if world > 1:
            # a stage that fails on one rank: every rank raises, nothing changed anywhere
            engine.fail_stage = rank == world - 1
            rows_before = engine.rows.copy()
            with pytest.raises(MemoryError):
                sh.rebalance()
            assert sh.blocks == blocks and engine.commits[-1] is False
            np.testing.assert_array_equal(engine.rows, rows_before)
            check_all(sh, engine, cur, q, rng, f"rank {rank} after a failed stage")
            engine.fail_stage = False
            # a rank with adopted rows: refused on every rank before anything is staged
            engine.adopted = rank == 0
            exports = engine.exports
            with pytest.raises(RuntimeError, match="adopted"):
                sh.rebalance()
            assert sh.blocks == blocks and engine.exports == exports + (rank != 0)
            engine.adopted = False
            assert sh.rebalance() > 0 and sh.blocks == shard_bounds(len(cur), world)
            check_all(sh, engine, cur, q, rng, f"rank {rank} after the refusals")
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("readback", [False, True], ids=["mirror_exchanged", "mirror_read_back"])
@pytest.mark.parametrize("world", [1, 2, 3])
def test_rebalance_over_gloo(world, readback):
    mp.spawn(_worker, args=(world, _free_port(), readback), nprocs=world, join=True)


def _threshold_worker(rank, world, port):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from types import SimpleNamespace

        from oracle import vectorbase_oracle as O
        from typeagent_py_b200.sharded import ShardedVectorBase, shard_bounds

        settings = SimpleNamespace(embedding_model=O.FakeEmbeddingModel(), min_score=0.85, max_matches=None)
        engine = RebalanceEngine()
        with pytest.raises(ValueError):
            ShardedVectorBase(settings, engine=engine, rebalance_at=0.9)
        sh = ShardedVectorBase(settings, engine=engine, rebalance_at=1.5)
        amp, exp = preset("coarse", D)
        v, q, _ = dyadic_corpus(400, D, 2, amp, exp, seed=5)
        n = 60 * world
        sh.deserialize(v[:n])
        # the last block may hold 1.5 * (rows / world) rows: appends up to that bound leave the blocks alone
        last = shard_bounds(n, world)[-1]
        size = last[1] - last[0]
        m = 0
        while world > 1 and (size + m + 1) * world <= 1.5 * (n + m + 1):
            m += 1
        if world > 1:
            sh.add_embeddings(None, v[n: n + m])
            assert sh.blocks[-1] == (last[0], n + m), "rebalanced below the threshold"
            sh.add_embeddings(None, v[n + m: n + m + 1])  # one row more: above it
            assert sh.blocks == shard_bounds(n + m + 1, world)
            cur = v[: n + m + 1]
            # a removal that empties the first block (and takes the last row) rebalances too
            gone = np.append(np.arange(*sh.blocks[0]), len(cur) - 1)
            sh.remove_embeddings(gone)
            cur = np.delete(cur, gone, axis=0)
            assert sh.blocks == shard_bounds(len(cur), world)
        else:
            sh.add_embeddings(None, v[n: n + 50])  # one rank always holds everything: never above 1.5x
            cur = v[: n + 50]
            assert sh.blocks == [(0, len(cur))]
        check_all(sh, engine, cur, q, np.random.default_rng(3), f"rank {rank} rebalance_at")
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [1, 2, 3])
def test_rebalance_at_fires_exactly_above_its_threshold(world):
    mp.spawn(_threshold_worker, args=(world, _free_port()), nprocs=world, join=True)


def _deferred_worker(rank, world, port):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from types import SimpleNamespace

        from oracle import vectorbase_oracle as O
        from typeagent_py_b200.sharded import ShardedVectorBase, shard_bounds

        v, q = O.make_corpus(150, D, seed=14, n_queries=3)
        settings = SimpleNamespace(embedding_model=O.FakeEmbeddingModel(), min_score=0.85, max_matches=None)
        engine = DeferringRebalanceEngine(rank, spoil_ranks=set(range(world)))
        sh = ShardedVectorBase(settings, engine=engine)
        sh.deserialize(v[:60])
        sh.add_embeddings(None, v[60:])
        k = 6
        items, scores, counts = sh.search_tensors(q, k, 0.0, defer_check=True)
        assert sh.rebalance() > 0 and sh.blocks == shard_bounds(150, world)
        assert not engine.fixups and sh.finish() == 0  # the rebalance finished the lookup first
        for b in range(len(q)):
            want = O.lookup(v, q[b], k, 0.0)
            assert int(counts[b]) == len(want), (rank, b)
            assert items[b, :len(want)].tolist() == [h.item for h in want], (rank, b)
        got = sh.fuzzy_lookup_embeddings(q, k, 0.0)
        assert [[h.item for h in hits] for hits in got] == [[h.item for h in O.lookup(v, qq, k, 0.0)] for qq in q]
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_deferred_lookup_before_a_rebalance_is_merged_first(world):
    """A deferred lookup whose candidates every rank corrects at finish, then a rebalance: the rebalance finishes
    the lookup first, so its corrected candidates are exchanged and merged again before any row moves."""
    mp.spawn(_deferred_worker, args=(world, _free_port()), nprocs=world, join=True)
