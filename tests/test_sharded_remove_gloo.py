"""Host logic of ``ShardedVectorBase.remove_embeddings`` on CPU, over ``gloo`` with worlds 1, 2 and 3.

Every rank passes the same global ordinals; each removes its own block's share and recomputes the block starts
from the replicated list, without a collective.  The engine is the numpy stand-in of tests/test_sharded_gloo.py
with a ``remove_rows``.  After every step each rank's rows must be exactly its block of
``np.delete(corpus, removed)`` and every lookup must equal the oracle's over that array: removals inside one
block, spanning blocks, emptying a block, negative and repeated ordinals, appends after a removal, and
everything removed.
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

from tests.test_sharded_gloo import DeferringOracleEngine, OracleShardEngine, _free_port  # noqa: E402


class RemovingOracleEngine(OracleShardEngine):
    def __init__(self):
        super().__init__()
        self.removals = []  # local ordinals of every remove_rows call

    def remove_rows(self, local_ordinals):
        self.removals.append(np.asarray(local_ordinals).tolist())
        self.rows = np.delete(self.rows, local_ordinals, axis=0)


def removal_steps(n):
    """(ordinals, what) in order, against a corpus of n rows at the start."""
    return [
        ([], "nothing"),
        ([0], "the first row"),
        ([-1], "the last row, negative"),
        ([5, 5, 3, -2, 3], "repeated and negative, unordered"),
        (list(range(n // 3 - 4, n // 3 + 4)), "a run across the first block boundary"),
        (list(range(1, n // 2, 2)), "every other row of the first half"),
    ]


def check(sh, engine, corpus, q, rank, what):
    from oracle import vectorbase_oracle as O

    assert len(sh) == len(corpus), what
    lo, hi = sh.local_range
    assert sh._starts[0] == 0 and all(a <= b for a, b in zip(sh._starts, sh._starts[1:])), (what, sh._starts)
    np.testing.assert_array_equal(engine.rows.reshape(-1, corpus.shape[1]) if len(engine.rows) else
                                  np.zeros((0, corpus.shape[1]), np.float32), corpus[lo:hi], err_msg=what)
    if len(corpus) == 0:
        assert sh.fuzzy_lookup_embedding(q[0]) == []
        return
    for k, ms in ((7, 0.0), (len(corpus) + 3, 0.4)):
        got = sh.fuzzy_lookup_embeddings(q, k, ms)
        for qq, hits in zip(q, got):
            want = O.lookup(corpus, qq, k, ms)
            assert [h.item for h in hits] == [h.item for h in want], (rank, what, k, ms)


def _worker(rank: int, world: int, port: int, n_rows: int):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from types import SimpleNamespace

        from oracle import vectorbase_oracle as O
        from typeagent_py_b200.sharded import ShardedVectorBase, shard_bounds

        v, q = O.make_corpus(n_rows, 16, seed=11, n_queries=4)
        settings = SimpleNamespace(embedding_model=O.FakeEmbeddingModel(), min_score=0.85, max_matches=None)
        engine = RemovingOracleEngine()
        sh = ShardedVectorBase(settings, engine=engine)
        sh.deserialize(v)
        corpus = v.copy()
        for ordinals, what in removal_steps(n_rows):
            sh.remove_embeddings(ordinals)
            corpus = np.delete(corpus, ordinals, axis=0)
            check(sh, engine, corpus, q, rank, what)

        # out of range: IndexError on every rank, nothing removed anywhere
        calls, starts = len(engine.removals), list(sh._starts)
        for bad in ([len(corpus)], [0, -len(corpus) - 1], np.array([0.5])):
            with pytest.raises(IndexError):
                sh.remove_embeddings(bad)
        assert len(engine.removals) == calls and sh._starts == starts

        # empty one rank's block entirely (the middle one when there is one), then append after the removal
        lo, hi = sh._starts[world // 2], sh._starts[world // 2 + 1]
        sh.remove_embeddings(np.arange(lo, hi))
        corpus = np.delete(corpus, np.arange(lo, hi), axis=0)
        assert sh._starts[world // 2] == sh._starts[world // 2 + 1]
        check(sh, engine, corpus, q, rank, "an emptied block")
        extra = O.make_corpus(9, 16, seed=12)[0]
        sh.add_embeddings(None, extra)
        corpus = np.concatenate([corpus, extra])
        check(sh, engine, corpus, q, rank, "appended after removals")
        # 1% and 50% at random, the same draw on every rank
        rng = np.random.default_rng(13)
        for frac in (0.01, 0.5):
            pick = rng.choice(len(corpus), max(1, int(frac * len(corpus))), replace=False)
            sh.remove_embeddings(pick)
            corpus = np.delete(corpus, pick, axis=0)
            check(sh, engine, corpus, q, rank, f"random {frac}")
        sh.remove_embeddings(np.arange(-len(corpus), 0))
        check(sh, engine, corpus[:0], q, rank, "every row")
        assert sh._starts == [0] * (world + 1)
        assert shard_bounds(0, world) == [(0, 0)] * world
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,n_rows", [(1, 90), (2, 301), (3, 200)])
def test_sharded_remove_over_gloo(world, n_rows):
    mp.spawn(_worker, args=(world, _free_port(), n_rows), nprocs=world, join=True)


class DeferringRemovingEngine(DeferringOracleEngine):
    """The deferred exact fallback as the library has it: a removal first puts the real candidates of the
    outstanding searches in place (tav_remove_rows finishes them) and reports nothing, so a later finish() of the
    engine counts 0."""

    def remove_rows(self, local_ordinals):
        for counts, real in self.fixups:
            counts[0] = real
        self.fixups.clear()
        self.rows = np.delete(self.rows, local_ordinals, axis=0)


def _deferred_worker(rank: int, world: int, port: int):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from types import SimpleNamespace

        from oracle import vectorbase_oracle as O
        from typeagent_py_b200.sharded import ShardedVectorBase

        v, q = O.make_corpus(120, 16, seed=14, n_queries=3)
        settings = SimpleNamespace(embedding_model=O.FakeEmbeddingModel(), min_score=0.85, max_matches=None)
        sh = ShardedVectorBase(settings, engine=DeferringRemovingEngine(rank, spoil_ranks=set(range(world))))
        sh.deserialize(v)
        k = 6
        items, scores, counts = sh.search_tensors(q, k, 0.0, defer_check=True)
        sh.remove_embeddings(np.arange(0, 120, 7))  # rows of every rank
        sh.finish()
        for b in range(len(q)):
            want = O.lookup(v, q[b], k, 0.0)  # the search ran before the removal: the old rows
            assert int(counts[b]) == len(want), (rank, b)
            assert items[b, :len(want)].tolist() == [h.item for h in want], (rank, b)
        rows = np.delete(v, np.arange(0, 120, 7), axis=0)
        got = sh.fuzzy_lookup_embeddings(q, k, 0.0)
        assert [[h.item for h in hits] for hits in got] == [[h.item for h in O.lookup(rows, qq, k, 0.0)] for qq in q]
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [1, 2, 3])
def test_deferred_lookup_before_a_removal_is_merged_again(world):
    """A deferred lookup whose candidates every rank corrects, then a removal: the removal finishes the lookup
    first, so the corrected candidates are exchanged and merged again."""
    mp.spawn(_deferred_worker, args=(world, _free_port()), nprocs=world, join=True)
