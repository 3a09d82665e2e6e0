"""Host logic of per-query masks (2-D ``allowed=``) on ``ShardedVectorBase``, on CPU over ``gloo`` with worlds 1, 2
and 3, through the numpy stand-in engine of tests/test_sharded_filter_gloo.py.

What is under test is the product code in typeagent-py_b200/sharded.py: each rank cuts its block's columns out of
every query's mask (blocks that do not start on a 32-row word included), the filtered exchange and the threshold
exchange finish the job, every argument error is raised on every rank before any collective, and a local
failure raises on every rank.  Results are compared with one-process ``VectorBase`` semantics, query by query.
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
from tests.test_sharded_filter_gloo import (CountingDist, FilterEngine, _pack, make, oracle_lists,  # noqa: E402
                                            same_arrays, same_csr)
from tests.test_sharded_gloo import _free_port  # noqa: E402
from tests.test_sharded_range_gloo import exact_dots  # noqa: E402


def per_query(dots, min_score, masks, ties_low=False):
    """oracle_lists with query b restricted to masks[b]."""
    return [oracle_lists(dots[b:b + 1], min_score, allowed=masks[b], ties_low=ties_low)[0] for b in range(len(dots))]


def as_arrays(lists, k):
    b = len(lists)
    items = np.full((b, k), -1, np.int64)
    scores = np.zeros((b, k), np.float32)
    counts = np.zeros(b, np.int32)
    for i, hits in enumerate(lists):
        hits = hits[:k]
        counts[i] = len(hits)
        for j, (it, sc) in enumerate(hits):
            items[i, j], scores[i, j] = it, sc
    return items, scores, counts


def as_csr(lists):
    offsets = np.cumsum([0] + [len(h) for h in lists]).astype(np.int64)
    return (offsets, np.array([it for h in lists for it, _ in h], np.int64),
            np.array([sc for h in lists for _, sc in h], np.float32))


class QueryMaskEngine(FilterEngine):
    """FilterEngine whose per-rank steps also take a 2-D mask (this block's words, one row per query)."""

    def _query_bits(self, mask):
        return np.unpackbits(np.asarray(mask, np.uint32).view(np.uint8), axis=1,
                             bitorder="little")[:, : len(self.rows)].astype(bool)

    def search_rows_packed(self, queries, k, min_score, item_offset, ties_low_first, mask=None, mask_key=None,
                           mask_owner=None):
        if mask is None or np.ndim(mask) != 2:
            return super().search_rows_packed(queries, k, min_score, item_offset, ties_low_first, mask, mask_key,
                                              mask_owner)
        b = len(queries)
        if self.fail_topk:
            raise MemoryError("the local search failed on this rank")
        assert mask.shape[0] == b
        if len(self.rows) == 0:
            return _pack(b, k, [[]] * b)
        self.mask_uploads.append(id(mask))
        lists = per_query(exact_dots(queries, self.rows), min_score, self._query_bits(mask), ties_low_first)
        return _pack(b, k, [[(it + item_offset, sc) for it, sc in h] for h in lists])

    def range_local(self, queries, min_score, item_offset, ties_low_first, mask=None, mask_key=None,
                    mask_owner=None, subset=None, positions=None):
        from typeagent_py_b200.sharded import LocalRange

        if mask is None or np.ndim(mask) != 2:
            return super().range_local(queries, min_score, item_offset, ties_low_first, mask, mask_key, mask_owner,
                                       subset, positions)
        self.range_calls += 1
        b = len(queries)
        if len(self.rows) == 0:
            return LocalRange(np.zeros(b + 1, np.int64), None)
        self.mask_uploads.append(id(mask))
        offsets, items, scores = as_csr(per_query(exact_dots(queries, self.rows), min_score, self._query_bits(mask),
                                                  ties_low_first))
        items = items + item_offset

        def fetch(out_items, out_scores):
            np.asarray(out_items)[:] = items
            np.asarray(out_scores)[:] = scores

        return LocalRange(offsets, fetch)


def _worker(rank, world, port):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from typeagent_py_b200.vectorbase import VectorBase

        amp, exp = preset("coarse", 16)
        n = 301  # blocks start at 151 (W = 2) and at 101, 201 (W = 3): not on a 32-row word
        dup = [(n - 1 - j, j) for j in range(0, 40, 3)] + [(150 + j, j) for j in range(0, 20, 2)]
        v, q, _ = dyadic_corpus(n, 16, 6, amp, exp, seed=19, dup=dup)
        dots = exact_dots(q, v)
        rng = np.random.default_rng(7)
        masks = np.zeros((len(q), n), bool)
        for b, dens in enumerate([1.0, 0.5, 0.05, 0.0, 0.3, 0.8]):
            masks[b] = rng.random(n) < dens
        masks[1, [j for j, _ in dup]] = True       # equal scores in different blocks
        masks[4, [0, 100, 101, 150, 151, 200, 201, 300]] = True   # block edges
        sh = make(QueryMaskEngine())
        sh.deserialize(v)

        # ---- bool and packed masks, both tie orders, top-k and threshold searches
        words = VectorBase.pack_query_masks(masks)
        for mask in (masks, words):
            for tl in (False, True):
                for ms in (0.0, 0.55):
                    for k in (1, 7, n):
                        same_arrays(sh.search_arrays(q, k, ms, allowed=mask, ties_low_first=tl),
                                    as_arrays(per_query(dots, ms, masks, tl), min(k, n)),
                                    f"rank {rank} {mask.dtype} tl {tl} ms {ms} k {k}")
                    same_csr(sh.search_range(q, ms, ties_low_first=tl, allowed=mask),
                             as_csr(per_query(dots, ms, masks, tl)), f"rank {rank} range {mask.dtype} {tl} {ms}")

        # ---- one query, one mask row
        same_arrays(sh.search_arrays(q[2:3], 5, 0.0, allowed=masks[2:3]), as_arrays(per_query(dots[2:3], 0.0, masks[2:3]), 5),
                    f"rank {rank} one query")

        # ---- one cut per mask object and rows; the engine is handed the same words every time
        sh._engine.mask_uploads.clear()
        for _ in range(3):
            sh.search_arrays(q, 5, 0.0, allowed=masks)
        assert len(set(sh._engine.mask_uploads)) <= 1

        # ---- errors on every rank, before any collective
        counting = CountingDist(sh._dist)
        sh._dist = counting
        with pytest.raises(ValueError, match=f"query masks have 5 rows for {len(q)} queries"):
            sh.search_arrays(q, 5, 0.0, allowed=masks[:5])
        with pytest.raises(ValueError, match=f"query masks have 5 rows for {len(q)} queries"):
            sh.search_range(q, 0.5, allowed=masks[:5])
        with pytest.raises(ValueError, match=f"query masks have {n - 1} entries for {n} rows"):
            sh.search_arrays(q, 5, 0.0, allowed=masks[:, 1:])
        with pytest.raises(ValueError, match=f"query masks have {32 * 9} bits for {n} rows"):
            sh.search_range(q, 0.5, allowed=np.zeros((len(q), 9), np.uint32))
        with pytest.raises(ValueError, match="cannot be combined"):
            sh.search_arrays(q, 5, 0.0, allowed=masks, subset=[1, 2])
        with pytest.raises(ValueError, match="one mask per query"):
            sh.search_arrays(q, 5, 0.0, allowed=np.ones((len(q), n, 1), bool))
        assert counting.calls == 0
        sh._dist = counting.inner

        # ---- a local failure on one rank raises on every rank
        sh._engine.fail_topk = rank == world - 1
        with pytest.raises((MemoryError, RuntimeError)):
            sh.search_arrays(q, 5, 0.0, allowed=masks)
        sh._engine.fail_topk = False
        same_arrays(sh.search_arrays(q, 5, 0.0, allowed=masks), as_arrays(per_query(dots, 0.0, masks), 5),
                    f"rank {rank} after a failure")
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [1, 2, 3])
def test_per_query_masks_over_gloo(world):
    mp.spawn(_worker, args=(world, _free_port()), nprocs=world, join=True)


def test_block_mask_cuts_every_querys_columns():
    from typeagent_py_b200.sharded import block_mask
    from typeagent_py_b200.vectorbase import VectorBase

    rng = np.random.default_rng(3)
    for n in (1, 31, 32, 33, 301, 1000):
        masks = rng.random((4, n)) < 0.5
        words = VectorBase.pack_query_masks(masks)
        for lo, hi in ((0, n), (0, n // 2), (n // 3, n), (n // 3, 2 * n // 3 + 1), (n, n)):
            want = VectorBase.pack_query_masks(masks[:, lo:hi])
            np.testing.assert_array_equal(block_mask(masks, n, lo, hi, 4), want)
            np.testing.assert_array_equal(block_mask(words, n, lo, hi, 4), want)
            for b in range(4):  # each row is the 1-D cut of that query's mask
                np.testing.assert_array_equal(block_mask(masks, n, lo, hi, 4)[b], block_mask(masks[b], n, lo, hi))
    with pytest.raises(ValueError, match="3 rows for 4 queries"):
        block_mask(np.ones((3, 10), bool), 10, 0, 5, 4)
