"""Host logic of row-sharded per-query subsets (``subsets=``) on CPU, world sizes 1, 2 and 3 over ``gloo``.

The engine is the numpy stand-in of tests/test_sharded_filter_gloo.py plus ``CudaShardEngine``'s subsets steps
(``search_subsets_packed``, ``range_local(subsets=)``), following the library's semantics exactly on dyadic
corpora.  Under test is the product code around them (typeagent-py_b200/sharded.py): the split of every query's
subset into per-rank CSR shares, the exchanges, the merge by flat position and the decode, and the SPMD errors.
Every result is compared with a numpy statement of one-process ``VectorBase`` semantics over the whole corpus.
The CUDA side is covered by tests/test_gpu_sharded_subsets.py.
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
from tests.test_sharded_filter_gloo import (  # noqa: E402
    CountingDist, FilterEngine, _pack, hits, make, oracle_arrays, oracle_csr, oracle_lists, same_arrays, same_csr)
from tests.test_sharded_gloo import _free_port  # noqa: E402
from tests.test_sharded_range_gloo import exact_dots  # noqa: E402


class SubsetsEngine(FilterEngine):
    """FilterEngine plus the per-query subsets steps (test infrastructure): items are flat positions in the
    rank's share, mapped through ``positions`` to flat positions in the caller's ordinals."""

    def _lists(self, queries, min_score, local_offsets, local_ordinals, ties_low_first):
        dots = exact_dots(queries, self.rows)
        out = []
        for b in range(len(queries)):
            lo, hi = int(local_offsets[b]), int(local_offsets[b + 1])
            seg = np.asarray(local_ordinals[lo:hi], np.int64)
            lst = oracle_lists(dots[b:b + 1, seg], min_score, ties_low=ties_low_first)[0] if hi > lo else []
            out.append([(lo + it, sc) for it, sc in lst])
        return out

    def search_subsets_packed(self, queries, k, min_score, local_offsets, local_ordinals, positions, ties_low_first):
        b = len(queries)
        if self.fail_topk:
            raise MemoryError("the local search failed on this rank")
        if len(local_ordinals) == 0:
            return _pack(b, k, [[]] * b)
        buf = _pack(b, k, self._lists(queries, min_score, local_offsets, local_ordinals, ties_low_first))
        self.map_items(buf[: b * k * 8].view(torch.int64), positions)
        return buf

    def range_local(self, queries, min_score, item_offset, ties_low_first, mask=None, mask_key=None,
                    mask_owner=None, subset=None, positions=None, subsets=None):
        from typeagent_py_b200.sharded import LocalRange

        if subsets is None:
            return super().range_local(queries, min_score, item_offset, ties_low_first, mask, mask_key, mask_owner,
                                       subset, positions)
        self.range_calls += 1
        b = len(queries)
        if len(self.rows) == 0 or len(subsets[1]) == 0:
            return LocalRange(np.zeros(b + 1, np.int64), None)
        lists = self._lists(queries, min_score, subsets[0], subsets[1], ties_low_first)
        offsets = np.cumsum([0] + [len(h) for h in lists]).astype(np.int64)
        items = np.array([it for h in lists for it, _ in h], np.int64)
        scores = np.array([sc for h in lists for _, sc in h], np.float32)

        def fetch(out_items, out_scores):
            np.asarray(out_items)[:] = items
            np.asarray(out_scores)[:] = scores
            self.map_items(out_items, positions)

        return LocalRange(offsets, fetch)


def batch_subsets(n, world, b, rng):
    """One subset per query: duplicates across blocks, negatives, every block edge, one block only, empty."""
    from typeagent_py_b200.sharded import shard_bounds

    bounds = shard_bounds(n, world)
    edges = sorted({lo for lo, _ in bounds if lo < n} | {max(lo - 1, 0) for lo, _ in bounds} | {n - 1})
    last_lo, last_hi = bounds[-1]
    out = [
        np.concatenate([rng.permutation(n)[:40], [0, n - 1, 0, n - 1, n // 2] * 3]),
        np.array([-1, -n, 5, -(n // 2), 3, -1, n - 1], np.int64),
        np.array(edges, np.int64),
        np.arange(last_lo, last_hi)[::-2] if last_hi > last_lo else np.array([0]),
        np.empty(0, np.int64),
    ]
    return out[:b]


def oracle_batch_lists(dots, ms, subs, ties_low=False):
    return [oracle_lists(dots[i:i + 1], ms, subset=s, ties_low=ties_low)[0] if len(s) else [] for i, s in enumerate(subs)]


def oracle_batch_arrays(dots, k, ms, subs, ties_low=False):
    kk = max(1, min(k, max(len(s) for s in subs)))
    items, scores, counts = np.full((len(subs), kk), -1, np.int64), np.zeros((len(subs), kk), np.float32), \
        np.zeros(len(subs), np.int32)
    for i, lst in enumerate(oracle_batch_lists(dots, ms, subs, ties_low)):
        lst = lst[:kk]
        counts[i] = len(lst)
        for j, (it, sc) in enumerate(lst):
            items[i, j], scores[i, j] = it, sc
    return items, scores, counts


def oracle_batch_csr(dots, ms, subs, ties_low=False):
    lists = oracle_batch_lists(dots, ms, subs, ties_low)
    offsets = np.cumsum([0] + [len(h) for h in lists]).astype(np.int64)
    return (offsets, np.array([it for h in lists for it, _ in h], np.int64),
            np.array([sc for h in lists for _, sc in h], np.float32))


def _worker(rank, world, port):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        amp, exp = preset("coarse", 16)
        n = 301
        dup = [(n - 1 - j, j) for j in range(0, 40, 3)] + [(150 + j, j) for j in range(0, 20, 2)]
        v, q, _ = dyadic_corpus(n, 16, 5, amp, exp, seed=19, dup=dup)
        dots = exact_dots(q, v)
        sh = make(SubsetsEngine())
        sh.deserialize(v)
        rng = np.random.default_rng(7)
        subs = batch_subsets(n, world, len(q), rng)
        longest = max(len(s) for s in subs)
        for ms in (0.0, 0.5, float("nan")):
            for tl in (False, True):
                for k in (1, 7, longest, longest + 3):
                    same_arrays(sh.search_arrays(q, k, ms, subsets=subs, ties_low_first=tl),
                                oracle_batch_arrays(dots, k, ms, subs, tl), f"rank {rank} subsets ms {ms} tl {tl} k {k}")
                same_csr(sh.search_range(q, ms, ties_low_first=tl, subsets=subs),
                         oracle_batch_csr(dots, ms, subs, tl), f"rank {rank} range subsets ms {ms} tl {tl}")
                # each row equals the one-query subset lookup of the same object
                got = sh.search_arrays(q, 7, ms, subsets=subs, ties_low_first=tl)
                for b in range(len(q)):
                    one = sh.search_arrays(q[b:b + 1], 7, ms, subset=subs[b], ties_low_first=tl)
                    kb = one[0].shape[1]
                    assert got[2][b] == one[2][0]
                    assert got[0][b, :kb].tolist() == one[0][0].tolist()
        for mh in (None, 3, 0):
            got = sh.fuzzy_lookup_embeddings_in_subsets(q, [s.tolist() for s in subs], mh, 0.4)
            for b in range(len(q)):
                assert hits(got[b]) == hits(sh.fuzzy_lookup_embedding_in_subset(q[b], subs[b].tolist(), mh, 0.4)), (mh, b)

        # a k above the top-k merge's limit goes through the threshold exchange, cut to k
        import typeagent_py_b200.sharded as S

        saved = S.SUBSETS_MERGE_MAX_K
        S.SUBSETS_MERGE_MAX_K = 4
        try:
            for k in (5, longest):
                same_arrays(sh.search_arrays(q, k, 0.0, subsets=subs), oracle_batch_arrays(dots, k, 0.0, subs),
                            f"rank {rank} routed k {k}")
        finally:
            S.SUBSETS_MERGE_MAX_K = saved

        # every entry in the last block: the other ranks have no share at all
        last = [subs[3], subs[3][:3], subs[3][::-1]]
        for tl in (False, True):
            same_arrays(sh.search_arrays(q[:3], 6, 0.0, subsets=last, ties_low_first=tl),
                        oracle_batch_arrays(dots[:3], 6, 0.0, last, tl), f"rank {rank} no share tl {tl}")
            same_csr(sh.search_range(q[:3], 0.3, subsets=last, ties_low_first=tl),
                     oracle_batch_csr(dots[:3], 0.3, last, tl), f"rank {rank} range no share tl {tl}")

        # all-empty subsets, and no queries
        o, i, _ = sh.search_range(q[:2], 0.0, subsets=[[], []])
        assert o.tolist() == [0, 0, 0] and len(i) == 0
        assert sh.search_arrays(q[:2], 4, 0.0, subsets=[[], []])[2].tolist() == [0, 0]

        # errors: on every rank, before any collective
        counting = CountingDist(sh._dist)
        sh._dist = counting
        for call, exc in [
            (lambda: sh.search_arrays(q, 5, subsets=subs[:4]), ValueError),
            (lambda: sh.search_range(q, 0.0, subsets=subs[:4]), ValueError),
            (lambda: sh.search_arrays(q, 5, subsets=subs, subset=[1]), ValueError),
            (lambda: sh.search_range(q, 0.0, subsets=subs, allowed=np.ones(n, bool)), ValueError),
            (lambda: sh.search_arrays(q, 5, subsets=[[1], [0.5], [], [2], [3]]), IndexError),
            (lambda: sh.search_arrays(q, 5, subsets=[[1], [n], [], [2], [3]]), IndexError),
            (lambda: sh.search_range(q, 0.0, subsets=[[1], [-n - 1], [], [2], [3]]), IndexError),
            (lambda: sh.search_arrays(q, 0, subsets=subs), ValueError),
            (lambda: sh.fuzzy_lookup_embeddings_in_subsets(q, subs, -1), ValueError),
        ]:
            with pytest.raises(exc):
                call()
        assert counting.calls == 0, "an argument error entered a collective"
        sh._dist = counting.inner
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [1, 2, 3])
def test_subsets_over_gloo(world):
    mp.spawn(_worker, args=(world, _free_port()), nprocs=world, join=True)


def test_subsets_share_and_total_check():
    from typeagent_py_b200.sharded import check_subsets_total, subsets_share

    offsets = np.array([0, 4, 4, 7], np.int64)
    ordinals = np.array([0, 9, -1, 5, 3, -10, 4], np.int64)  # 10 rows
    pos, loff, lord = subsets_share(offsets, ordinals, 10, 4, 8)
    assert pos.tolist() == [3, 6] and loff.tolist() == [0, 1, 1, 2] and lord.tolist() == [1, 0]
    pos, loff, lord = subsets_share(offsets, ordinals, 10, 8, 10)
    assert pos.tolist() == [1, 2] and loff.tolist() == [0, 2, 2, 2] and lord.tolist() == [1, 1]
    check_subsets_total((1 << 32) - 1)
    with pytest.raises(ValueError, match="at most 2\\^32 - 1"):
        check_subsets_total(1 << 32)
