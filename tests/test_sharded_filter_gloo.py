"""Host logic of the row-sharded filtered and subset lookups on CPU, world sizes 1, 2 and 3 over ``gloo``.

The engine is a numpy stand-in with ``CudaShardEngine``'s per-rank steps (``search_rows_packed``,
``search_subset_packed``, ``map_items``, ``merge_ordered``, ``range_local`` with a mask or a subset) that follows
the library's semantics exactly on dyadic corpora (tests/exact.py).  What is under test is the product code
around them (typeagent-py_b200/sharded.py): the split of a subset into per-rank shares, the per-rank bits of a
row mask, per-rank predicate evaluation and its cache, the exchanges and the decode, and the SPMD errors.
Every result is compared with a numpy statement of one-process ``VectorBase`` semantics over the whole corpus.
The CUDA side is covered by tests/test_gpu_sharded_filter.py.
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

from tests.exact import dyadic_corpus, preset, scores_of  # noqa: E402
from tests.test_sharded_gloo import DeferringOracleEngine, OracleShardEngine, _free_port  # noqa: E402
from tests.test_sharded_range_gloo import RangeEngine, exact_dots  # noqa: E402


# ---------------------------------------------------------------- one-process semantics (the oracle)
def oracle_lists(dots, min_score, subset=None, allowed=None, ties_low=False):
    """Per query, every passing hit as (item, score) in ``VectorBase``'s order: score descending; equal scores
    by the tie key (the row, or the subset position) descending, or ascending with ``ties_low``.  Items are
    rows, or the subset's ordinals as given."""
    n = dots.shape[1]
    floor = np.float32(min_score)
    out = []
    for row in np.atleast_2d(dots):
        s = scores_of(row)
        if subset is None:
            keys = np.arange(n)
            rows = keys
            items = keys
        else:
            sub = np.asarray(subset, np.int64)
            keys = np.arange(len(sub))
            rows = np.where(sub < 0, sub + n, sub)
            items = sub
        sc = s[rows]
        ok = sc >= floor
        if allowed is not None:
            ok &= np.asarray(allowed, bool)[rows]
        idx = np.flatnonzero(ok)
        order = idx[np.lexsort((keys[idx] if ties_low else -keys[idx], -sc[idx].view(np.uint32).astype(np.int64)))]
        out.append([(int(items[j]), float(sc[j])) for j in order])
    return out


def oracle_arrays(dots, k, min_score, **kw):
    lists = oracle_lists(dots, min_score, **kw)
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


def oracle_csr(dots, min_score, **kw):
    lists = oracle_lists(dots, min_score, **kw)
    offsets = np.cumsum([0] + [len(h) for h in lists]).astype(np.int64)
    items = np.array([it for h in lists for it, _ in h], np.int64)
    scores = np.array([sc for h in lists for _, sc in h], np.float32)
    return offsets, items, scores


# ---------------------------------------------------------------- the stand-in engine
def _pack(b, k, hits_per_query):
    from typeagent_py_b200.sharded import packed_layout

    off_s, off_c, total = packed_layout(b, k)
    buf = np.zeros(total, np.uint8)
    items = buf[: b * k * 8].view(np.int64).reshape(b, k)
    scores = buf[off_s: off_s + b * k * 4].view(np.float32).reshape(b, k)
    counts = buf[off_c: off_c + b * 4].view(np.int32)
    items[:] = -1
    for i, hits in enumerate(hits_per_query):
        hits = hits[:k]
        counts[i] = len(hits)
        for j, (it, sc) in enumerate(hits):
            items[i, j], scores[i, j] = it, sc
    return torch.from_numpy(buf)


class FilterEngine(RangeEngine):
    """CPU stand-in for CudaShardEngine's filtered and subset steps (test infrastructure)."""

    def __init__(self, fail_topk=False, **kw):
        super().__init__(**kw)
        self.mask_uploads = []
        self.fail_topk = fail_topk

    def remove_rows(self, local_ordinals):
        self.rows = np.delete(self.rows, local_ordinals, axis=0)

    def _mask_bits(self, mask):
        return np.unpackbits(np.asarray(mask, np.uint32).view(np.uint8), bitorder="little")[: len(self.rows)].astype(bool)

    def search_rows_packed(self, queries, k, min_score, item_offset, ties_low_first, mask=None, mask_key=None,
                           mask_owner=None):
        b = len(queries)
        if self.fail_topk:
            raise MemoryError("the local search failed on this rank")
        if len(self.rows) == 0:
            return _pack(b, k, [[]] * b)
        allowed = None
        if mask is not None:
            self.mask_uploads.append(mask_key)
            allowed = self._mask_bits(mask)
        lists = oracle_lists(exact_dots(queries, self.rows), min_score, allowed=allowed, ties_low=ties_low_first)
        return _pack(b, k, [[(it + item_offset, sc) for it, sc in h] for h in lists])

    def search_subset_packed(self, queries, k, min_score, local_subset, positions, ties_low_first):
        b = len(queries)
        if self.fail_topk:
            raise MemoryError("the local search failed on this rank")
        if len(local_subset) == 0:
            return _pack(b, k, [[]] * b)
        # items are positions in the local subset: the oracle over the dots of its rows, in its order
        dots = exact_dots(queries, self.rows)[:, np.asarray(local_subset, np.int64)]
        lists = oracle_lists(dots, min_score, ties_low=ties_low_first)
        buf = _pack(b, k, lists)
        self.map_items(buf[: b * k * 8].view(torch.int64), positions)
        return buf

    def map_items(self, items, table):
        a = items.numpy().reshape(-1)
        table = np.asarray(table, np.int64)
        ok = (a >= 0) & (a < len(table))
        a[ok] = table[a[ok]]
        return items

    def merge_ordered(self, gathered, world, n_queries, k, order):
        from typeagent_py_b200.sharded import packed_layout

        off_s, off_c, _ = packed_layout(n_queries, k)
        g = gathered.numpy()
        out_i = np.full((n_queries, k), -1, np.int64)
        out_s = np.zeros((n_queries, k), np.float32)
        out_c = np.zeros(n_queries, np.int32)
        for q in range(n_queries):
            cand = []
            for r in range(world):
                items = g[r, : n_queries * k * 8].view(np.int64).reshape(n_queries, k)
                scores = g[r, off_s: off_s + n_queries * k * 4].view(np.float32).reshape(n_queries, k)
                counts = g[r, off_c: off_c + n_queries * 4].view(np.int32)
                for j in range(counts[q]):
                    it, sc = int(items[q, j]), scores[q, j]
                    tie = {0: r * k + (k - 1 - j), 1: -(r * k + j), 2: it, 3: -it}[order]
                    cand.append((int(sc.view(np.uint32)), tie, it, sc))
            cand.sort(key=lambda c: (c[0], c[1]), reverse=True)
            cand = cand[:k]
            out_c[q] = len(cand)
            for j, c in enumerate(cand):
                out_i[q, j], out_s[q, j] = c[2], c[3]
        return torch.from_numpy(out_i), torch.from_numpy(out_s), torch.from_numpy(out_c)

    def range_local(self, queries, min_score, item_offset, ties_low_first, mask=None, mask_key=None,
                    mask_owner=None, subset=None, positions=None):
        from typeagent_py_b200.sharded import LocalRange

        if mask is None and subset is None:
            return super().range_local(queries, min_score, item_offset, ties_low_first)
        self.range_calls += 1
        b = len(queries)
        if len(self.rows) == 0 or (subset is not None and len(subset) == 0):
            return LocalRange(np.zeros(b + 1, np.int64), None)
        dots = exact_dots(queries, self.rows)
        if subset is not None:
            offsets, items, scores = oracle_csr(dots[:, np.asarray(subset, np.int64)], min_score, ties_low=ties_low_first)
        else:
            self.mask_uploads.append(mask_key)
            offsets, items, scores = oracle_csr(dots, min_score, allowed=self._mask_bits(mask), ties_low=ties_low_first)
            items = items + item_offset

        def fetch(out_items, out_scores):
            np.asarray(out_items)[:] = items
            np.asarray(out_scores)[:] = scores
            if subset is not None:
                self.map_items(out_items, positions)

        return LocalRange(offsets, fetch)


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


def make(engine=None):
    from types import SimpleNamespace

    from oracle import vectorbase_oracle as O
    from typeagent_py_b200.sharded import ShardedVectorBase

    settings = SimpleNamespace(embedding_model=O.FakeEmbeddingModel(), min_score=0.85, max_matches=None)
    return ShardedVectorBase(settings, engine=engine or FilterEngine())


def same_arrays(got, want, what):
    for g, w, name in zip(got, want, ("items", "scores", "counts")):
        np.testing.assert_array_equal(np.asarray(g).view(np.uint32) if name == "scores" else g,
                                      np.asarray(w).view(np.uint32) if name == "scores" else w, err_msg=f"{what}: {name}")


def same_csr(got, want, what):
    np.testing.assert_array_equal(got[0], want[0], err_msg=f"{what}: offsets")
    np.testing.assert_array_equal(got[1], want[1], err_msg=f"{what}: items")
    np.testing.assert_array_equal(got[2].view(np.uint32), want[2].view(np.uint32), err_msg=f"{what}: scores")


def hits(lst):
    return [(h.item, h.score) for h in lst]


def subsets(n, world, rng):
    from typeagent_py_b200.sharded import shard_bounds

    b = shard_bounds(n, world)
    starts = [lo for lo, _ in b if lo < n]
    return {
        "unsorted": rng.permutation(n)[: n // 2],
        "duplicates": np.concatenate([rng.permutation(n)[:60], [0, n - 1, 0, n - 1, n // 2] * 3]),
        "negative": np.array([-1, -n, 5, -(n // 2), 3, -1, n - 1], np.int64),
        "block_edges": np.array(sorted({s for s in starts} | {max(s - 1, 0) for s in starts} | {n - 1}), np.int64),
        "one_rank": np.arange(b[-1][0], b[-1][1])[::-2] if b[-1][1] > b[-1][0] else np.array([0]),
        "everything_twice": np.concatenate([np.arange(n), np.arange(n)[::-1]]),
    }


def _worker(rank, world, port):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        amp, exp = preset("coarse", 16)
        n = 301
        # copies of early rows in every later block: equal scores on different ranks
        dup = [(n - 1 - j, j) for j in range(0, 40, 3)] + [(150 + j, j) for j in range(0, 20, 2)]
        v, q, _ = dyadic_corpus(n, 16, 5, amp, exp, seed=17, dup=dup)
        dots = exact_dots(q, v)
        sh = make()
        sh.deserialize(v)
        lo, hi = sh.local_range
        rng = np.random.default_rng(5)

        # ---- subsets: search_arrays, search_range, fuzzy_lookup_embedding_in_subset
        for name, sub in subsets(n, world, rng).items():
            for ms in (0.0, 0.5):
                for tl in (False, True):
                    for k in (1, 7, len(sub), len(sub) + 3):
                        got = sh.search_arrays(q, k, ms, subset=sub, ties_low_first=tl)
                        kk = max(1, min(k, len(sub)))
                        same_arrays(got, oracle_arrays(dots, kk, ms, subset=sub, ties_low=tl),
                                    f"rank {rank} subset {name} ms {ms} tl {tl} k {k}")
                    same_csr(sh.search_range(q, ms, ties_low_first=tl, subset=sub),
                             oracle_csr(dots, ms, subset=sub, ties_low=tl), f"rank {rank} range subset {name} {ms} {tl}")
                for mh in (None, 3, 0):
                    kk = {None: 10, 3: 3, 0: len(sub)}[mh]
                    want = oracle_lists(dots[2:3], ms, subset=sub)[0][:kk]
                    assert hits(sh.fuzzy_lookup_embedding_in_subset(q[2], sub.tolist(), mh, ms)) == want, (rank, name, mh)
                    assert hits(sh.fuzzy_lookup_embedding_in_subset(q[2], sub, mh, ms)) == want
        assert sh.fuzzy_lookup_embedding_in_subset(q[0], [], 5, 0.0) == []
        assert sh.search_arrays(q, 4, 0.0, subset=[])[2].tolist() == [0] * len(q)
        o, i, _ = sh.search_range(q, 0.0, subset=np.array([], np.int64))
        assert o.tolist() == [0] * (len(q) + 1) and len(i) == 0

        # ---- row masks: bool and packed, blocks that do not start on a word
        from typeagent_py_b200.vectorbase import VectorBase

        allowed = rng.random(n) < 0.4
        allowed[[j for j, _ in dup]] = True
        words = VectorBase.pack_row_mask(allowed)
        for mask in (allowed, words):
            for ms in (0.0, 0.5):
                for tl in (False, True):
                    for k in (1, 9, n):
                        same_arrays(sh.search_arrays(q, k, ms, allowed=mask, ties_low_first=tl),
                                    oracle_arrays(dots, min(k, n), ms, allowed=allowed, ties_low=tl),
                                    f"rank {rank} mask {mask.dtype} {ms} {tl} {k}")
                    same_csr(sh.search_range(q, ms, ties_low_first=tl, allowed=mask),
                             oracle_csr(dots, ms, allowed=allowed, ties_low=tl), f"rank {rank} range mask {ms} {tl}")
        # ties low-first alone
        same_arrays(sh.search_arrays(q, 12, 0.25, ties_low_first=True), oracle_arrays(dots, 12, 0.25, ties_low=True),
                    f"rank {rank} ties_low")
        # an unchanged mask object is cut to this block once per rows, and the engine is handed the same words
        # under the same key every time (the key CudaShardEngine's VectorBase skips a repeated upload by)
        import typeagent_py_b200.sharded as S

        cuts, real_cut = [], S.block_mask
        S.block_mask = lambda *a: cuts.append(a[2:]) or real_cut(*a)
        try:
            fresh = words.copy()
            sh._engine.mask_uploads.clear()
            sh.search_arrays(q, 3, 0.0, allowed=fresh)
            sh.search_arrays(q, 5, 0.0, allowed=fresh)
            sh.search_range(q, 0.5, allowed=fresh)
        finally:
            S.block_mask = real_cut
        assert cuts == [(lo, hi)], cuts
        keys = sh._engine.mask_uploads
        assert len(keys) == (3 if hi > lo else 0) and len(set(keys)) <= 1

        # ---- predicates: only this rank's rows, once per cache key
        calls = []

        def pred(i):
            calls.append(i)
            return bool(allowed[i])

        for mh in (None, 4, n):
            for ms in (0.0, 0.5):
                kk = 10 if mh is None else mh
                want = oracle_lists(dots[1:2], ms, allowed=allowed, ties_low=True)[0][:kk]
                assert hits(sh.fuzzy_lookup_embedding(q[1], mh, ms, predicate=pred)) == want, (rank, mh, ms)
        assert sorted(calls) == list(range(lo, hi)), (rank, len(calls))
        assert sh.fuzzy_lookup_embedding(q[1], 0, 0.0, predicate=pred) == []
        # rows appended: a new cache key, the predicate runs again over this rank's (new) rows only
        extra = dyadic_corpus(7, 16, 1, amp, exp, seed=18)[0]
        sh.add_embeddings(None, extra)
        both = np.concatenate([v, extra])
        allowed2 = np.concatenate([allowed, np.ones(7, bool)])
        calls.clear()

        def pred2(i):
            calls.append(i)
            return bool(allowed2[i])

        want = oracle_lists(exact_dots(q[3:4], both), 0.25, allowed=allowed2, ties_low=True)[0][:6]
        assert hits(sh.fuzzy_lookup_embedding(q[3], 6, 0.25, predicate=pred2)) == want
        lo2, hi2 = sh.local_range
        assert sorted(calls) == list(range(lo2, hi2))
        sh.remove_embeddings(np.arange(n, n + 7))

        # ---- errors on every rank, before any exchange, and no collective left open
        counting = CountingDist(sh._dist)
        sh._dist = counting
        with pytest.raises(IndexError, match="out of bounds"):
            sh.fuzzy_lookup_embedding_in_subset(q[0], [0, n], 3, 0.0)
        with pytest.raises(IndexError, match="out of bounds"):
            sh.fuzzy_lookup_embedding_in_subset(q[0], [-n - 1], 3, 0.0)
        with pytest.raises(IndexError, match="integer"):
            sh.fuzzy_lookup_embedding_in_subset(q[0], [0.5, 1.0], 3, 0.0)
        with pytest.raises(IndexError):
            sh.search_arrays(q, 3, 0.0, subset=np.array([n + 2]))
        with pytest.raises(IndexError):
            sh.search_range(q, 0.0, subset=[3, -n - 5])
        with pytest.raises(ValueError, match="cannot be combined"):
            sh.search_arrays(q, 3, 0.0, subset=[1], allowed=allowed)
        with pytest.raises(ValueError, match="cannot be combined"):
            sh.search_range(q, 0.0, subset=[1], allowed=allowed)
        with pytest.raises(ValueError, match="row mask"):
            sh.search_arrays(q, 3, 0.0, allowed=allowed[:-1])
        with pytest.raises(ValueError, match="row mask"):
            sh.search_range(q, 0.0, allowed=words[:-1])
        with pytest.raises(ValueError):
            sh.search_arrays(q, 0, 0.0, subset=[1])
        with pytest.raises(ValueError):
            sh.fuzzy_lookup_embedding(q[0], -1, 0.0, predicate=pred)
        with pytest.raises(ValueError, match="not aligned"):
            sh.fuzzy_lookup_embedding_in_subset(q[0][:5], [1, 2], 3, 0.0)
        # NaN min_score and empty subsets return at once
        assert sh.fuzzy_lookup_embedding_in_subset(q[0], [1, 2], 3, float("nan")) == []
        assert sh.search_arrays(q, 3, float("nan"), subset=[1])[2].tolist() == [0] * len(q)
        assert counting.calls == 0, counting.calls
        sh._dist = counting.inner

        # a predicate that raises on one rank raises on every rank
        def bad_pred(i):
            if rank == world - 1:
                raise KeyError("no such message")
            return True

        with pytest.raises((KeyError, RuntimeError)):
            sh.fuzzy_lookup_embedding(q[0], 3, 0.0, predicate=bad_pred)
        assert hits(sh.fuzzy_lookup_embedding(q[0], 3, 0.0, predicate=pred)) == \
            oracle_lists(dots[0:1], 0.0, allowed=allowed, ties_low=True)[0][:3]

        # a local search that fails on one rank raises on every rank, and nobody is left in the all-gather
        bad = make(FilterEngine(fail_topk=(rank == world - 1)))
        bad.deserialize(v)
        for call in (lambda: bad.search_arrays(q, 4, 0.0, allowed=allowed),
                     lambda: bad.search_arrays(q, 4, 0.0, subset=[3, 1, -1]),
                     lambda: bad.fuzzy_lookup_embedding(q[0], 4, 0.0, predicate=pred)):
            with pytest.raises((MemoryError, RuntimeError)):
                call()
        bad._engine.fail_topk = False
        same_arrays(bad.search_arrays(q, 4, 0.0, subset=[3, 1, -1]), oracle_arrays(dots, 3, 0.0, subset=[3, 1, -1]),
                    f"rank {rank} after a failure")

        # ---- empty blocks: fewer rows than ranks
        tiny = make()
        tiny.deserialize(v[: max(world - 1, 1)])
        m = max(world - 1, 1)
        tdots = exact_dots(q, v[:m])
        same_arrays(tiny.search_arrays(q, 2, 0.0, subset=[0, -1, 0]), oracle_arrays(tdots, 2, 0.0, subset=[0, -1, 0]),
                    f"rank {rank} tiny subset")
        tmask = np.ones(m, bool)
        same_arrays(tiny.search_arrays(q, 2, 0.0, allowed=tmask, ties_low_first=True),
                    oracle_arrays(tdots, min(2, m), 0.0, allowed=tmask, ties_low=True), f"rank {rank} tiny mask")
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [1, 2, 3])
def test_filtered_and_subset_lookups_over_gloo(world):
    mp.spawn(_worker, args=(world, _free_port()), nprocs=world, join=True)


class DeferringFilterEngine(FilterEngine):
    """Deferred lookups spoiled on some ranks and repaired at finish(), as DeferringOracleEngine does, plus the
    filtered steps."""

    def __init__(self, rank, spoil_ranks):
        super().__init__()
        self.rank, self.spoil_ranks, self.fail_rank, self.fixups = rank, spoil_ranks, None, []

    def search_packed(self, queries, k, min_score, item_offset, defer_check=False):
        from typeagent_py_b200.sharded import packed_layout

        buf = OracleShardEngine.search_packed(self, queries, k, min_score, item_offset)
        if defer_check and self.rank in self.spoil_ranks:
            _, off_c, _ = packed_layout(len(queries), k)
            counts = buf.numpy()[off_c: off_c + 4 * len(queries)].view(np.int32)
            self.fixups.append((counts, int(counts[0])))
            counts[0] = 0
        return buf

    def finish(self):
        return DeferringOracleEngine.finish(self)


def _deferred_worker(rank, world, port):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        amp, exp = preset("coarse", 16)
        n = 200
        v, q, _ = dyadic_corpus(n, 16, 4, amp, exp, seed=23)
        dots = exact_dots(q, v)
        sh = make(DeferringFilterEngine(rank, spoil_ranks={0}))
        sh.deserialize(v)
        # a deferred lookup, then a filtered one: the filtered lookup finishes it first, and its result is merged
        # again with the corrected candidates
        items, scores, counts = sh.search_tensors(q, 5, 0.0, defer_check=True)
        allowed = np.ones(n, bool)
        allowed[::3] = False
        got = sh.search_arrays(q, 6, 0.0, allowed=allowed)
        same_arrays(got, oracle_arrays(dots, 6, 0.0, allowed=allowed), f"rank {rank} filtered after deferred")
        assert sh._pending == [] and sh._engine.fixups == []
        fresh = sh.search_tensors(q, 5, 0.0)  # not deferred: never spoiled
        same_arrays((items.numpy(), scores.numpy(), counts.numpy()), tuple(t.numpy() for t in fresh),
                    f"rank {rank} deferred lookup repaired")
        # the same with a predicate
        sh.search_tensors(q, 5, 0.0, defer_check=True)
        assert hits(sh.fuzzy_lookup_embedding(q[0], 4, 0.0, predicate=lambda i: bool(allowed[i]))) == \
            oracle_lists(dots[0:1], 0.0, allowed=allowed, ties_low=True)[0][:4]
        assert sh._pending == []
    finally:
        dist.destroy_process_group()


def test_deferred_lookup_before_a_filtered_one_over_gloo():
    mp.spawn(_deferred_worker, args=(2, _free_port()), nprocs=2, join=True)


def test_block_mask_and_subset_share():
    from typeagent_py_b200.sharded import block_mask, subset_share
    from typeagent_py_b200.vectorbase import VectorBase

    rng = np.random.default_rng(1)
    for n in (1, 31, 32, 33, 100, 257):
        allowed = rng.random(n) < 0.5
        words = VectorBase.pack_row_mask(allowed)
        for lo, hi in ((0, n), (0, 0), (n // 3, n // 3 + 17), (min(5, n), n), (n, n)):
            hi = min(hi, n)
            want = VectorBase.pack_row_mask(allowed[lo:hi])
            np.testing.assert_array_equal(block_mask(allowed, n, lo, hi), want)
            np.testing.assert_array_equal(block_mask(words, n, lo, hi), want)
    with pytest.raises(ValueError, match="100 entries for 101 rows"):
        block_mask(np.ones(100, bool), 101, 0, 50)
    with pytest.raises(ValueError, match="bits for 65 rows"):
        block_mask(np.zeros(2, np.uint32), 65, 0, 50)
    sub = np.array([5, -1, 9, 0, 5, -10], np.int64)
    pos, local = subset_share(sub, 10, 5, 10)
    assert pos.tolist() == [0, 1, 2, 4] and local.tolist() == [0, 4, 4, 0]
    pos, local = subset_share(sub, 10, 0, 5)
    assert pos.tolist() == [3, 5] and local.tolist() == [0, 0]


def _routing_worker(rank, world, port):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        # k >= rows searched > 8192: one threshold search laid out [B, rows], as tav_search routes it on one GPU,
        # with ties low-first alone, a mask, or a subset (the stand-in's search_packed raises if reached)
        amp, exp = preset("fine", 8)
        n = 8300
        v, q, _ = dyadic_corpus(n, 8, 3, amp, exp, seed=29, dup=[(8000 + j, j) for j in range(0, 200, 3)])
        dots = exact_dots(q, v)
        sh = make()
        sh.deserialize(v)
        for ms in (0.5, 0.0):
            for k in (n, n + 5):
                same_arrays(sh.search_arrays(q, k, ms, ties_low_first=True), oracle_arrays(dots, n, ms, ties_low=True),
                            f"rank {rank} routed ties_low {ms} {k}")
            allowed = np.arange(n) % 3 != 1
            same_arrays(sh.search_arrays(q, n, ms, allowed=allowed, ties_low_first=True),
                        oracle_arrays(dots, n, ms, allowed=allowed, ties_low=True), f"rank {rank} routed mask {ms}")
            sub = np.concatenate([np.arange(n)[::-1], np.arange(0, 400)])
            same_arrays(sh.search_arrays(q, len(sub), ms, subset=sub),
                        oracle_arrays(dots, len(sub), ms, subset=sub), f"rank {rank} routed subset {ms}")
        assert sh._engine.range_calls >= 6
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [1, 2, 3])
def test_routed_filtered_lookups_over_gloo(world):
    mp.spawn(_routing_worker, args=(world, _free_port()), nprocs=world, join=True)
