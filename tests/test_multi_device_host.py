"""Host logic of ``VectorBase(settings, devices=[...])`` on CPU: the block layout rules, the ``devices=`` argument,
the refusals of what a multi-device index does not offer, and the dispatch to ``tav_multi_*`` through a stand-in
for libtavec.

The stand-in keeps each shard's "device" rows as numpy arrays and changes them only through the entry points the
class calls (create, clear, append, remove, write, row mask), and its multi-device searches read those rows through
the block starts the class passes.  So the tests see what each shard is told, and that the shards laid end to end
always equal the host mirror.  The library itself is covered on the GPU by tests/test_gpu_multi_device.py.
"""

from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import typeagent_py_b200 as tab
from oracle import vectorbase_oracle as O
from typeagent_py_b200 import _capi
from typeagent_py_b200.multi import (MERGE_MAX_K, check_devices, even_starts, layout_plan, removal_plan,
                                     write_plan)


# ---------------------------------------------------------------------------------------------------- layout rules
def test_first_sync_splits_evenly_and_reloads_every_shard():
    new, steps = layout_plan(None, 10, 3)
    assert new == [0, 4, 8, 10]
    assert steps == [(0, 0, 4, True), (0, 4, 8, True), (0, 8, 10, True)]


def test_fewer_rows_than_shards_leaves_empty_blocks():
    new, steps = layout_plan(None, 2, 4)
    assert new == [0, 1, 2, 2, 2]
    assert steps[2:] == [(0, 2, 2, True), (0, 2, 2, True)]
    assert layout_plan(None, 0, 3)[0] == [0, 0, 0, 0]


def test_appends_join_the_last_block():
    new, steps = layout_plan([0, 4, 8, 10], 13, 3)
    assert new == [0, 4, 8, 13]
    assert steps == [(0, 4, 4, False), (0, 8, 8, False), (0, 10, 13, False)]


def test_no_change_is_no_step():
    new, steps = layout_plan([0, 4, 8, 10], 10, 3)
    assert new == [0, 4, 8, 10]
    assert all(drop == 0 and lo == hi and not reload for drop, lo, hi, reload in steps)


def test_resplit_when_the_largest_block_exceeds_twice_the_even_share():
    # 27 of 30 rows in the last block: 27 * 3 > 2 * 30
    new, steps = layout_plan([0, 1, 2, 3], 30, 3)
    assert new == [0, 10, 20, 30]
    assert steps[0] == (0, 1, 10, False)       # keeps its row, gains a suffix: in place
    assert steps[1] == (0, 10, 20, True)       # its old row moves to block 0: reloaded
    assert steps[2] == (0, 20, 30, True)
    # exactly twice the even share is not above it
    assert layout_plan([0, 1, 2, 6], 6, 3)[0] == [0, 1, 2, 6]
    assert layout_plan([0, 1, 2, 7], 7, 3)[0] == [0, 3, 6, 7]


def test_resplit_updates_a_block_that_loses_a_prefix_in_place():
    # removals shrank blocks 0 and 1: block 2 holds 7 of 9 rows
    new, steps = layout_plan([0, 1, 2, 9], 9, 3)
    assert new == [0, 3, 6, 9]
    assert steps[0] == (0, 1, 3, False)
    assert steps[1] == (0, 3, 6, True)
    assert steps[2] == (4, 9, 9, False)        # drops rows [2, 6), keeps [6, 9)


def test_removal_plan_routes_ordinals_to_their_blocks():
    per, new = removal_plan([0, 3, 6, 9], np.array([1, 2, 7, 10]))  # row 10 is not on the devices yet
    assert [p.tolist() for p in per] == [[1, 2], [], [1]]
    assert new == [0, 1, 4, 6]
    per, new = removal_plan([0, 3, 6, 9], np.array([3, 4, 5]))
    assert [p.tolist() for p in per] == [[], [0, 1, 2], []]
    assert new == [0, 3, 3, 6]                  # block 1 is empty now


def test_write_plan_crosses_block_boundaries():
    assert write_plan([0, 3, 6, 8], 2, 5) == [(0, 2, 0, 1), (1, 0, 1, 4), (2, 0, 4, 5)]
    assert write_plan([0, 3, 6, 8], 7, 4) == [(2, 1, 0, 1)]    # rows past 8 are not on the devices yet
    assert write_plan([0, 3, 3, 8], 2, 2) == [(0, 2, 0, 1), (2, 0, 1, 2)]
    assert even_starts(5, 2) == [0, 3, 5]


# ---------------------------------------------------------------------------------------------- devices= argument
def _settings():
    return tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel())


@pytest.mark.parametrize("devices, exc", [([], ValueError), (list(range(33)), ValueError), ([0, -1], ValueError),
                                          (["0"], TypeError), ([True], TypeError), (3, TypeError), ("01", TypeError),
                                          ([0.0], TypeError)])
def test_devices_argument_errors(devices, exc):
    with pytest.raises(exc):
        tab.VectorBase(_settings(), devices=devices)


def test_devices_is_exclusive_with_device():
    with pytest.raises(ValueError, match="cannot be combined"):
        tab.VectorBase(_settings(), device=0, devices=[0, 0])
    assert check_devices((0, np.int64(1), 0)) == [0, 1, 0]
    assert len(check_devices([0] * 32)) == 32


def test_default_is_one_device():
    base = tab.VectorBase(_settings())
    assert base._multi is None and base._device == 0
    assert tab.VectorBase(_settings(), device=1)._device == 1
    assert tab.VectorBase(_settings(), devices=[2, 0])._device == 2


# ------------------------------------------------------------------------------------------------------- refusals
def test_refusals_come_before_any_library_call(monkeypatch):
    def no_library():
        raise AssertionError("the library was called")

    monkeypatch.setattr(_capi, "load", no_library)
    base = tab.VectorBase(_settings(), devices=[0, 0])
    v, q = O.make_corpus(20, 8, seed=1, n_queries=2)
    base.add_embeddings(None, v)
    with pytest.raises(NotImplementedError, match="devices="):
        base.search_arrays(q, 3, subsets=[[0], [1]])
    with pytest.raises(NotImplementedError, match="per-query masks"):
        base.search_arrays(q, 3, allowed=np.ones((2, 20), bool))
    with pytest.raises(NotImplementedError, match="per-query subsets"):
        base.search_range(q, 0.5, subsets=[[0], [1]])
    with pytest.raises(NotImplementedError, match="per-query masks"):
        base.search_range(q, 0.5, allowed=np.ones((2, 20), bool))
    with pytest.raises(NotImplementedError):
        base.fuzzy_lookup_embeddings_in_subsets(q, [[0], [1]])
    with pytest.raises(NotImplementedError, match="search_device"):
        base.search_device(object(), 3)
    with pytest.raises(NotImplementedError, match="search_range_device"):
        base.search_range_device(object(), 0.5, 10)
    with pytest.raises(NotImplementedError, match="finish_search"):
        base.finish_search()
    with pytest.raises(NotImplementedError, match="from_device_tensor"):
        tab.VectorBase.from_device_tensor(_settings(), object(), devices=[0, 0])


# ------------------------------------------------------------------------------------------------------- dispatch
def _view(addr, ctype, n):
    addr = C.cast(addr, C.c_void_p).value if not isinstance(addr, int) else addr
    return np.ctypeslib.as_array(C.cast(addr, C.POINTER(ctype)), (n,)) if n else np.zeros(0, np.dtype(ctype))


def _ranked(vectors, q, floor, ties_low, allowed=None, subset=None):
    """(keys, scores) of every passing row of one query, in the library's order (the stand-in's arithmetic)."""
    if subset is not None:
        n = len(vectors)
        rows = np.where(subset < 0, subset + n, subset)
        keys = np.arange(len(subset))
    else:
        rows = keys = np.arange(len(vectors))
    s = np.clip((vectors[rows] @ q + np.float32(1)) / np.float32(2), 0, 1).astype(np.float32)
    ok = s >= floor
    if allowed is not None:
        ok &= allowed[rows]
    keys, s = keys[ok], s[ok]
    order = np.lexsort((keys if ties_low else -keys, -s.astype(np.float64)))
    return keys[order], s[order]


class MultiStandIn:
    """The entry points a multi-device VectorBase calls, over numpy copies of each shard's rows (test
    infrastructure)."""

    def __init__(self):
        self.shards = {}     # handle -> {"rows", "mask", "device"}
        self.calls = []      # (name, shard number, detail) of every row-changing call
        self.multi = None
        self.searches = []   # (kind, flags, k) of every multi-device search
        self.error = ""
        self._hits = None

    def tav_last_error(self):
        return self.error.encode()

    def _fail(self, rc, msg):
        self.error = msg
        return rc

    def _g(self, ix):
        return list(self.shards).index(C.cast(ix, C.c_void_p).value if not isinstance(ix, int) else ix)

    def _shard(self, ix):
        return self.shards[C.cast(ix, C.c_void_p).value if not isinstance(ix, int) else ix]

    def tav_create(self, device, dim, dtype, flags, reserve, out):
        h = 1000 + len(self.shards)
        self.shards[h] = {"rows": None, "mask": None, "device": device}
        out._obj.value = h
        return 0

    def tav_destroy(self, ix):
        return 0

    def tav_multi_create(self, home, n, arr, out):
        self.multi = [arr[i] for i in range(n)]
        assert self.multi == list(self.shards)[-n:]
        out._obj.value = 7
        return 0

    def tav_multi_destroy(self, m):
        return 0

    def tav_clear(self, ix):
        self.calls.append(("clear", self._g(ix), None))
        self._shard(ix).update(rows=None, mask=None)
        return 0

    def tav_append(self, ix, rows, n, dim, src_dtype, on_device, stream):
        new = _view(rows, C.c_float, n * dim).reshape(n, dim).copy()
        s = self._shard(ix)
        s["rows"] = new if s["rows"] is None else np.concatenate([s["rows"], new])
        s["mask"] = None
        self.calls.append(("append", self._g(ix), n))
        return 0

    def tav_remove_rows(self, ix, ordinals, n, stream):
        idx = _view(ordinals, C.c_int64, n).copy()
        s = self._shard(ix)
        if idx.size and (idx.min() < 0 or idx.max() >= len(s["rows"])):
            return self._fail(_capi.TAV_ERR_RANGE, "index out of bounds")
        s["rows"] = np.delete(s["rows"], idx, axis=0)
        s["mask"] = None
        self.calls.append(("remove", self._g(ix), idx.tolist()))
        return 0

    def tav_write_rows(self, ix, first, rows, n, dim, src_dtype, on_device, stream):
        s = self._shard(ix)
        assert first + n <= len(s["rows"])
        s["rows"][first:first + n] = _view(rows, C.c_float, n * dim).reshape(n, dim)
        self.calls.append(("write", self._g(ix), (first, n)))
        return 0

    def tav_set_row_mask(self, ix, bits, n_rows, on_device, stream):
        s = self._shard(ix)
        assert n_rows == len(s["rows"])
        words = _view(bits, C.c_uint32, (n_rows + 31) // 32).copy()
        s["mask"] = np.unpackbits(words.view(np.uint8), bitorder="little")[:n_rows].astype(bool)
        self.calls.append(("mask", self._g(ix), n_rows))
        return 0

    def _corpus(self, starts_p, flags):
        """The rows and mask the blocks make, checked against the starts the class passed."""
        shards = [self.shards[h] for h in self.multi]
        starts = _view(starts_p, C.c_int64, len(shards) + 1)
        parts, masks = [], []
        for g, s in enumerate(shards):
            rows = s["rows"] if s["rows"] is not None else np.zeros((0, 0), np.float32)
            assert starts[g + 1] - starts[g] == len(rows), "starts do not match the shards"
            if len(rows):
                parts.append(rows)
                if flags & _capi.TAV_USE_ROW_MASK:
                    assert s["mask"] is not None, f"shard {g} has no row mask"
                    masks.append(s["mask"])
        rows = np.concatenate(parts) if parts else np.zeros((0, 0), np.float32)
        return rows, (np.concatenate(masks) if masks else None)

    def tav_multi_search(self, m, starts, qp, nq, k, floor, flags, sub, sub_len, ip, sp, cp):
        assert flags & ~(_capi.TAV_FORCE_SCAN | _capi.TAV_FORCE_MMA | _capi.TAV_USE_ROW_MASK |
                         _capi.TAV_TIES_LOW_FIRST) == 0
        self.searches.append(("topk", flags, k))
        floor = np.float32(getattr(floor, "value", floor))
        rows, mask = self._corpus(starts, flags)
        q = _view(qp, C.c_float, nq * rows.shape[1]).reshape(nq, -1)
        subset = _view(sub, C.c_int64, sub_len).copy() if sub_len else (np.zeros(0, np.int64) if sub else None)
        items = _view(ip, C.c_int64, nq * k).reshape(nq, k)
        scores = _view(sp, C.c_float, nq * k).reshape(nq, k)
        counts = _view(cp, C.c_int32, nq)
        for b in range(nq):
            keys, s = _ranked(rows, q[b], floor, flags & _capi.TAV_TIES_LOW_FIRST, mask, subset)
            keys, s = keys[:k], s[:k]
            counts[b] = len(keys)
            items[b, :len(keys)] = subset[keys] if subset is not None else keys
            scores[b, :len(keys)] = s
        return 0

    def tav_multi_range_search(self, m, starts, qp, nq, floor, flags, sub, sub_len, hint, op):
        self.searches.append(("range", flags, None))
        floor = np.float32(getattr(floor, "value", floor))
        rows, mask = self._corpus(starts, flags)
        q = _view(qp, C.c_float, nq * rows.shape[1]).reshape(nq, -1)
        subset = _view(sub, C.c_int64, sub_len).copy() if sub_len else None
        offsets = _view(op, C.c_int64, nq + 1)
        its, scs = [], []
        offsets[0] = 0
        for b in range(nq):
            keys, s = _ranked(rows, q[b], floor, flags & _capi.TAV_TIES_LOW_FIRST, mask, subset)
            its.append(subset[keys] if subset is not None else keys)
            scs.append(s)
            offsets[b + 1] = offsets[b] + len(keys)
        self._hits = (np.concatenate(its).astype(np.int64), np.concatenate(scs).astype(np.float32))
        return 0

    def tav_multi_range_fetch(self, m, first, n, ip, sp):
        _view(ip, C.c_int64, n)[:] = self._hits[0][first:first + n]
        _view(sp, C.c_float, n)[:] = self._hits[1][first:first + n]
        return 0

    def device_rows(self):
        parts = [s["rows"] for s in (self.shards[h] for h in self.multi) if s["rows"] is not None]
        return np.concatenate(parts) if parts else np.zeros((0, 0), np.float32)


@pytest.fixture
def lib(monkeypatch):
    stand_in = MultiStandIn()
    monkeypatch.setattr(_capi, "load", lambda: stand_in)
    return stand_in


def _make(world, n, d=8, seed=0):
    v, q = O.make_corpus(n, d, seed=seed, n_queries=4)
    base = tab.VectorBase(_settings(), devices=[0] * world)
    base.add_embeddings(None, v)
    return base, q


def _expect_topk(base, q, k, floor=0.0, ties_low=False, allowed=None, subset=None):
    v = base._vectors
    out = []
    for b in range(len(q)):
        keys, s = _ranked(v, q[b], np.float32(floor), ties_low, allowed,
                          None if subset is None else np.asarray(subset, np.int64))
        items = np.asarray(subset, np.int64)[keys] if subset is not None else keys
        out.append((items[:k].tolist(), s[:k].tolist()))
    return out


def _got_topk(res):
    items, scores, counts = res
    return [(items[b, :c].tolist(), scores[b, :c].tolist()) for b, c in enumerate(counts)]


def _check_all(base, lib, q):
    """Every lookup kind over the multi-device index equals the stand-in's arithmetic over the mirror."""
    base.search_arrays(q, 1)  # brings the device up to date
    assert np.array_equal(lib.device_rows().reshape(len(base), -1), base._vectors)
    assert list(base._multi.starts) == sorted(base._multi.starts) and base._multi.starts[-1] == len(base)
    assert _got_topk(base.search_arrays(q, 5, 0.4)) == _expect_topk(base, q, 5, 0.4)
    assert _got_topk(base.search_arrays(q, 5, ties_low_first=True)) == _expect_topk(base, q, 5, ties_low=True)
    n = len(base)
    sub = [n - 1, 0, -1, 1 % n, 0]
    assert _got_topk(base.search_arrays(q, 3, subset=sub)) == _expect_topk(base, q, 3, subset=sub)
    allowed = np.arange(n) % 3 != 1
    assert _got_topk(base.search_arrays(q, 4, allowed=allowed)) == _expect_topk(base, q, 4, allowed=allowed)
    offsets, items, scores = base.search_range(q, 0.45)
    want = _expect_topk(base, q, n, 0.45)
    assert [(items[a:b].tolist(), scores[a:b].tolist()) for a, b in zip(offsets[:-1], offsets[1:])] == want
    hits = base.fuzzy_lookup_embedding(q[0], max_hits=2)
    assert [(h.item, h.score) for h in hits] == list(zip(*_expect_topk(base, q[:1], 2)[0]))
    hits = base.fuzzy_lookup_embedding_in_subset(q[1], [0, n - 1, 0], max_hits=5)
    want_items, want_scores = _expect_topk(base, q[1:2], 5, subset=[0, n - 1, 0])[0]
    assert [(h.item, h.score) for h in hits] == list(zip(want_items, want_scores))


def test_lookups_dispatch_to_the_multi_device_calls(lib):
    base, q = _make(3, 40)
    _check_all(base, lib, q)
    assert {kind for kind, _, _ in lib.searches} == {"topk", "range"}
    assert base._multi.starts == [0, 14, 28, 40]


def test_appends_go_to_the_last_shard_until_a_resplit(lib):
    base, q = _make(3, 30)
    _check_all(base, lib, q)
    lib.calls.clear()
    v, _ = O.make_corpus(5, 8, seed=3)
    base.add_embeddings(None, v)
    _check_all(base, lib, q)
    assert [c for c in lib.calls if c[0] != "mask"] == [("append", 2, 5)]
    assert base._multi.starts == [0, 10, 20, 35]
    lib.calls.clear()
    v, _ = O.make_corpus(60, 8, seed=4)       # 65 of 95 rows in the last block: re-split
    base.add_embeddings(None, v)
    _check_all(base, lib, q)
    assert base._multi.starts == [0, 32, 64, 95]
    changes = [c for c in lib.calls if c[0] != "mask"]
    assert ("append", 0, 22) in changes and ("clear", 1, None) in changes and ("clear", 2, None) in changes


def test_removals_and_overwrites_go_to_the_owning_shards(lib):
    base, q = _make(3, 30)
    _check_all(base, lib, q)
    lib.calls.clear()
    base.remove_embeddings([11, 12, 29, -30])
    assert [c for c in lib.calls] == [("remove", 0, [0]), ("remove", 1, [1, 2]), ("remove", 2, [9])]
    assert base._multi.starts == [0, 9, 17, 26]
    _check_all(base, lib, q)
    lib.calls.clear()
    base.remove_embeddings(list(range(9, 17)))   # empties block 1
    assert base._multi.starts == [0, 9, 9, 18]
    _check_all(base, lib, q)
    lib.calls.clear()
    rows, _ = O.make_corpus(4, 8, seed=9)
    base.set_embeddings_at(7, rows)              # rows 7..10 across blocks 0 and 2
    assert [c for c in lib.calls if c[0] == "write"] == [("write", 0, (7, 2)), ("write", 2, (0, 2))]
    _check_all(base, lib, q)


def test_clear_deserialize_and_vectors_setter_reload_every_shard(lib):
    base, q = _make(3, 30)
    _check_all(base, lib, q)
    v, _ = O.make_corpus(7, 8, seed=5)
    base.deserialize(v)
    lib.calls.clear()
    _check_all(base, lib, q)
    assert sorted(c[:2] for c in lib.calls if c[0] in ("clear", "append")) == [
        ("append", 0), ("append", 1), ("append", 2), ("clear", 0), ("clear", 1), ("clear", 2)]
    base.clear()
    assert base.search_arrays(q, 3)[2].tolist() == [0, 0, 0, 0]
    base._vectors = O.make_corpus(2, 8, seed=6)[0]
    _check_all(base, lib, q)
    assert base._multi.starts == [0, 1, 2, 2]


def test_fewer_rows_than_shards(lib):
    base, q = _make(8, 3)
    _check_all(base, lib, q)
    assert base._multi.starts == [0, 1, 2, 3, 3, 3, 3, 3, 3]


def test_predicate_mask_is_cut_per_block(lib):
    base, q = _make(3, 50)
    # below _PREDICATE_MASK_ROWS rows the predicate becomes a row mask up front
    hits = base.fuzzy_lookup_embedding(q[0], max_hits=6, predicate=lambda i: i % 2 == 0)
    allowed = np.arange(50) % 2 == 0
    keys, s = _ranked(base._vectors, q[0], np.float32(0), True, allowed)
    assert [(h.item, h.score) for h in hits] == list(zip(keys[:6].tolist(), s[:6].tolist()))
    assert sorted(g for name, g, _ in lib.calls if name == "mask") == [0, 1, 2]
    assert lib.searches[-1][1] & _capi.TAV_TIES_LOW_FIRST


def test_k_beyond_the_merge_is_served_by_the_threshold_search(lib):
    base, q = _make(2, MERGE_MAX_K + 10, d=4)
    items, scores, counts = base.search_arrays(q[:1], MERGE_MAX_K + 5)
    assert lib.searches[-1][0] == "range"
    want_items, want_scores = _expect_topk(base, q[:1], MERGE_MAX_K + 5)[0]
    assert items[0, :counts[0]].tolist() == want_items and scores[0, :counts[0]].tolist() == want_scores

