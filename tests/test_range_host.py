"""Host logic of the threshold search (``VectorBase.search_range`` and ``fuzzy_lookup_embeddings(max_hits=0)``)
on CPU: ``tav_range_search`` / ``tav_range_fetch`` are served by a FakeLib that computes the hits with the
oracle, so what is tested is the Python side — CSR assembly, the capacity hint carried from one search to the
next, argument checks and the lists built from the CSR result."""

from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import typeagent_py_b200 as tab
from oracle import vectorbase_oracle as O
from tests.fake_lib import FakeLib, _addr, _view
from tests.parity import assert_hits_match
from typeagent_py_b200 import _capi


class RangeFakeLib(FakeLib):
    """FakeLib plus the two threshold-search entry points (oracle arithmetic, the library's tie order)."""

    def __init__(self, base):
        super().__init__(base)
        self.range_calls = []   # (n_queries, min_score, flags, subset_len, expected_hits)
        self.hits = ([], [])

    def tav_range_search(self, ix, qp, nq, floor, flags, sub_ptr, sub_len, item_offset, expected, op, stream):
        floor = float(getattr(floor, "value", floor))
        v = self.base._vectors
        dim = v.shape[1]
        q = _view(qp, C.c_float, nq * dim).reshape(nq, dim).copy()
        sub = _view(sub_ptr, C.c_int64, sub_len).copy() if _addr(sub_ptr) else None
        self.range_calls.append((nq, floor, flags, None if sub is None else len(sub), expected))
        offsets = _view(op, C.c_int64, nq + 1)
        items, scores = [], []
        offsets[0] = 0
        for b in range(nq):
            rows = v if sub is None else v[sub]
            with np.errstate(invalid="ignore"):
                s = O.score_from_cosine(rows @ q[b]).astype(np.float32)
                ok = s >= np.float32(floor)
            if flags & _capi.TAV_USE_ROW_MASK:
                ok &= self.mask
            pos = np.flatnonzero(ok)
            tie = pos if flags & _capi.TAV_TIES_LOW_FIRST else -pos
            order = pos[np.lexsort((tie, -s[pos]))]
            items += [int(sub[p]) if sub is not None else int(p) for p in order]
            scores += [float(s[p]) for p in order]
            offsets[b + 1] = len(items)
        self.hits = (items, scores)
        return 0

    def tav_range_fetch(self, ix, first, n, ip, sp, flags, stream):
        _view(ip, C.c_int64, n)[:] = self.hits[0][first:first + n]
        _view(sp, C.c_float, n)[:] = self.hits[1][first:first + n]
        return 0


def make(v):
    base = tab.VectorBase(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()))
    base.add_embeddings(None, v)
    fake = RangeFakeLib(base)
    base._ensure_device = lambda: (fake, None)
    return base, fake


def test_csr_result_per_query():
    v, q = O.make_corpus(400, 16, seed=3, n_queries=4)
    base, fake = make(v)
    offsets, items, scores = base.search_range(q, 0.55)
    assert offsets.dtype == np.int64 and items.dtype == np.int64 and scores.dtype == np.float32
    assert offsets.shape == (5,) and offsets[0] == 0 and offsets[-1] == len(items) == len(scores)
    assert (np.diff(offsets) >= 0).all()
    for b in range(4):
        got = {"items": items[offsets[b]:offsets[b + 1]].tolist(), "scores": scores[offsets[b]:offsets[b + 1]].tolist()}
        assert_hits_match(got, O.lookup(v, q[b], len(v), 0.55), min_score=0.55, what=f"q{b}")
    one = base.search_range(q[1], 0.55)  # a single query as a 1-D vector
    np.testing.assert_array_equal(one[1], items[offsets[1]:offsets[2]])


def test_capacity_hint_is_the_previous_total():
    v, q = O.make_corpus(300, 8, seed=5, n_queries=3)
    base, fake = make(v)
    first = base.search_range(q, 0.5)
    second = base.search_range(q[:1], 0.9)
    base.search_range(q, 0.0)
    assert [c[4] for c in fake.range_calls] == [0, int(first[0][-1]), int(second[0][-1])]


def test_empty_inputs_need_no_library_call():
    v, q = O.make_corpus(50, 8, seed=7, n_queries=2)
    base, fake = make(v)
    for offsets, items, scores in (base.search_range(q, float("nan")), base.search_range(q[:0], 0.0),
                                   base.search_range(q, 0.0, subset=[])):
        assert (offsets == 0).all() and len(items) == len(scores) == 0
    assert base.search_range(q, float("nan"))[0].shape == (3,)
    assert fake.range_calls == []
    empty = tab.VectorBase(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()))
    assert empty.fuzzy_lookup_embeddings(np.zeros((2, 3), np.float32), max_hits=0) == [[], []]


def test_argument_errors():
    v, q = O.make_corpus(60, 8, seed=9, n_queries=2)
    base, fake = make(v)
    with pytest.raises(ValueError, match="cannot be combined"):
        base.search_range(q, 0.0, subset=[1, 2], allowed=np.ones(60, bool))
    with pytest.raises(ValueError):
        base.search_range(np.zeros((2, 5), np.float32), 0.0)      # wrong width
    with pytest.raises(IndexError):
        base.search_range(q, 0.0, subset=[1.5, 2.0])               # non-integer ordinals
    with pytest.raises(ValueError):
        base.search_range(q, 0.0, allowed=np.ones(59, bool))       # mask of the wrong length
    assert fake.range_calls == []


def test_subset_mask_and_tie_order_are_passed_through():
    v, q = O.make_corpus(200, 8, seed=11, n_queries=1)
    v[10] = v[20] = v[30]  # exact ties
    base, fake = make(v)
    hi = base.search_range(q, 0.0)[1].tolist()
    lo = base.search_range(q, 0.0, ties_low_first=True)[1].tolist()
    assert fake.range_calls[-1][2] & _capi.TAV_TIES_LOW_FIRST
    pos = [hi.index(r) for r in (10, 20, 30)]
    assert [hi[p] for p in sorted(pos)] == [30, 20, 10] and [lo[p] for p in sorted(pos)] == [10, 20, 30]
    sub = [5, -1, 5, 7]
    offsets, items, _ = base.search_range(q, 0.0, subset=sub)
    assert fake.range_calls[-1][3] == 4 and sorted(items.tolist()) == sorted(sub)
    allowed = np.arange(200) % 3 == 0
    _, items, _ = base.search_range(q, 0.0, allowed=allowed)
    assert fake.range_calls[-1][2] & _capi.TAV_USE_ROW_MASK and all(i % 3 == 0 for i in items)


@pytest.mark.parametrize("min_score", [0.0, 0.5, 0.62, 1.5])
def test_fuzzy_lookup_embeddings_max_hits_0_is_the_oracle_lookup(min_score):
    v, q = O.make_corpus(500, 24, seed=13, n_queries=5)
    base, fake = make(v)
    got = base.fuzzy_lookup_embeddings(q, max_hits=0, min_score=min_score)
    assert len(fake.range_calls) == 1 and fake.searches == []  # one threshold search, no [B, N] arrays
    for b in range(5):
        assert all(isinstance(h, tab.ScoredInt) for h in got[b])
        assert_hits_match(got[b], O.lookup(v, q[b], 0, min_score), min_score=min_score, what=f"q{b}")
    # other max_hits values keep the top-k search
    base.fuzzy_lookup_embeddings(q, max_hits=7, min_score=min_score)
    assert len(fake.searches) == 1 and fake.searches[0][1] == 7
