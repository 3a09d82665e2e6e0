"""Host logic of per-query subsets (``subsets=``, ``fuzzy_lookup_embeddings_in_subsets``) through a stand-in of the
library: the CSR layout handed to ``tav_search_subsets``, argument errors, ``k``, the ``max_hits=0`` routing, empty
subsets and the ``EmbeddingIndex`` delegation.  Runs without a GPU."""

from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import typeagent_py_b200 as tab
from oracle import vectorbase_oracle as O
from tests.fake_lib import FakeLib, _view
from typeagent_py_b200 import _capi


class SubsetsLib(FakeLib):
    """FakeLib plus the two subsets entry points: query b is the stand-in's one-query subset search."""

    def __init__(self, base):
        super().__init__(base)
        self.calls = []       # (entry point, n_queries, k, flags, offsets, ordinals)
        self.hits = None      # (items, scores) of the last threshold search

    def _csr(self, nq, offp, ordp):
        offsets = _view(offp, C.c_int64, nq + 1).copy()
        ordinals = _view(ordp, C.c_int64, int(offsets[-1])).copy() if offsets[-1] else np.empty(0, np.int64)
        return offsets, ordinals

    def _one(self, q, k, floor, flags, sub):
        items, scores, counts = np.zeros((1, k), np.int64), np.zeros((1, k), np.float32), np.zeros(1, np.int32)
        if len(sub):
            sub = np.ascontiguousarray(sub)
            super().tav_search(None, q.ctypes.data, 1, k, floor, flags, sub.ctypes.data, len(sub), 0,
                               items.ctypes.data, scores.ctypes.data, counts.ctypes.data, None)
        return items[0, :counts[0]], scores[0, :counts[0]]

    def tav_search_subsets(self, ix, qp, nq, k, floor, flags, offp, ordp, ip, sp, cp, stream):
        floor = float(getattr(floor, "value", floor))
        dim = self.base._vectors.shape[1]
        q = _view(qp, C.c_float, nq * dim).reshape(nq, dim).copy()
        offsets, ordinals = self._csr(nq, offp, ordp)
        self.calls.append(("topk", nq, k, flags, offsets, ordinals))
        items = _view(ip, C.c_int64, nq * k).reshape(nq, k)
        scores = _view(sp, C.c_float, nq * k).reshape(nq, k)
        counts = _view(cp, C.c_int32, nq)
        items[:], scores[:] = -1, 0
        for b in range(nq):
            it, sc = self._one(q[b], k, floor, flags, ordinals[offsets[b]:offsets[b + 1]])
            counts[b] = len(it)
            items[b, :len(it)], scores[b, :len(it)] = it, sc
        return 0

    def tav_range_search_subsets(self, ix, qp, nq, floor, flags, offp, ordp, outp, stream):
        floor = float(getattr(floor, "value", floor))
        dim = self.base._vectors.shape[1]
        q = _view(qp, C.c_float, nq * dim).reshape(nq, dim).copy()
        offsets, ordinals = self._csr(nq, offp, ordp)
        self.calls.append(("range", nq, None, flags, offsets, ordinals))
        out = _view(outp, C.c_int64, nq + 1)
        parts = [self._one(q[b], max(1, offsets[b + 1] - offsets[b]), floor, flags,
                           ordinals[offsets[b]:offsets[b + 1]]) for b in range(nq)]
        out[0] = 0
        out[1:] = np.cumsum([len(p[0]) for p in parts])
        self.hits = (np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]))
        return 0

    def tav_range_fetch(self, ix, first, n, ip, sp, flags, stream):
        _view(ip, C.c_int64, n)[:] = self.hits[0][first:first + n]
        _view(sp, C.c_float, n)[:] = self.hits[1][first:first + n]
        return 0


def setup(n=400, d=16, b=5, seed=0):
    v, q = O.make_corpus(n, d, seed=seed, n_queries=b)
    base = tab.VectorBase(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()))
    base.add_embeddings(None, v)
    fake = SubsetsLib(base)
    base._ensure_device = lambda: (fake, None)
    return base, fake, v, q


SUBSETS = [[3, 3, -1, 17], list(range(0, 400, 3)), [], np.array([5], np.int32), np.arange(-50, 0).reshape(5, 10)]


def test_csr_layout_and_flags():
    base, fake, _, q = setup()
    base.search_arrays(q, 7, 0.25, subsets=SUBSETS, ties_low_first=True)
    kind, nq, k, flags, offsets, ordinals = fake.calls[-1]
    assert kind == "topk" and nq == 5 and k == 7 and flags == _capi.TAV_TIES_LOW_FIRST
    assert offsets.tolist() == [0, 4, 4 + 134, 138, 139, 189]
    assert ordinals.tolist() == [3, 3, -1, 17, *range(0, 400, 3), 5, *range(-50, 0)]
    base.force_path = "scan"   # the path options are not subsets flags
    base.search_range(q, 0.25, subsets=SUBSETS)
    assert fake.calls[-1][0] == "range" and fake.calls[-1][3] == 0


def test_rows_equal_one_query_searches_and_k_is_the_longest_subset():
    base, fake, _, q = setup()
    for k in (1, 5, 134, 1000):
        items, scores, counts = base.search_arrays(q, k, 0.3, subsets=SUBSETS)
        assert items.shape == (5, min(k, 134))
        for b, sub in enumerate(SUBSETS):
            i1, s1, c1 = base.search_arrays(q[b:b + 1], k, 0.3, subset=np.asarray(sub).reshape(-1))
            kb = i1.shape[1]
            assert counts[b] == c1[0]
            assert items[b, :kb].tolist() == i1[0].tolist() and scores[b, :kb].tolist() == s1[0].tolist()
            assert (items[b, kb:] == -1).all() and (scores[b, kb:] == 0).all()


def test_empty_cases_do_no_work():
    base, fake, _, q = setup()
    items, scores, counts = base.search_arrays(q[:2], 4, 0.0, subsets=[[], []])
    assert items.shape == (2, 1) and (items == -1).all() and (counts == 0).all()
    items, _, counts = base.search_arrays(q[:2], 4, float("nan"), subsets=[[1], [2]])
    assert (counts == 0).all()
    offsets, items, scores = base.search_range(q[:2], 0.0, subsets=[[], []])
    assert offsets.tolist() == [0, 0, 0] and len(items) == 0 and len(scores) == 0
    assert base.search_arrays(q[:0], 4, 0.0, subsets=[])[0].shape == (0, 1)
    assert fake.calls == []


def test_errors_before_any_work():
    base, fake, _, q = setup()
    with pytest.raises(ValueError, match="4 subsets for 5 queries"):
        base.search_arrays(q, 5, subsets=SUBSETS[:4])
    with pytest.raises(ValueError, match="4 subsets for 5 queries"):
        base.search_range(q, 0.0, subsets=SUBSETS[:4])
    with pytest.raises(ValueError, match="cannot be combined"):
        base.search_arrays(q, 5, subsets=SUBSETS, subset=[1, 2])
    with pytest.raises(ValueError, match="cannot be combined"):
        base.search_arrays(q, 5, subsets=SUBSETS, allowed=np.ones(400, bool))
    with pytest.raises(ValueError, match="cannot be combined"):
        base.search_range(q, 0.0, subsets=SUBSETS, subset=[1])
    with pytest.raises(IndexError, match="must be of integer"):
        base.search_arrays(q, 5, subsets=[[1], [0.5], [], [2], [3]])
    with pytest.raises(IndexError, match="must be of integer"):
        base.search_range(q, 0.0, subsets=[[1], [True], [], [2], [3]])
    with pytest.raises(ValueError, match="max_hits must be >= 0"):
        base.fuzzy_lookup_embeddings_in_subsets(q, SUBSETS, -1)
    with pytest.raises(ValueError, match="Expected 2D"):
        base.fuzzy_lookup_embeddings_in_subsets(q[0], SUBSETS[:1])
    assert fake.calls == []


@pytest.mark.parametrize("max_hits", [None, 0, 1, 5, 500])
@pytest.mark.parametrize("min_score", [None, 0.4])
def test_fuzzy_lookup_embeddings_in_subsets_equals_the_per_query_lookup(max_hits, min_score):
    base, fake, _, q = setup()
    subsets = [list(np.asarray(s).reshape(-1)) for s in SUBSETS]
    got = base.fuzzy_lookup_embeddings_in_subsets(q, subsets, max_hits, min_score)
    assert fake.calls[-1][0] == ("range" if max_hits == 0 else "topk")
    if max_hits is None:
        assert fake.calls[-1][2] == 10
    for b in range(len(q)):
        want = base.fuzzy_lookup_embedding_in_subset(q[b], subsets[b], max_hits, min_score)
        assert [(h.item, h.score) for h in got[b]] == [(h.item, h.score) for h in want]


def test_embedding_index_delegates():
    _, _, v, q = setup()
    index = tab.EmbeddingIndex(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()), v)
    vb = index._vector_base
    fake = SubsetsLib(vb)
    vb._ensure_device = lambda: (fake, None)
    got = index.get_indexes_of_nearest_in_subsets_batch(q, SUBSETS, 3, 0.2)
    want = vb.fuzzy_lookup_embeddings_in_subsets(q, SUBSETS, 3, 0.2)
    assert [[(h.item, h.score) for h in r] for r in got] == [[(h.item, h.score) for h in r] for r in want]
