"""Grouped lookups on CPU: the numpy statement of their semantics (also the GPU tests' oracle), checked against the
reference's own chunk -> message fold, and the host logic of ``search_groups`` / ``search_range_groups`` /
``fuzzy_lookup_embedding_grouped`` through a stand-in library.  Runs without a GPU."""

from __future__ import annotations

import ctypes as C
import sys

import numpy as np
import pytest

import typeagent_py_b200 as tab
from oracle import ref_loader
from oracle import vectorbase_oracle as O
from tests.fake_lib import FakeLib, _view
from typeagent_py_b200 import _capi


# ---------------------------------------------------------------------------------------------- the oracle
def grouped_hits(scores, groups, min_score=0.0, allowed=None, ties_low_first=False):
    """One query's grouped threshold search: (groups int64, scores float32, rows int64) of every group's leader.

    The hit list is the library's: rows with float32 score >= float32(min_score) (and ``allowed``), by score
    descending, equal scores by row descending (ascending with ``ties_low_first``).  A group's leader is its first
    row in that list; the result lists the leaders in that order."""
    s = np.asarray(scores, np.float32)
    groups = np.asarray(groups, np.int64)
    with np.errstate(invalid="ignore"):
        ok = s >= np.float32(min_score)
    if allowed is not None:
        ok &= np.asarray(allowed, bool)
    rows = np.flatnonzero(ok)
    order = np.lexsort((rows if ties_low_first else -rows, -s[rows].astype(np.float64)))
    rows = rows[order]
    _, first = np.unique(groups[rows], return_index=True)
    lead = rows[np.sort(first)]
    return groups[lead], s[lead], lead.astype(np.int64)


def grouped_topk(scores_bn, groups, k, min_score=0.0, allowed=None, ties_low_first=False):
    """``search_groups``' arrays for scores float32 [B, N]: group ids, scores, rows [B, k] and counts [B].
    ``allowed``: bool [N], or bool [B, N] (one mask per query)."""
    b = len(scores_bn)
    g_out = np.full((b, k), -1, np.int64)
    s_out = np.zeros((b, k), np.float32)
    r_out = np.full((b, k), -1, np.int64)
    counts = np.zeros(b, np.int32)
    for i in range(b):
        a = None if allowed is None else (allowed[i] if np.ndim(allowed) == 2 else allowed)
        g, s, r = grouped_hits(scores_bn[i], groups, min_score, a, ties_low_first)
        n = min(k, len(g))
        g_out[i, :n], s_out[i, :n], r_out[i, :n], counts[i] = g[:n], s[:n], r[:n], n
    return g_out, s_out, r_out, counts


def first_occurrences(items, scores, groups):
    """The first hit of every group in one query's ``search_range`` list: (groups, scores, rows)."""
    g = np.asarray(groups, np.int64)[items]
    _, first = np.unique(g, return_index=True)
    keep = np.sort(first)
    return g[keep], scores[keep], items[keep]


def _scores(v, q):
    return O.score_from_cosine(np.atleast_2d(q) @ v.T).astype(np.float32)


@pytest.fixture
def reference_modules(monkeypatch):
    """The reference's modules for one test only: what it imports under ``typeagent`` (and the loader's stubs) leaves
    ``sys.modules`` afterwards, and the loader forgets it loaded them, so later tests see no typeagent imported."""
    before = set(sys.modules)
    monkeypatch.setattr(ref_loader, "_loaded", ref_loader._loaded)
    yield
    for name in set(sys.modules) - before:
        if name.split(".")[0] in ("typeagent", "typechat", "stamina"):
            del sys.modules[name]


def test_oracle_equals_the_reference_fold(reference_modules):
    """On tie-free data the oracle is the reference's fold of its own every-hit lookup (max_hits=0)."""
    mi = ref_loader.load_reference_module("typeagent.storage.memory.messageindex")
    core = ref_loader.load_reference_module("typeagent.knowpro.interfaces_core")
    tli = ref_loader.load_reference_module("typeagent.knowpro.textlocindex")
    rng = np.random.default_rng(3)
    v, qs = O.make_corpus(500, 24, seed=5, n_queries=4)
    for groups in (np.repeat(np.arange(100), 5), rng.integers(0, 60, 500), np.arange(500)):
        ref = ref_loader.make_reference_vectorbase(v)
        for q, min_score in zip(qs, (0.0, 0.5, 0.55, 0.6)):
            hits = ref.fuzzy_lookup_embedding(q, max_hits=0, min_score=min_score)
            locs = [tli.ScoredTextLocation(core.TextLocation(int(groups[h.item])), h.score) for h in hits]
            folded = mi.MessageTextIndex.to_scored_message_ordinals(None, locs)
            g, s, _ = grouped_hits(_scores(v, q)[0], groups, min_score)
            assert [m.message_ordinal for m in folded] == g.tolist()
            assert np.array_equal(np.float32([m.score for m in folded]), s)


def test_oracle_ties_and_empty_groups():
    s = np.float32([0.5, 0.9, 0.9, 0.1, 0.9, 0.7])
    groups = np.array([0, 1, 2, 3, 1, 0])
    g, sc, r = grouped_hits(s, groups, 0.2)
    assert g.tolist() == [1, 2, 0] and r.tolist() == [4, 2, 5]  # group 3 has no passing row
    g, sc, r = grouped_hits(s, groups, 0.2, ties_low_first=True)
    assert g.tolist() == [1, 2, 0] and r.tolist() == [1, 2, 5]
    g, _, r = grouped_hits(s, groups, 0.2, allowed=[True, False, True, True, True, False])
    assert g.tolist() == [1, 2, 0] and r.tolist() == [4, 2, 0]


# ---------------------------------------------------------------------------------------------- the host logic
class GroupLib(FakeLib):
    """FakeLib plus the grouped entry points, computed with the oracle above."""

    def __init__(self, base):
        super().__init__(base)
        self.groups = None
        self.group_uploads = 0
        self.grouped = []  # (n_queries, k, flags) per grouped search
        self.redo = 0
        self._leaders = None

    def tav_set_row_groups(self, ix, gp, n_rows, on_device, stream):
        assert not on_device
        self.groups = _view(gp, C.c_int32, n_rows).copy()
        self.group_uploads += 1
        return 0

    def _query_inputs(self, qp, nq, flags):
        v = self.base._vectors
        assert self.groups is not None and len(self.groups) == len(v)
        q = _view(qp, C.c_float, nq * v.shape[1]).reshape(nq, v.shape[1]).copy()
        allowed = self.mask if flags & _capi.TAV_USE_ROW_MASK else None
        return _scores(v, q), allowed, bool(flags & _capi.TAV_TIES_LOW_FIRST)

    def tav_search_groups(self, ix, qp, nq, k, floor, flags, gp, sp, rp, cp, stream, redone):
        floor = float(getattr(floor, "value", floor))
        self.grouped.append((nq, k, flags))
        s, allowed, ties = self._query_inputs(qp, nq, flags)
        g, sc, r, c = grouped_topk(s, self.groups, k, floor, allowed, ties)
        _view(gp, C.c_int64, nq * k)[:] = g.ravel()
        _view(sp, C.c_float, nq * k)[:] = sc.ravel()
        _view(rp, C.c_int64, nq * k)[:] = r.ravel()
        _view(cp, C.c_int32, nq)[:] = c
        C.cast(redone, C.POINTER(C.c_int))[0] = self.redo
        return 0

    def tav_range_search_groups(self, ix, qp, nq, floor, flags, hint, op, stream):
        floor = float(getattr(floor, "value", floor))
        self.grouped.append((nq, None, flags))
        s, allowed, ties = self._query_inputs(qp, nq, flags)
        parts = [grouped_hits(s[i], self.groups, floor, allowed, ties) for i in range(nq)]
        offsets = _view(op, C.c_int64, nq + 1)
        offsets[0] = 0
        offsets[1:] = np.cumsum([len(p[0]) for p in parts])
        self._leaders = [np.concatenate([p[j] for p in parts]) if parts else np.empty(0) for j in range(3)]
        return 0

    def tav_range_fetch_groups(self, ix, first, n, gp, sp, rp, flags, stream):
        g, s, r = self._leaders
        _view(gp, C.c_int64, n)[:] = g[first:first + n]
        _view(sp, C.c_float, n)[:] = s[first:first + n]
        _view(rp, C.c_int64, n)[:] = r[first:first + n]
        return 0

    def tav_remove_rows(self, ix, ordinals, n, stream):
        return 0


def setup(n=240, d=16, b=3, seed=0):
    v, q = O.make_corpus(n, d, seed=seed, n_queries=b)
    base = tab.VectorBase(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()))
    base.add_embeddings(None, v)
    fake = GroupLib(base)
    calls = []

    def ensure():
        calls.append(1)
        return fake, None

    base._ensure_device = ensure
    return base, fake, calls, v, q


def test_search_groups_and_range_groups_follow_the_oracle():
    base, fake, _, v, q = setup()
    groups = np.repeat(np.arange(60), 4)
    g, s, r, c = base.search_groups(q, 7, groups, min_score=0.4)
    want = grouped_topk(_scores(v, q), groups, 7, 0.4)
    for got, exp in zip((g, s, r, c), want):
        assert np.array_equal(got, exp)
    assert g.dtype == np.int64 and s.dtype == np.float32 and r.dtype == np.int64 and c.dtype == np.int32
    offsets, g, s, r = base.search_range_groups(q, groups, min_score=0.5, ties_low_first=True)
    scores = _scores(v, q)
    for i in range(len(q)):
        eg, es, er = grouped_hits(scores[i], groups, 0.5, ties_low_first=True)
        sl = slice(offsets[i], offsets[i + 1])
        assert np.array_equal(g[sl], eg) and np.array_equal(s[sl], es) and np.array_equal(r[sl], er)
    assert fake.grouped[-1][2] & _capi.TAV_TIES_LOW_FIRST


def test_k_is_clamped_and_max_hits_defaults():
    base, fake, _, v, q = setup(n=40)
    groups = np.arange(40) % 13
    g, s, r, c = base.search_groups(q, 1000, groups)
    assert g.shape == (len(q), 40) and fake.grouped[-1][1] == 40
    assert (c == 13).all()
    hits = base.fuzzy_lookup_embedding_grouped(q[0], groups)
    assert len(hits) == 10 and fake.grouped[-1][1] == 10
    eg, es, _ = grouped_hits(_scores(v, q[:1])[0], groups)
    assert [h.item for h in hits] == eg[:10].tolist() and [h.score for h in hits] == es[:10].tolist()
    every = base.fuzzy_lookup_embedding_grouped(q[0], groups, max_hits=0)
    assert [h.item for h in every] == eg.tolist()
    assert base.fuzzy_lookup_embedding_grouped(q[0], groups, max_hits=3, min_score=2.0) == []
    with pytest.raises(ValueError):
        base.search_groups(q, 0, groups)


def test_bad_groups_are_refused_before_device_work():
    base, fake, calls, _, q = setup(n=50)
    bad = [np.arange(49), np.arange(50, dtype=np.float64), np.arange(50).reshape(5, 10),
           np.r_[np.arange(49), -1], np.r_[np.arange(49), 2**31], list(range(51))]
    for groups in bad:
        with pytest.raises(ValueError):
            base.search_groups(q, 3, groups)
        with pytest.raises(ValueError):
            base.search_range_groups(q, groups)
        with pytest.raises(ValueError):
            base.fuzzy_lookup_embedding_grouped(q[0], groups)
    assert calls == [] and fake.group_uploads == 0 and fake.grouped == []
    base.search_groups(q, 3, list(range(50)))  # any integer sequence of the right length
    assert fake.group_uploads == 1


def test_one_upload_and_reuploads_after_row_changes():
    base, fake, _, v, q = setup(n=60)
    groups = np.arange(60) // 3
    for _ in range(3):
        base.search_groups(q, 4, groups)
        base.search_range_groups(q, groups)
    assert fake.group_uploads == 1
    base.add_embeddings(None, v[:3])
    groups2 = np.arange(63) // 3
    base.search_groups(q, 4, groups2)
    base.search_groups(q, 4, groups2)
    assert fake.group_uploads == 2
    base.remove_embeddings([0, 1, 2])
    with pytest.raises(ValueError):
        base.search_groups(q, 4, groups2)  # 63 groups for 60 rows
    base.search_groups(q, 4, groups)
    assert fake.group_uploads == 3
    base.deserialize(base.serialize().copy())
    base._ensure_device = lambda: (fake, None)
    base.search_groups(q, 4, groups)
    assert fake.group_uploads == 4
    base.search_groups(q, 4, groups)
    assert fake.group_uploads == 4


def test_last_redone_and_masks_reach_the_library():
    base, fake, _, v, q = setup(n=64)
    groups = np.arange(64) // 8
    fake.redo = 2
    base.search_groups(q, 3, groups)
    assert base.last_redone == 2
    allowed = np.arange(64) % 2 == 0
    g, _, r, _ = base.search_groups(q, 3, groups, allowed=allowed)
    assert fake.grouped[-1][2] & _capi.TAV_USE_ROW_MASK and (r[r >= 0] % 2 == 0).all()
    assert np.array_equal(g, grouped_topk(_scores(v, q), groups, 3, 0.0, allowed)[0])


def test_empty_index_and_nan_floor():
    base = tab.VectorBase(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()))
    assert base.fuzzy_lookup_embedding_grouped(np.ones(3, np.float32), []) == []
    base, fake, _, v, q = setup(n=20)
    g, s, r, c = base.search_groups(q, 5, np.zeros(20, int), min_score=float("nan"))
    assert (c == 0).all() and (g == -1).all() and (r == -1).all() and fake.grouped == []


def test_devices_refusal():
    base = tab.VectorBase(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()), devices=[0, 0])
    q = np.ones((1, 4), np.float32)
    with pytest.raises(NotImplementedError, match="devices="):
        base.search_groups(q, 2, [])
    with pytest.raises(NotImplementedError, match="devices="):
        base.search_range_groups(q, [])
    with pytest.raises(NotImplementedError, match="devices="):
        base.fuzzy_lookup_embedding_grouped(q[0], [])


def test_signatures_are_bound():
    for name in ("tav_set_row_groups", "tav_range_search_groups", "tav_range_fetch_groups", "tav_search_groups"):
        assert name in _capi.SIGNATURES
