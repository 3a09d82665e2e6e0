"""Host logic of row removal and overwrite (``VectorBase.remove_embeddings`` / ``set_embeddings_at`` and
friends, ``EmbeddingIndex.remove_at``) on CPU, through a stand-in for libtavec.

The stand-in keeps its own copy of the "device" rows and changes it only through the entry points the class
calls (append, clear, remove, write), and its searches read that copy.  So the tests see what the class sends
to the library: the removal list and the overwritten rows, no re-upload (no clear, no re-append), the
generation kept, the row mask dropped on removal, and the device rows equal to the host mirror afterwards.  The
library itself is covered on the GPU by tests/test_gpu_remove.py.
"""

from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import typeagent_py_b200 as tab
from oracle import vectorbase_oracle as O
from typeagent_py_b200 import _capi


def _view(addr, ctype, n):
    addr = C.cast(addr, C.c_void_p).value if not isinstance(addr, int) else addr
    return np.ctypeslib.as_array(C.cast(addr, C.POINTER(ctype)), (n,)).copy() if n else np.zeros(0)


class StandInLib:
    """The entry points VectorBase calls, over a numpy copy of the device rows (test infrastructure)."""

    def __init__(self):
        self.rows = None
        self.dim = 0
        self.calls = []   # (name, detail) of every row-changing call
        self.mask = None  # bool [rows] or None (dropped)
        self.mask_uploads = 0

    def tav_last_error(self):
        return self.error.encode()

    def _fail(self, rc, msg):
        self.error = msg
        return rc

    def tav_create(self, device, dim, dtype, flags, reserve, out):
        out._obj.value = 1
        return 0

    def tav_destroy(self, ix):
        return 0

    def tav_set_timing(self, ix, on):
        return 0

    def tav_dim(self, ix):
        return self.dim

    def tav_clear(self, ix):
        self.calls.append(("clear", None))
        self.rows = None
        self.mask = None
        return 0

    def tav_append(self, ix, ptr, n, dim, dtype, on_device, stream):
        self.calls.append(("append", n))
        self.dim = dim
        new = _view(ptr, C.c_float, n * dim).reshape(n, dim).astype(np.float32)
        self.rows = new if self.rows is None else np.concatenate([self.rows, new])
        return 0

    def tav_remove_rows(self, ix, ptr, n, stream):
        ords = _view(ptr, C.c_int64, n).astype(np.int64)
        self.calls.append(("remove", ords.tolist()))
        if ((ords < -len(self.rows)) | (ords >= len(self.rows))).any():
            return self._fail(_capi.TAV_ERR_RANGE, "index out of bounds")
        self.rows = np.delete(self.rows, ords, axis=0)
        self.mask = None
        return 0

    def tav_write_rows(self, ix, first, ptr, n, dim, dtype, on_device, stream):
        self.calls.append(("write", (first, n)))
        if first < 0 or first + n > len(self.rows):
            return self._fail(_capi.TAV_ERR_RANGE, "rows out of range")
        self.rows[first:first + n] = _view(ptr, C.c_float, n * dim).reshape(n, dim)
        return 0

    def tav_set_row_mask(self, ix, bits, n_rows, on_device, stream):
        words = _view(bits, C.c_uint32, (n_rows + 31) // 32).astype(np.uint32)
        self.mask = np.unpackbits(words.view(np.uint8), bitorder="little")[:n_rows].astype(bool)
        self.mask_uploads += 1
        return 0

    def tav_search(self, ix, qp, nq, k, floor, flags, sub_ptr, sub_len, item_offset, ip, sp, cp, stream):
        floor = float(getattr(floor, "value", floor))
        v, dim = self.rows, self.dim
        q = _view(qp, C.c_float, nq * dim).reshape(nq, dim)
        items = np.ctypeslib.as_array(C.cast(ip, C.POINTER(C.c_int64)), (nq * k,)).reshape(nq, k)
        scores = np.ctypeslib.as_array(C.cast(sp, C.POINTER(C.c_float)), (nq * k,)).reshape(nq, k)
        counts = np.ctypeslib.as_array(C.cast(cp, C.POINTER(C.c_int32)), (nq,))
        for b in range(nq):
            if flags & _capi.TAV_USE_ROW_MASK:
                assert self.mask is not None and len(self.mask) == len(v), "masked search without a current mask"
                mask = self.mask
                hits = O.lookup(v, q[b], k, floor, predicate=lambda i: bool(mask[i]))
            else:
                hits = O.lookup(v, q[b], k, floor)
            counts[b] = len(hits)
            for j, h in enumerate(hits):
                items[b, j], scores[b, j] = h.item + item_offset, h.score
        return 0

    def row_changes(self):
        return [c for c in self.calls if c[0] in ("clear", "append", "remove", "write")]


@pytest.fixture
def lib(monkeypatch):
    stand_in = StandInLib()
    monkeypatch.setattr(_capi, "load", lambda: stand_in)
    return stand_in


def make(n=40, d=8, seed=0):
    v, q = O.make_corpus(n, d, seed=seed, n_queries=3)
    base = tab.VectorBase(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()))
    base.add_embeddings(None, v)
    return base, v, q


def lookups(base, q, k=6):
    return [[(h.item, h.score) for h in base.fuzzy_lookup_embedding(qq, k, 0.0)] for qq in q]


def fresh_lookups(rows, q, k=6):
    return [[(h.item, h.score) for h in O.lookup(rows, qq, k, 0.0)] for qq in q]


REMOVALS = {
    "none": [],
    "first": [0],
    "last": [39],
    "negative": [-1, -40],
    "repeated, unordered": [7, 3, 7, 3, 30],
    "every other row": list(range(0, 40, 2)),
    "one long run": list(range(5, 33)),
    "all rows": list(range(40)),
    "numpy array": np.array([[1, 2], [38, -3]]),
}


@pytest.mark.parametrize("kind", list(REMOVALS))
def test_remove_is_np_delete_on_host_and_device_without_reupload(lib, kind):
    base, v, q = make()
    lookups(base, q)  # the device copy exists and is current
    before = list(lib.row_changes())
    gen = base._generation
    base.remove_embeddings(REMOVALS[kind])
    want = np.delete(v, REMOVALS[kind], axis=0)
    np.testing.assert_array_equal(base.serialize(), want)
    assert len(base) == len(want) and base._ix_rows == len(want) and base._generation == gen
    np.testing.assert_array_equal(lib.rows, want)
    new_calls = lib.row_changes()[len(before):]
    if np.size(REMOVALS[kind]):
        assert [c[0] for c in new_calls] == ["remove"]
        assert new_calls[0][1] == sorted(set(int(i) % 40 for i in np.ravel(REMOVALS[kind])))
    else:
        assert new_calls == []
    if len(want):
        assert lookups(base, q) == fresh_lookups(want, q)
    assert lib.row_changes()[len(before):] == new_calls, "a lookup after the removal must not re-upload"


def test_boolean_mask_removes_its_rows(lib):
    base, v, q = make()
    lookups(base, q)
    mask = np.arange(40) % 3 == 1
    base.remove_embeddings(mask)
    np.testing.assert_array_equal(base.serialize(), np.delete(v, mask, axis=0))
    np.testing.assert_array_equal(lib.rows, np.delete(v, mask, axis=0))
    assert lib.calls[-1] == ("remove", np.flatnonzero(mask).tolist())


@pytest.mark.parametrize("bad", [[40], [-41], [3, 40], np.array([1.0]), ["a"], np.ones(39, bool),
                                 np.ones((2, 40), bool)])
def test_invalid_removal_leaves_everything_unchanged(lib, bad):
    base, v, q = make()
    lookups(base, q)
    calls = len(lib.calls)
    with pytest.raises(ValueError if np.asarray(bad).dtype == bool else IndexError):
        np.delete(v, bad, axis=0)  # numpy's own error for the same argument
    with pytest.raises(ValueError if np.asarray(bad).dtype == bool else IndexError):
        base.remove_embeddings(bad)
    np.testing.assert_array_equal(base.serialize(), v)
    np.testing.assert_array_equal(lib.rows, v)
    assert len(lib.calls) == calls and len(base) == 40 and base._ix_rows == 40


def test_remove_embedding_at_and_embedding_index_remove_at(lib):
    base, v, q = make()
    with pytest.raises(IndexError, match="Index 40 out of bounds for embedding index of size 40"):
        base.remove_embedding_at(40)
    with pytest.raises(IndexError, match="Index -1 out of bounds"):
        base.remove_embedding_at(-1)  # positions, unlike ordinals, do not wrap
    base.remove_embedding_at(4)
    np.testing.assert_array_equal(base.serialize(), np.delete(v, 4, axis=0))

    ix = tab.EmbeddingIndex(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()), v)
    with pytest.raises(IndexError, match="Index 40 out of bounds for embedding index of size 40"):
        ix.remove_at(40)
    ix.remove_at(0)
    ix.remove_at(len(ix) - 1)
    np.testing.assert_array_equal(ix.serialize(), v[1:-1])


def test_removal_before_pending_appends_reach_the_device(lib):
    base, v, q = make()
    lookups(base, q)
    extra = O.make_corpus(10, 8, seed=1)[0]
    base.add_embeddings(None, extra)  # host only until the next lookup
    both = np.concatenate([v, extra])
    base.remove_embeddings([2, 39, 40, 45])  # two on the device, two not yet there
    want = np.delete(both, [2, 39, 40, 45], axis=0)
    assert lib.calls[-1] == ("remove", [2, 39])
    assert base._ix_rows == 38
    assert lookups(base, q) == fresh_lookups(want, q)
    np.testing.assert_array_equal(lib.rows, want)


def test_removal_without_a_device_copy_touches_only_the_host(lib):
    base, v, _ = make()
    base.remove_embeddings([0, 1])
    assert lib.calls == []
    np.testing.assert_array_equal(base.serialize(), v[2:])


def test_rows_adopted_from_deserialize_are_not_written(lib):
    base, v, q = make()
    data = v.copy()
    base.deserialize(data)
    lookups(base, q)
    base.remove_embeddings([0])
    base.set_embeddings_at(0, np.zeros((1, 8), np.float32))
    np.testing.assert_array_equal(data, v)
    want = np.delete(v, 0, axis=0)
    want[0] = 0
    np.testing.assert_array_equal(base.serialize(), want)
    np.testing.assert_array_equal(lib.rows, want)


def test_removal_drops_row_and_predicate_masks_even_back_at_the_old_size(lib):
    base, v, q = make()
    allowed = np.arange(40) % 3 != 0
    base.search_arrays(q, 5, 0.0, allowed=allowed)
    pred = lambda i: i % 2 == 0  # noqa: E731
    base.fuzzy_lookup_embedding(q[0], 5, 0.0, predicate=pred)
    assert base._predicate_masks and lib.mask_uploads == 2
    base.remove_embeddings([0])
    assert base._predicate_masks == {} and base._mask_key is None and lib.mask is None
    base.add_embedding(None, v[0])  # back to 40 rows, same generation
    rows = np.concatenate([v[1:], v[:1]])
    got = base.search_arrays(q, 5, 0.0, allowed=allowed)
    assert lib.mask_uploads == 3, "the mask of the old ordinals must not be reused"
    want = [O.lookup(rows, qq, 5, 0.0, predicate=lambda i: bool(allowed[i])) for qq in q]
    assert [list(got[0][b, :got[2][b]]) for b in range(3)] == [[h.item for h in w] for w in want]
    hits = base.fuzzy_lookup_embedding(q[0], 5, 0.0, predicate=pred)
    assert [h.item for h in hits] == [h.item for h in O.lookup(rows, q[0], 5, 0.0, predicate=pred)]


def test_overwrite_updates_host_and_device_in_place(lib):
    base, v, q = make()
    allowed = np.arange(40) % 2 == 0
    base.search_arrays(q, 5, 0.0, allowed=allowed)
    gen, uploads = base._generation, lib.mask_uploads
    new = O.make_corpus(5, 8, seed=2)[0]
    base.set_embeddings_at(10, new)
    base.set_embedding_at(39, new[0])
    want = v.copy()
    want[10:15] = new
    want[39] = new[0]
    np.testing.assert_array_equal(base.serialize(), want)
    np.testing.assert_array_equal(lib.rows, want)
    assert [c[0] for c in lib.row_changes()] == ["clear", "append", "write", "write"]
    assert base._generation == gen
    base.search_arrays(q, 5, 0.0, allowed=allowed)
    assert lib.mask_uploads == uploads, "an overwrite keeps the ordinals, so the mask stays"
    assert lookups(base, q) == fresh_lookups(want, q)


def test_overwrite_errors(lib):
    base, v, q = make()
    lookups(base, q)
    calls = len(lib.calls)
    with pytest.raises(ValueError, match="Embedding size mismatch: expected 8, got 7"):
        base.set_embeddings_at(0, np.zeros((2, 7), np.float32))
    with pytest.raises(ValueError, match="Expected 2D"):
        base.set_embeddings_at(0, np.zeros(8, np.float32))
    with pytest.raises(IndexError):
        base.set_embeddings_at(39, np.zeros((2, 8), np.float32))
    with pytest.raises(IndexError):
        base.set_embeddings_at(-1, np.zeros((1, 8), np.float32))
    with pytest.raises(IndexError, match="Index 40 out of bounds"):
        base.set_embedding_at(40, np.zeros(8, np.float32))
    with pytest.raises(ValueError, match="Embedding size mismatch"):
        base.set_embedding_at(0, np.zeros(9, np.float32))
    assert len(lib.calls) == calls
    np.testing.assert_array_equal(base.serialize(), v)


def test_device_only_rows_cannot_change(lib):
    base, _, _ = make()
    base._device_only_rows = 5  # what from_device_tensor leaves (it needs a CUDA tensor)
    with pytest.raises(RuntimeError):
        base.remove_embeddings([0])
    with pytest.raises(RuntimeError):
        base.set_embeddings_at(0, np.zeros((1, 8), np.float32))
