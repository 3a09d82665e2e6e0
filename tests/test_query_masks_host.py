"""Host logic of per-query masks (2-D ``allowed=``) through the ``tests/fake_lib.py`` stand-in: packing, shapes,
errors, the upload cache, and B == 1.  Runs without a GPU."""

from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import typeagent_py_b200 as tab
from oracle import vectorbase_oracle as O
from tests.fake_lib import FakeLib, _view
from typeagent_py_b200 import _capi


class QueryMaskLib(FakeLib):
    """FakeLib plus tav_set_query_masks: a TAV_USE_QUERY_MASKS search is one masked search per query."""

    def __init__(self, base):
        super().__init__(base)
        self.qmasks = None
        self.qmask_uploads = 0

    def tav_set_query_masks(self, ix, bits, n_queries, n_rows, stride, on_device, stream):
        assert not on_device
        words = _view(bits, C.c_uint32, n_queries * stride).reshape(n_queries, stride).copy()
        self.qmasks = np.unpackbits(words.view(np.uint8), axis=1, bitorder="little")[:, :n_rows].astype(bool)
        self.qmask_uploads += 1
        return 0

    def tav_search(self, ix, qp, nq, k, floor, flags, sub_ptr, sub_len, item_offset, ip, sp, cp, stream):
        if not flags & _capi.TAV_USE_QUERY_MASKS:
            return super().tav_search(ix, qp, nq, k, floor, flags, sub_ptr, sub_len, item_offset, ip, sp, cp, stream)
        assert len(self.qmasks) == nq and not flags & _capi.TAV_USE_ROW_MASK
        dim = self.base._vectors.shape[1]
        for b in range(nq):
            self.mask = self.qmasks[b]
            row = lambda p, size, i: C.c_void_p(C.cast(p, C.c_void_p).value + i * size)  # noqa: E731
            rc = super().tav_search(ix, row(qp, 4 * dim, b), 1, k, floor,
                                    (flags & ~_capi.TAV_USE_QUERY_MASKS) | _capi.TAV_USE_ROW_MASK, None, 0,
                                    item_offset, row(ip, 8 * k, b), row(sp, 4 * k, b), row(cp, 4, b), stream)
            if rc:
                return rc
        return 0


def setup(n=300, d=16, b=5, seed=0):
    v, q = O.make_corpus(n, d, seed=seed, n_queries=b)
    base = tab.VectorBase(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()))
    base.add_embeddings(None, v)
    fake = QueryMaskLib(base)
    base._ensure_device = lambda: (fake, None)
    return base, fake, v, q


def want(v, q, k, masks):
    out = []
    for b in range(len(q)):
        hits = O.lookup(v, q[b], k, 0.0, predicate=lambda i, m=masks[b]: bool(m[i]))
        hits.sort(key=lambda h: (np.float32(h.score), h.item), reverse=True)
        out.append([h.item for h in hits])
    return out


def test_pack_query_masks_matches_pack_row_mask_per_row():
    rng = np.random.default_rng(1)
    for n in (1, 31, 32, 33, 100, 257):
        m = rng.random((4, n)) < 0.5
        packed = tab.VectorBase.pack_query_masks(m)
        assert packed.dtype == np.uint32 and packed.shape == (4, (n + 31) // 32)
        for b in range(4):
            assert np.array_equal(packed[b], tab.VectorBase.pack_row_mask(m[b]))


@pytest.mark.parametrize("packed", [False, True])
def test_each_query_searches_its_own_rows(packed):
    base, fake, v, q = setup()
    masks = np.random.default_rng(2).random((len(q), len(v))) < 0.3
    allowed = base.pack_query_masks(masks) if packed else masks
    items, _, counts = base.search_arrays(q, 7, 0.0, allowed=allowed)
    assert fake.searches[-1][2] & _capi.TAV_USE_ROW_MASK   # the stand-in's per-query fan-out
    for b, w in enumerate(want(v, q, 7, masks)):
        assert items[b, :counts[b]].tolist() == w
        assert all(masks[b][i] for i in w)


def test_one_query_batch():
    base, fake, v, q = setup(b=1)
    masks = np.random.default_rng(3).random((1, len(v))) < 0.2
    items, _, counts = base.search_arrays(q, 5, 0.0, allowed=masks)
    assert items[0, :counts[0]].tolist() == want(v, q, 5, masks)[0]
    assert fake.qmask_uploads == 1


def test_one_dimensional_allowed_is_unchanged():
    base, fake, v, q = setup()
    mask = np.random.default_rng(4).random(len(v)) < 0.5
    base.search_arrays(q, 5, 0.0, allowed=mask)
    assert fake.qmask_uploads == 0 and fake.mask_uploads == 1
    assert fake.searches[-1][2] & _capi.TAV_USE_ROW_MASK


def test_shape_errors():
    base, _, v, q = setup()
    n = len(v)
    masks = np.ones((len(q), n), bool)
    with pytest.raises(ValueError, match=f"query masks have 4 rows for {len(q)} queries"):
        base.search_arrays(q, 5, 0.0, allowed=masks[:4])
    with pytest.raises(ValueError, match=f"query masks have {n - 1} entries for {n} rows"):
        base.search_arrays(q, 5, 0.0, allowed=masks[:, 1:])
    with pytest.raises(ValueError, match=f"query masks have {32 * ((n + 31) // 32 + 1)} bits for {n} rows"):
        base.search_arrays(q, 5, 0.0, allowed=np.zeros((len(q), (n + 31) // 32 + 1), np.uint32))
    with pytest.raises(ValueError, match="cannot be combined"):
        base.search_arrays(q, 5, 0.0, allowed=masks, subset=[1, 2])


def test_upload_once_per_mask_object_rows_and_generation():
    base, fake, v, q = setup()
    masks = np.random.default_rng(5).random((len(q), len(v))) < 0.5
    for _ in range(3):
        base.search_arrays(q, 5, 0.0, allowed=masks)
    assert fake.qmask_uploads == 1
    other = masks.copy()
    base.search_arrays(q, 5, 0.0, allowed=other)
    assert fake.qmask_uploads == 2
    base.search_arrays(q, 5, 0.0, allowed=other)
    assert fake.qmask_uploads == 2
    base.add_embedding(None, v[0])            # rows changed: the masks no longer fit
    with pytest.raises(ValueError, match="entries for"):
        base.search_arrays(q, 5, 0.0, allowed=other)
    grown = np.ones((len(q), len(v) + 1), bool)
    base.search_arrays(q, 5, 0.0, allowed=grown)
    assert fake.qmask_uploads == 3
    base.remove_embeddings([0])               # a removal forgets the uploaded masks
    shrunk = np.ones((len(q), len(v)), bool)
    base.search_arrays(q, 5, 0.0, allowed=shrunk)
    assert fake.qmask_uploads == 4
