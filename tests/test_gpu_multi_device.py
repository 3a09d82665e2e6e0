"""``VectorBase(settings, devices=[...])`` on the GPU: every lookup over W shard indexes, fanned out and merged inside
libtavec (``tav_multi_*``), equals bit for bit the same lookup on a one-device ``VectorBase`` over the same rows, and
``expected_topk`` on exact-arithmetic (dyadic) corpora.

Shards share one GPU here (``devices=[0] * W``), which exercises every step of the fan-out, the peer copies into the
merge slabs and the merges; the same cases run on distinct devices when the machine has more than one.
"""

from __future__ import annotations

import asyncio
import sqlite3

import numpy as np
import pytest

import typeagent_py_b200 as tab
from oracle import ref_loader
from oracle import vectorbase_oracle as O
from tests.exact import dyadic_corpus, expected_topk, preset
from tests.parity import assert_hits_match

pytestmark = pytest.mark.gpu

DTYPES = ["bfloat16", "float16", "float32"]


def _device_count() -> int:
    import torch

    return torch.cuda.device_count()


def _layouts():
    yield "shared-2", [0, 0]
    yield "shared-3", [0, 0, 0]
    yield "shared-8", [0] * 8


def _distinct():
    n = _device_count()
    if n < 2:
        pytest.skip("one CUDA device: distinct-device runs need two or more")
    return list(range(n))


def _pair(devices, dtype, rows, normalize=False):
    settings = tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel())
    multi = tab.VectorBase(settings, devices=devices, storage_dtype=dtype, normalize=normalize)
    one = tab.VectorBase(settings, storage_dtype=dtype, normalize=normalize)
    if len(rows):
        multi.add_embeddings(None, rows)
        one.add_embeddings(None, rows)
    return multi, one


def _same(got, want, what=""):
    assert len(got) == len(want), what
    for g, w in zip(got, want):
        g, w = np.asarray(g), np.asarray(w)
        assert g.dtype == w.dtype and g.shape == w.shape, what
        if g.dtype == np.float32:
            g, w = g.view(np.uint32), w.view(np.uint32)
        np.testing.assert_array_equal(g, w, err_msg=what)


def _both(multi, one, fn, what=""):
    got = fn(multi)
    _same(got, fn(one), what)
    return got


def _hits(lists):
    return [[(h.item, np.float32(h.score).view(np.uint32)) for h in hits] for hits in lists]


def _check_topk(multi, one, q, dots, ks=(10, 100, 3000), paths=(None, "scan", "mma"), floors=(0.0,)):
    for path in paths:
        multi.force_path = one.force_path = path
        for b in (1, 64, 256):
            for k in ks:
                if path == "mma" and (k > 2048 or b < 1):
                    continue
                for floor in floors:
                    what = f"path={path} B={b} k={k} floor={floor}"
                    got = _both(multi, one, lambda vb: vb.search_arrays(q[:b], k, floor), what)
                    k_eff = max(1, min(k, dots.shape[1]))
                    _same(got, expected_topk(dots[:b], k_eff, floor), what)
    multi.force_path = one.force_path = None


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name,devices", list(_layouts()), ids=[n for n, _ in _layouts()])
def test_topk_equals_one_device_and_exact(name, devices, dtype):
    amp, exp = preset("fine", 64)
    v, q, dots = dyadic_corpus(5000, 64, 256, amp, exp, seed=11)
    multi, one = _pair(devices, dtype, v)
    _check_topk(multi, one, q, dots)
    hits = _both(multi, one, lambda vb: _hits([vb.fuzzy_lookup_embedding(q[3], 7)]))
    assert hits


@pytest.mark.parametrize("dtype", DTYPES)
def test_min_score_edges(dtype):
    amp, exp = preset("coarse", 32)
    v, q, dots = dyadic_corpus(3000, 32, 64, amp, exp, seed=12)
    multi, one = _pair([0, 0, 0], dtype, v)
    s = np.sort(np.clip((dots[0] + 1) * 0.5, 0, 1))
    floors = (0.0, 1.0, float(s[len(s) // 2]), float(np.nextafter(s[-5], np.float32(2))), float("nan"), -1.0, 2.0)
    _check_topk(multi, one, q, dots, ks=(10, 100), paths=(None, "scan"), floors=floors)
    for floor in floors:
        _both(multi, one, lambda vb: vb.search_range(q[:16], floor), f"range floor={floor}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name,devices", list(_layouts()), ids=[n for n, _ in _layouts()])
def test_subset_with_repeats_and_negative_ordinals(name, devices, dtype):
    amp, exp = preset("coarse", 32)
    v, q, _ = dyadic_corpus(2000, 32, 64, amp, exp, seed=13, dup=[(1999, 5), (1000, 5)])
    multi, one = _pair(devices, dtype, v)
    rng = np.random.default_rng(3)
    sub = rng.integers(-2000, 2000, size=700)
    sub[:6] = [5, 1999, 1000, 5, -1, -2000]
    for ties in (False, True):
        for k in (1, 10, 700):
            _both(multi, one, lambda vb: vb.search_arrays(q, k, 0.3, subset=sub, ties_low_first=ties), f"k={k}")
        _both(multi, one, lambda vb: vb.search_range(q, 0.4, subset=sub, ties_low_first=ties), "range subset")
    _both(multi, one, lambda vb: _hits([vb.fuzzy_lookup_embedding_in_subset(q[0], sub.tolist(), 20)]))
    _both(multi, one, lambda vb: _hits([vb.fuzzy_lookup_embedding_in_subset(q[1], sub.tolist(), 0)]))
    before = multi.search_arrays(q, 10)
    with pytest.raises(IndexError, match="out of bounds"):
        multi.search_arrays(q, 10, subset=[0, 2000])
    with pytest.raises(IndexError, match="out of bounds"):
        multi.search_range(q, 0.5, subset=[-2001])
    _same(multi.search_arrays(q, 10), before)
    assert len(multi) == 2000


@pytest.mark.parametrize("dtype", DTYPES)
def test_row_mask_and_predicate_in_reference_order(dtype):
    amp, exp = preset("coarse", 32)
    dup = [(r, 7) for r in range(100, 3000, 97)]   # tie-heavy: one row repeated in every block
    v, q, dots = dyadic_corpus(3000, 32, 32, amp, exp, seed=14, dup=dup)
    multi, one = _pair([0, 0, 0], dtype, v)
    allowed = (np.arange(3000) % 5) != 2
    for path in (None, "scan", "mma"):
        multi.force_path = one.force_path = path
        got = _both(multi, one, lambda vb: vb.search_arrays(q, 50, 0.2, allowed=allowed), f"mask {path}")
        _same(got, expected_topk(dots, 50, 0.2, allowed=allowed))
    multi.force_path = one.force_path = None
    _both(multi, one, lambda vb: vb.search_arrays(q, 50, allowed=allowed, ties_low_first=True))
    _both(multi, one, lambda vb: vb.search_range(q, 0.5, allowed=allowed))

    def pred(i):
        return i % 3 != 1

    for k in (5, 300):
        _both(multi, one, lambda vb: _hits([vb.fuzzy_lookup_embedding(q[b], k, 0.1, predicate=pred) for b in range(4)]),
              f"predicate k={k}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name,devices", list(_layouts()), ids=[n for n, _ in _layouts()])
def test_threshold_search_and_every_hit(name, devices, dtype):
    amp, exp = preset("fine", 64)
    v, q, dots = dyadic_corpus(6000, 64, 64, amp, exp, seed=15)
    multi, one = _pair(devices, dtype, v)
    for path in (None, "scan", "mma"):
        multi.force_path = one.force_path = path
        for floor in (0.55, 0.7, 0.0):
            offsets, items, scores = _both(multi, one, lambda vb: vb.search_range(q, floor), f"{path} {floor}")
            blocks = np.searchsorted(multi._multi.starts[1:], items, side="right")
            if floor == 0.55:
                assert len(set(blocks.tolist())) == len(devices)   # hits in every block
    multi.force_path = one.force_path = None
    _both(multi, one, lambda vb: _hits(vb.fuzzy_lookup_embeddings(q[:8], max_hits=0, min_score=0.6)), "max_hits=0")
    _both(multi, one, lambda vb: _hits([vb.fuzzy_lookup_embedding(q[0], max_hits=0, min_score=0.6)]))


def test_fewer_rows_than_shards():
    amp, exp = preset("fine", 16)
    v, q, dots = dyadic_corpus(3, 16, 8, amp, exp, seed=16)
    for dtype in DTYPES:
        multi, one = _pair([0] * 8, dtype, v)
        _same(_both(multi, one, lambda vb: vb.search_arrays(q, 5)), expected_topk(dots, 3, 0.0))
        _both(multi, one, lambda vb: vb.search_range(q, 0.0))
        _both(multi, one, lambda vb: vb.search_arrays(q, 2, subset=[2, -3, 2]))
        _both(multi, one, lambda vb: vb.search_arrays(q, 3, allowed=np.array([True, False, True])))
        assert multi._multi.starts == [0, 1, 2, 3, 3, 3, 3, 3, 3]


def _all_lookups(multi, one, q, what):
    n = len(one)
    _both(multi, one, lambda vb: vb.search_arrays(q, 20, 0.3), what)
    _both(multi, one, lambda vb: vb.search_range(q, 0.6), what)
    if n:
        _both(multi, one, lambda vb: vb.search_arrays(q, 10, subset=[n - 1, 0, -1, n // 2]), what)
        allowed = np.arange(n) % 4 != 0
        _both(multi, one, lambda vb: vb.search_arrays(q, 10, allowed=allowed), what)
    assert np.array_equal(multi.serialize(), one.serialize())


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name,devices", list(_layouts()), ids=[n for n, _ in _layouts()])
def test_row_changes(name, devices, dtype):
    amp, exp = preset("fine", 32)
    v, q, _ = dyadic_corpus(9000, 32, 32, amp, exp, seed=17)
    multi, one = _pair(devices, dtype, v[:600])
    _all_lookups(multi, one, q, "start")
    for vb in (multi, one):
        vb.add_embeddings(None, v[600:700])
    _all_lookups(multi, one, q, "append")
    for vb in (multi, one):
        vb.add_embeddings(None, v[700:9000])
    _all_lookups(multi, one, q, "append with a re-split")
    _both(multi, one, lambda vb: vb.search_arrays(q[:2], 8500, 0.2), "k beyond the merge")
    assert multi._multi.starts[-1] == 9000 and max(np.diff(multi._multi.starts)) * len(devices) <= 2 * 9000
    lo, hi = multi._multi.starts[1], multi._multi.starts[2]
    for vb in (multi, one):
        vb.remove_embeddings(list(range(lo, hi)) + [0, -1])     # empties block 1
    assert multi._multi.starts[2] == multi._multi.starts[1]
    _all_lookups(multi, one, q, "removal")
    first = max(0, min(multi._multi.starts[1] - 3, len(one) - 40))
    for vb in (multi, one):
        vb.set_embeddings_at(first, v[:40])                     # across the boundary of blocks 0, 1 (empty) and 2
    _all_lookups(multi, one, q, "overwrite")
    for vb in (multi, one):
        vb.clear()
    _all_lookups(multi, one, q, "clear")
    for vb in (multi, one):
        vb.deserialize(v[:1234])
    _all_lookups(multi, one, q, "deserialize")
    for vb in (multi, one):
        vb.add_embeddings(None, v[1234:1300])
        vb.remove_embeddings([5, 600])
        vb.set_embeddings_at(1, v[2000:2010])
    _all_lookups(multi, one, q, "mixed")


def test_exact_redo_of_a_float32_row_beyond_fp16():
    amp, exp = preset("fine", 64)
    v, q, dots = dyadic_corpus(8192, 64, 64, amp, exp, seed=18)
    # one row beyond the fp16 range, in block 1 of 3: that shard's tensor-core search is redone exactly.  A single
    # non-zero element keeps its dots exact in any order.
    v[5000] = 0
    v[5000, 3] = np.float32(2.0 ** 17)
    dots[:, 5000] = q[:, 3] * np.float32(2.0 ** 17)
    multi, one = _pair([0, 0, 0], "float32", v)
    for path in (None, "scan", "mma"):
        multi.force_path = one.force_path = path
        got = _both(multi, one, lambda vb: vb.search_arrays(q, 30, 0.0), f"redo {path}")
        _same(got, expected_topk(dots, 30, 0.0), f"redo {path}")
        _both(multi, one, lambda vb: vb.search_range(q, 0.75), f"range redo {path}")
        multi.force_path = None
        _same(multi.search_arrays(q, 30, 0.0), got, f"multi {path} / default")


def test_random_data_parity_and_normalize():
    v, q = O.make_corpus(12000, 128, seed=19, n_queries=32)
    multi, one = _pair([0, 0, 0], "float32", v)
    items, scores, counts = multi.search_arrays(q, 25, 0.2)
    for b in range(len(q)):
        got = [O.Hit(int(i), float(s)) for i, s in zip(items[b, :counts[b]], scores[b, :counts[b]])]
        assert_hits_match(got, O.lookup(v, q[b], 25, 0.2), min_score=0.2, what=f"query {b}")
    multi.force_path = one.force_path = "scan"
    _both(multi, one, lambda vb: vb.search_arrays(q, 25, 0.2))
    rng = np.random.default_rng(20)
    raw = rng.standard_normal((5000, 96)).astype(np.float32) * np.float32(3.0)
    for dtype in DTYPES:
        multi, one = _pair([0, 0, 0], dtype, raw, normalize=True)
        for path in ("scan", "scan2"):
            multi.force_path = one.force_path = path
            _both(multi, one, lambda vb: vb.search_arrays(raw[:40], 15), f"normalize {dtype} {path}")
            _both(multi, one, lambda vb: vb.search_range(raw[:40], 0.8), f"normalize range {dtype} {path}")


def test_distinct_devices():
    devices = _distinct()
    amp, exp = preset("fine", 64)
    v, q, dots = dyadic_corpus(5000, 64, 256, amp, exp, seed=21)
    for dtype in DTYPES:
        multi, one = _pair(devices, dtype, v)
        _check_topk(multi, one, q, dots, ks=(10, 3000))
        _both(multi, one, lambda vb: vb.search_range(q, 0.6))
        _both(multi, one, lambda vb: vb.search_arrays(q, 10, subset=[-1, 4, 4999, 4]))
        _all_lookups(multi, one, q, "distinct")
        for vb in (multi, one):
            vb.remove_embeddings(list(range(100, 2600)))
        _all_lookups(multi, one, q, "distinct after removal")


@pytest.mark.skipif(not ref_loader.reference_available(), reason="reference sources neither mounted nor vendored")
def test_install_with_devices_on_reference_built_indexes():
    from tests.golden import cases as GC
    from tests.test_install_real import DictEmbeddingModel, _assert_terms_match, _terms, load_all

    mods = load_all()
    rel_mem = mods["typeagent.storage.memory.reltermsindex"]
    rel_sql = mods["typeagent.storage.sqlite.reltermsindex"]
    schema = ref_loader.load_reference_module("typeagent.storage.sqlite.schema")
    vb = mods["typeagent.aitools.vectorbase"]
    ep, epq = GC.episode53()
    vectors = ep[:100]
    texts = [f"term{i:05d}" for i in range(len(vectors))]
    q_texts = [f"query{i}" for i in range(len(epq))]
    table = {**dict(zip(texts, vectors)), **dict(zip(q_texts, epq))}

    def run(min_score, max_hits):
        settings = vb.TextEmbeddingIndexSettings(embedding_model=DictEmbeddingModel(table), min_score=min_score,
                                                 max_matches=max_hits)
        mem = rel_mem.TermEmbeddingIndex(settings)
        db = sqlite3.connect(":memory:")
        db.execute(schema.RELATED_TERMS_FUZZY_SCHEMA)
        sql = rel_sql.SqliteRelatedTermsFuzzy(db, settings)

        async def go():
            await mem.add_terms(texts)
            await sql.add_terms(texts)
            return (_terms(await mem.lookup_terms(q_texts)), _terms(await sql.lookup_terms(q_texts)),
                    _terms([await mem.lookup_term(q_texts[1])]))

        return asyncio.run(go()), mem

    for min_score, max_hits in ((0.85, 50), (0.0, 10)):
        want, _ = run(min_score, max_hits)                       # the reference on numpy
        try:
            tab.install()
            one, _ = run(min_score, max_hits)
        finally:
            tab.uninstall()
        try:
            tab.install(devices=[0, 0])
            got, mem = run(min_score, max_hits)
            assert mem._vectorbase._multi is not None and mem._vectorbase._multi.world == 2
        finally:
            tab.uninstall()
        assert got == one
        for g, w in zip(got, want):
            _assert_terms_match(g, w)


def test_merges_of_alternating_k_keep_their_shared_memory():
    """``tav_merge_topk`` and ``tav_merge_topk_ordered`` order 0 launch the same merge kernel.  A small-k merge of one
    must not lower the kernel's shared-memory grant under a large-k merge of the other (the multi-device search
    merges with order 0 at any k up to 8192)."""
    import ctypes as C

    import torch

    from typeagent_py_b200 import _capi

    lib = _capi.load()

    def merge(ordered, k):
        items = torch.zeros((2, 1, k), dtype=torch.int64, device="cuda")
        scores = torch.zeros((2, 1, k), dtype=torch.float32, device="cuda")
        counts = torch.zeros((2, 1), dtype=torch.int32, device="cuda")
        out = (torch.empty((1, k), dtype=torch.int64, device="cuda"),
               torch.empty((1, k), dtype=torch.float32, device="cuda"),
               torch.empty((1,), dtype=torch.int32, device="cuda"))
        args = [0, 2, 1, k, C.c_void_p(items.data_ptr()), C.c_void_p(scores.data_ptr()), C.c_void_p(counts.data_ptr()),
                0, 0, 0]
        outs = [C.c_void_p(t.data_ptr()) for t in out]
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        if ordered:
            _capi.check(lib.tav_merge_topk_ordered(*args, 0, *outs, stream))
        else:
            _capi.check(lib.tav_merge_topk(*args, *outs, stream))
        torch.cuda.synchronize()
        assert int(out[2][0]) == 0

    for ordered_first in (True, False):
        merge(ordered_first, 8192)
        merge(not ordered_first, 4000)
        merge(ordered_first, 8192)
        merge(not ordered_first, 10)
        merge(ordered_first, 8192)
