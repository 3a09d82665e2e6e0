"""Threshold search into caller device tensors (``search_range_device`` / ``tav_range_search_into``) bit for bit:
offsets, items and score bits, no tolerances.  The result is the one ``search_range`` gives, sized on the device:
synchronous, and deferred (no host synchronisation, flagged queries completed by ``finish_search``).  Dyadic
corpora (tests/exact.py) make every path's float32 dots exact, so every case is compared with the exact
expectation of tests/test_gpu_range.py; random rows are compared with ``search_range`` on the same index."""

from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import typeagent_py_b200 as tab
from oracle import vectorbase_oracle as O
from tests.exact import dyadic_corpus, preset
from tests.test_gpu_exact import min_score_for, row_mask
from tests.test_gpu_mma import make_base
from tests.test_gpu_query_masks import expected_range_masked
from tests.test_gpu_range import assert_same_range, expected_range
from typeagent_py_b200 import _capi

pytestmark = pytest.mark.gpu

OFFSET = (1 << 32) + 5
SENTINEL_ITEM = -7
SENTINEL_BITS = 0x7FC0BEEF  # a NaN pattern no score has


def cuda(x):
    import torch

    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()


def filled(b, cap):
    """out tensors for B queries and `cap` hits, every slot holding the sentinel"""
    import torch

    return (torch.full((b + 1,), -1, dtype=torch.int64, device="cuda"),
            torch.full((cap,), SENTINEL_ITEM, dtype=torch.int64, device="cuda"),
            torch.full((cap,), SENTINEL_BITS, dtype=torch.int32, device="cuda").view(torch.float32))


def run(base, q, ms, cap, defer, **kw):
    """-> ((offsets, items, scores) numpy, queries redone).  The synchronous form must leave nothing to finish."""
    import torch

    out = filled(len(q), cap)
    got = base.search_range_device(cuda(q), ms, cap, out=out, defer_check=defer, **kw)
    assert all(g is o for g, o in zip(got, out))
    if defer:
        redone = base.finish_search()
    else:
        assert not base._pending
        lib, ix = base._ensure_device()
        n = C.c_int(-1)
        _capi.check(lib.tav_finish_search(ix, None, C.byref(n)))
        redone = n.value
        assert redone == 0, "a synchronous search left queries to finish"
    torch.cuda.synchronize()
    return tuple(t.cpu().numpy() for t in got), redone


def assert_prefix(got, want, cap, what):
    """offsets complete, the first `cap` hits equal to the full result, every slot past the result untouched"""
    go, gi, gs = got
    wo, wi, ws = want
    np.testing.assert_array_equal(go, wo, err_msg=f"{what}: offsets")
    n = min(cap, len(wi))
    assert_same_range((np.array([0, n]), gi[:n], gs[:n]), (np.array([0, n]), wi[:n], ws[:n]), what)
    assert (gi[n:] == SENTINEL_ITEM).all(), f"{what}: items written past the result or the capacity"
    assert (gs[n:].view(np.uint32) == SENTINEL_BITS).all(), f"{what}: scores written past the result or the capacity"


# ---------------------------------------------------------------- 1. dyadic corpora, every scorer and filter
P = pytest.param
SCORERS = [  # (storage, force_path, queries)
    P("float32", "scan", 5, id="scan-f32"),
    P("bfloat16", "scan", 5, id="scan-bf16"),
    P("float16", "scan", 5, id="scan-fp16"),
    P("bfloat16", "mma", 18, id="mma-bf16"),
    P("float16", "mma", 18, id="mma-fp16"),
    P("float32", "mma", 18, id="mma_split-f32"),
]
FILTERS = ["none", "row_mask", "query_masks", "ties_low", "subset", "item_offset"]


@pytest.mark.parametrize("flt", FILTERS)
@pytest.mark.parametrize("storage,path,b", SCORERS)
def test_dyadic_every_scorer_and_filter(storage, path, b, flt):
    n, d = 6000, 64
    amp, exp = preset("fine", d)
    v, q, dots = dyadic_corpus(n, d, b, amp, exp, seed=n + b + FILTERS.index(flt))
    base = make_base(v, storage, path)
    rng = np.random.default_rng(b)
    kw, want_of = {}, None
    if flt == "row_mask":
        kw["allowed"] = row_mask("half", n, seed=3)
        want_of = lambda ms: expected_range(dots, ms, kw["allowed"])  # noqa: E731
    elif flt == "query_masks":
        kw["allowed"] = rng.random((b, n)) < 0.5
        want_of = lambda ms: expected_range_masked(dots, ms, kw["allowed"])  # noqa: E731
    elif flt == "ties_low":
        kw["ties_low_first"] = True
        want_of = lambda ms: expected_range(dots, ms, ties_low=True)  # noqa: E731
    elif flt == "subset":
        sub = rng.choice(n, 2500, replace=False)
        sub[:2] = [n - 1, n - 1]  # a repeated ordinal is scored twice
        kw["subset"] = sub
        base.force_path = "scan"  # a subset takes the row scan
        want_of = lambda ms: expected_range(dots[:, sub], ms, positions=sub)  # noqa: E731
    elif flt == "item_offset":
        kw["item_offset"] = OFFSET
        want_of = lambda ms: expected_range(dots, ms, item_offset=OFFSET)  # noqa: E731
    else:
        want_of = lambda ms: expected_range(dots, ms)  # noqa: E731
    for ms_kind in ("hit", "hit+ulp", "hit-ulp"):
        ms = min_score_for(ms_kind, dots, n // 8)
        want = want_of(ms)
        for defer in (False, True):
            got, redone = run(base, q, ms, int(want[0][-1]), defer, **kw)
            assert_same_range(got, want, f"{storage} {path} {flt} {ms_kind} defer={defer}")
            assert redone == 0  # the default regions hold these hits
        t = base.last_timing()
        assert t["path"] == ("scan" if base.force_path == "scan" else "mma_split" if storage == "float32" else "mma"), t


# ---------------------------------------------------------------- 2. capacity
@pytest.mark.parametrize("storage,path,b,ms", [
    P("bfloat16", "scan", 3, "hit", id="scan-small_segments"),
    P("float32", "scan", 3, "-2", id="scan-radix"),
    P("float16", "mma", 17, "hit", id="mma-small_segments"),
    P("bfloat16", "mma", 16, "-2", id="mma-radix"),
])
def test_capacity_prefix_and_untouched_slots(storage, path, b, ms):
    n, d = 6000, 64
    amp, exp = preset("coarse" if ms == "-2" else "fine", d)
    v, q, dots = dyadic_corpus(n, d, b, amp, exp, seed=b + 40)
    ms = min_score_for(ms, dots, n // 8)
    want = expected_range(dots, ms)
    total = int(want[0][-1])
    cut = int(want[0][1]) + (int(want[0][2]) - int(want[0][1])) // 2  # inside query 1's hits
    base = make_base(v, storage, path)
    for cap in (0, total - 1, total, total + 1, cut):
        for defer in (False, True):
            got, _ = run(base, q, ms, cap, defer, expected_hits=total)
            assert_prefix(got, want, cap, f"cap {cap} of {total} defer={defer}")


# ---------------------------------------------------------------- 3. overflowed regions
@pytest.mark.parametrize("storage,path", [("bfloat16", "scan"), ("float32", "scan"), ("bfloat16", "mma"),
                                          ("float32", "mma")])
def test_overflow_completed_by_finish(storage, path):
    amp, exp = preset("coarse", 64)
    b = 3 if path == "scan" else 20
    v, q, dots = dyadic_corpus(7000, 64, b, amp, exp, seed=77)
    want = expected_range(dots, -2.0)
    total = int(want[0][-1])
    base = make_base(v, storage, path)
    for cap in (total, total // 2):
        # expected_hits = 1: regions (or segments) of a few dozen keys for thousands of hits per query
        got, redone = run(base, q, -2.0, cap, True, expected_hits=1)
        assert_prefix(got, want, cap, f"deferred cap {cap}")
        if path == "scan":
            assert redone == b
        else:
            assert 0 < redone <= b
        got, _ = run(base, q, -2.0, cap, False, expected_hits=1)
        assert_prefix(got, want, cap, f"synchronous cap {cap}")


# ---------------------------------------------------------------- 4. the split form's fp16-range fallback
def test_split_form_beyond_fp16_range_redone_by_the_row_scan():
    amp, exp = preset("fine", 64)
    v, q, _ = dyadic_corpus(5000, 64, 16, amp, exp, seed=65)
    v = v.copy()
    v[5] = 70000.0  # beyond the fp16 range: the two-plane form cannot carry this row
    dots = (q.astype(np.float64) @ v.astype(np.float64).T).astype(np.float32)
    want = expected_range(dots, 0.0)
    base = make_base(v, "float32", "mma")
    cap = int(want[0][-1]) + 500  # the abandoned tensor-core pass must not write these slots either
    got, redone = run(base, q, 0.0, cap, True)
    assert redone == 16
    assert_prefix(got, want, cap, "split overflow, deferred")
    assert_same_range(base.search_range(q, 0.0), want, "search_range")
    got, _ = run(base, q, 0.0, cap, False)
    assert_prefix(got, want, cap, "split overflow, synchronous")


# ---------------------------------------------------------------- 5. no host synchronisation
@pytest.fixture(scope="module")
def hold_cycles():
    import torch

    torch.cuda._sleep(1000)  # loads the kernel
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    cycles = 20_000_000
    start.record()
    torch.cuda._sleep(cycles)
    end.record()
    end.synchronize()
    return int(cycles * 200 / start.elapsed_time(end))


@pytest.mark.parametrize("storage,path,b", [("bfloat16", "mma", 16), ("float32", "mma", 16), ("float16", "scan", 4),
                                            ("float32", "scan", 1)])
def test_deferred_call_does_not_synchronise(storage, path, b, hold_cycles):
    import torch

    amp, exp = preset("fine", 64)
    v, q, dots = dyadic_corpus(6000, 64, b, amp, exp, seed=b + 7)
    want = expected_range(dots, 0.4)
    cap = int(want[0][-1]) + 100
    base = make_base(v, storage, path)
    qd = cuda(q)
    out = filled(b, cap)
    base.search_range_device(qd, 0.4, cap, out=out, defer_check=True)  # warm-up: buffers of this shape
    base.finish_search()
    stream = torch.cuda.current_stream()
    torch.cuda._sleep(hold_cycles)
    got = base.search_range_device(qd, 0.4, cap, out=out, defer_check=True)
    assert not stream.query(), "the deferred call waited for the stream"
    assert base.finish_search() == 0
    torch.cuda.synchronize()
    assert_prefix(tuple(t.cpu().numpy() for t in got), want, cap, "after the hold")


# ---------------------------------------------------------------- 6. interleaving
def test_deferred_range_and_topk_finished_together_across_a_mask_upload_and_streams():
    import torch

    amp, exp = preset("fine", 64)
    v, q, dots = dyadic_corpus(6000, 64, 16, amp, exp, seed=606)
    base = make_base(v, "bfloat16", "mma")
    qd = cuda(q)
    want = expected_range(dots, 0.45)
    cap = int(want[0][-1])
    r1 = base.search_range_device(qd, 0.45, cap, defer_check=True, expected_hits=1)  # overflows: flagged
    t1 = base.search_device(qd, 50, 0.0, defer_check=True)
    mask = row_mask("half", 6000, seed=1)
    r2 = base.search_range_device(qd, 0.45, cap, defer_check=True, allowed=mask)  # uploads the mask first
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        r3 = base.search_range_device(qd, 0.45, cap, defer_check=True, expected_hits=1)
        t2 = base.search_device(qd, 50, 0.0, defer_check=True)
        base.finish_search()
    torch.cuda.synchronize()
    def np3(r):  # the hits the offsets count (the masked search fills less than its room)
        o, i, s = (x.cpu().numpy() for x in r)
        return o, i[:o[-1]], s[:o[-1]]

    assert_same_range(np3(r1), want, "first deferred range (finished by the mask upload)")
    assert_same_range(np3(r2), expected_range(dots, 0.45, mask), "masked deferred range")
    assert_same_range(np3(r3), want, "deferred range on the side stream")
    from tests.exact import expected_topk

    for t in (t1, t2):
        wi, ws, wc = expected_topk(dots, 50, 0.0)
        np.testing.assert_array_equal(t[2].cpu().numpy(), wc)
        np.testing.assert_array_equal(t[0].cpu().numpy(), wi)
        np.testing.assert_array_equal(t[1].cpu().numpy().view(np.uint32), ws.view(np.uint32))


def test_more_deferred_searches_than_the_cap():
    import torch

    amp, exp = preset("fine", 64)
    v, q, dots = dyadic_corpus(6000, 64, 2, amp, exp, seed=64)
    want = expected_range(dots, 0.45)
    cap = int(want[0][-1])
    base = make_base(v, "float16", "scan")
    qd = cuda(q)
    outs = [base.search_range_device(qd, 0.45, cap, defer_check=True, expected_hits=1) for _ in range(70)]
    redone = base.finish_search()
    assert 0 < redone <= 70 * 2  # the 65th call finished the first 64 itself
    torch.cuda.synchronize()
    for i, r in enumerate(outs):
        assert_same_range(tuple(x.cpu().numpy() for x in r), want, f"search {i}")


def test_fetch_after_it_is_a_state_error():
    amp, exp = preset("fine", 32)
    v, q, dots = dyadic_corpus(3000, 32, 2, amp, exp, seed=12)
    base = make_base(v, "float32", "scan")
    lib, ix = base._ensure_device()
    base.search_range(q, 0.5)
    base.search_range_device(cuda(q), 0.5, 10)
    items, scores = np.empty(1, np.int64), np.empty(1, np.float32)
    rc = lib.tav_range_fetch(ix, 0, 1, items.ctypes.data_as(C.c_void_p), scores.ctypes.data_as(C.c_void_p), 0, None)
    assert rc == _capi.TAV_ERR_STATE
    assert_same_range(base.search_range(q, 0.5), expected_range(dots, 0.5), "search_range after")


@pytest.mark.parametrize("trigger", ["finish", "mask_upload", "sync_topk"])
def test_redo_leaves_the_last_range_search_fetchable(trigger):
    """A deferred search whose regions overflowed, then tav_range_search, then a call that finishes the deferred
    search: the fetch still returns tav_range_search's hits (the redo sorts into the caller's tensors only)."""
    import torch

    amp, exp = preset("fine", 64)
    v, q, dots = dyadic_corpus(6000, 64, 16, amp, exp, seed=99)
    want_dev, want_host = expected_range(dots, 0.45), expected_range(dots[:3], 0.6)
    for path in ("scan", "mma"):
        base = make_base(v, "bfloat16", path)
        lib, ix = base._ensure_device()
        got = base.search_range_device(cuda(q), 0.45, int(want_dev[0][-1]), defer_check=True, expected_hits=1)
        qh = np.ascontiguousarray(q[:3])
        offsets = np.zeros(4, np.int64)
        _capi.check(lib.tav_range_search(ix, qh.ctypes.data_as(C.c_void_p), 3, C.c_float(0.6), 0, None, 0, 0, 0,
                                         offsets.ctypes.data_as(C.c_void_p), None))
        if trigger == "finish":
            assert base.finish_search() > 0
        elif trigger == "mask_upload":
            base._use_row_mask(lib, ix, np.ones(6000, bool))
        else:
            base.force_path = "mma"
            base.search_arrays(q, 10, 0.0)  # a synchronous tensor-core top-k finishes what is outstanding
        n = int(offsets[-1])
        items, scores = np.empty(n, np.int64), np.empty(n, np.float32)
        _capi.check(lib.tav_range_fetch(ix, 0, n, items.ctypes.data_as(C.c_void_p), scores.ctypes.data_as(C.c_void_p),
                                        0, None))
        assert_same_range((offsets, items, scores), want_host, f"{path} {trigger}: fetch after the redo")
        base.finish_search()
        torch.cuda.synchronize()
        assert_same_range(tuple(x.cpu().numpy() for x in got), want_dev, f"{path} {trigger}: the deferred search")


# ---------------------------------------------------------------- 7. random rows
@pytest.mark.parametrize("storage", ["float32", "bfloat16"])
def test_random_rows_1m_equal_search_range(storage):
    import torch

    gen = torch.Generator(device="cuda").manual_seed(7)
    t = torch.randn((1_000_000, 768), generator=gen, device="cuda")
    t = torch.nn.functional.normalize(t, dim=1).to(getattr(torch, storage)).contiguous()
    qd = torch.nn.functional.normalize(torch.randn((64, 768), generator=gen, device="cuda"), dim=1).contiguous()
    base = tab.VectorBase.from_device_tensor(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()), t)
    want = base.search_range(qd.cpu().numpy(), 0.55)
    assert want[0][-1] > 64 * 1000
    for defer in (False, True):
        got = base.search_range_device(qd, 0.55, int(want[0][-1]), defer_check=defer)
        base.finish_search()
        assert_same_range(tuple(x.cpu().numpy() for x in got), want, f"1M {storage} defer={defer}")
        # tiny regions: every query's segments overflow and the tensor-core re-pass completes them, one pass for
        # all of them; its keys are the tensor cores' own, so the result is search_range's
        got = base.search_range_device(qd, 0.55, int(want[0][-1]), defer_check=defer, expected_hits=64)
        redone = base.finish_search()
        assert 0 < redone <= 64 if defer else redone == 0
        assert_same_range(tuple(x.cpu().numpy() for x in got), want, f"1M {storage} overflow defer={defer}")
        assert base.last_timing()["path"] == ("mma_split" if storage == "float32" else "mma")
    del base, t
    torch.cuda.empty_cache()


# ---------------------------------------------------------------- 8. edge cases
def test_edges_give_zero_offsets_and_write_nothing():
    amp, exp = preset("fine", 64)
    v, q, dots = dyadic_corpus(3000, 64, 3, amp, exp, seed=8)
    v = v.copy()
    v[7] = np.nan
    for storage, path in (("float32", "scan"), ("bfloat16", "mma")):
        base = make_base(v, storage, path)
        d = dots.copy()
        d[:, 7] = np.nan
        for defer in (False, True):
            assert_prefix(run(base, q, 0.0, 3000 * 3, defer)[0], expected_range(d, 0.0), 3000 * 3, f"NaN row {storage}")
            for qq, ms, kw in ((q[:0], 0.0, {}), (q, float("nan"), {}), (q, 0.0, {"subset": []})):
                got, _ = run(base, qq, ms, 16, defer, **kw)
                assert_prefix(got, (np.zeros(len(qq) + 1, np.int64), np.empty(0, np.int64), np.empty(0, np.float32)),
                              16, f"edge {storage} b={len(qq)} ms={ms} {kw}")
    empty = tab.VectorBase(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()))
    empty.add_embeddings(None, np.zeros((0, 64), np.float32))
    got, _ = run(empty, q, 0.0, 4, True)
    assert_prefix(got, (np.zeros(4, np.int64), np.empty(0, np.int64), np.empty(0, np.float32)), 4, "empty corpus")


# ---------------------------------------------------------------- 9. at scale
def test_10m_bf16_deferred_overflow_every_hit():
    """10M x 768 bf16, B = 16, ~30k hits per query: the default regions overflow; deferred, then finished."""
    import torch

    from tests import exact_torch as T
    from tests import test_gpu_scale_exact as S

    try:
        c = S.corpus("10M")
        q = c.q[:16].contiguous()
        _, s, _ = S.np3(T.topk_ref(c.dots(q), 30_000, 0.0))
        ms = float(np.median(s[:, -1]))
        want = S.np3(T.range_ref(c.dots(q), ms))
        assert np.median(np.diff(want[0])) > 16_384
        total = int(want[0][-1])
        for path in ("mma", "scan"):
            c.base.force_path = path
            out = filled(16, total)
            c.base.search_range_device(q, ms, total, out=out, defer_check=True, expected_hits=0)
            redone = c.base.finish_search()
            assert redone > 0
            torch.cuda.synchronize()
            assert_same_range(S.np3(out), want, f"10M deferred {path}")
    finally:
        S._CORPORA.clear()
        torch.cuda.empty_cache()
