"""Threshold search (``search_range`` / ``tav_range_search``, and ``max_hits=0`` lookups routed to it) bit for
bit, every query, no tolerances: on dyadic corpora (tests/exact.py) every row's float32 dot is exact, so the
expected result is the float32 score map, the ``>=`` compare and the library's order (score descending,
then row descending, or row ascending with ties-low), written below.  Ids name the branch they cover:
small segments (<= 4096 hits: one CTA, bitonic) or radix (larger: multi-CTA LSD radix sort), overflow
re-pass (a capacity hint below the hits), routing of ``tav_search`` with k >= rows > 8192."""

from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from oracle import vectorbase_oracle as O
from tests.exact import dyadic_corpus, preset, scores_of
from tests.golden import cases as GC
from tests.parity import assert_hits_match
from tests.test_gpu_exact import min_score_for, row_mask
from tests.test_gpu_mma import make_base
from typeagent_py_b200 import _capi

pytestmark = pytest.mark.gpu


def expected_range(dots, min_score, allowed=None, ties_low=False, positions=None, item_offset=0):
    """offsets int64 [B + 1], items int64 [T], scores float32 [T] from float32 dots [B, N]; ``positions``:
    the item of each column (subset ordinals), default the column itself."""
    dots = np.atleast_2d(np.asarray(dots, np.float32))
    floor = np.float32(min_score)
    offsets, items, scores = [0], [], []
    for row in dots:
        s = scores_of(row)
        with np.errstate(invalid="ignore"):
            ok = s >= floor  # False for NaN scores and a NaN floor
        if allowed is not None:
            ok &= np.asarray(allowed, bool)
        pos = np.flatnonzero(ok)
        order = pos[np.lexsort((pos if ties_low else -pos, -s[pos].view(np.uint32).astype(np.int64)))]
        items.append(order if positions is None else np.asarray(positions, np.int64)[order])
        scores.append(s[order])
        offsets.append(offsets[-1] + len(order))
    return (np.array(offsets, np.int64), np.concatenate(items).astype(np.int64) + item_offset,
            np.concatenate(scores).astype(np.float32))


def assert_same_range(got, want, what):
    go, gi, gs = got
    wo, wi, ws = want
    np.testing.assert_array_equal(go, wo, err_msg=f"{what}: offsets")
    bad = np.flatnonzero((gi != wi) | (gs.view(np.uint32) != ws.view(np.uint32)))
    if len(bad):
        j = bad[0]
        q = np.searchsorted(wo, j, side="right") - 1
        raise AssertionError(f"{what}: {len(bad)} of {len(wi)} hits differ, first in q{q} at rank {j - wo[q]}: "
                             f"({gi[j]}, {gs[j]!r}) vs ({wi[j]}, {ws[j]!r})")


def main_kernels(base):
    return sum(1 for name, _ in base.last_timing()["kernels"] if name == "main")


P = pytest.param
# (storage, n, d, b, preset, mask, ties_low, min_score kind)
DYADIC = [
    P("float32", 6000, 64, 3, "fine", None, False, "0", id="f32-small_segments-min0"),
    P("bfloat16", 6000, 64, 3, "fine", None, False, "-2", id="bf16-radix-everything"),
    P("float16", 6000, 72, 2, "coarse", None, False, "-2", id="fp16-radix-everything-coarse_ties"),
    P("float32", 6000, 64, 5, "coarse", None, True, "0", id="f32-ties_low-coarse"),
    P("bfloat16", 6000, 64, 2, "fine", None, True, "-2", id="bf16-radix-ties_low"),
    P("float16", 9000, 56, 9, "fine", "half", False, "0", id="fp16-mask_half-B9_two_blocks"),
    P("bfloat16", 6000, 64, 3, "fine", "bit0", False, "-2", id="bf16-mask_bit0"),
    P("float32", 6000, 136, 3, "coarse", "bit31", True, "0", id="f32-mask_bit31-ties_low-coarse"),
    P("bfloat16", 6000, 64, 2, "fine", None, False, "hit", id="bf16-min_at_a_hit"),
    P("float16", 6000, 64, 2, "fine", None, False, "hit+ulp", id="fp16-min_ulp_above_a_hit"),
    P("float32", 6000, 64, 2, "fine", None, False, "hit-ulp", id="f32-min_ulp_below_a_hit"),
    P("bfloat16", 6000, 64, 3, "coarse", None, False, "1", id="bf16-min1-clipped_ties"),
    P("float32", 6000, 64, 3, "fine", None, False, "1.5", id="f32-min_above_1-empty"),
    P("float16", 3000, 8, 3, "fine", None, False, "nan", id="fp16-min_nan-empty"),
    P("float32", 100, 18, 4, "fine", None, False, "0", id="f32-N100-unaligned_rows"),
]
# the tensor-core collection: bf16 / fp16 on the MAIN kernel, float32 through its fp16 planes (mma_split)
DYADIC_MMA = [
    P("bfloat16", 6000, 64, 20, "fine", None, False, "0", id="mma-bf16-min0"),
    P("float16", 6000, 72, 17, "coarse", None, False, "-2", id="mma-fp16-radix-everything-coarse"),
    P("bfloat16", 6000, 64, 16, "coarse", None, True, "0", id="mma-bf16-ties_low-coarse"),
    P("float16", 9000, 56, 130, "fine", "half", False, "0", id="mma-fp16-mask_half-B130_two_chunks"),
    P("bfloat16", 6000, 64, 16, "fine", "bit0", False, "-2", id="mma-bf16-mask_bit0"),
    P("float16", 6000, 64, 16, "coarse", "bit31", True, "0", id="mma-fp16-mask_bit31-ties_low"),
    P("bfloat16", 6000, 64, 16, "fine", None, False, "hit", id="mma-bf16-min_at_a_hit"),
    P("float16", 6000, 64, 16, "fine", None, False, "hit+ulp", id="mma-fp16-min_ulp_above_a_hit"),
    P("bfloat16", 6000, 64, 16, "fine", None, False, "hit-ulp", id="mma-bf16-min_ulp_below_a_hit"),
    P("bfloat16", 6000, 64, 16, "coarse", None, False, "1", id="mma-bf16-min1-clipped_ties"),
    P("float16", 6000, 64, 16, "fine", None, False, "1.5", id="mma-fp16-min_above_1-empty"),
    P("bfloat16", 100, 8, 16, "fine", None, False, "0", id="mma-bf16-N100-ragged_tile"),
    P("float32", 6000, 64, 20, "fine", None, False, "0", id="mma_split-min0"),
    P("float32", 6000, 136, 16, "coarse", "half", True, "-2", id="mma_split-radix-mask_half-ties_low"),
    P("float32", 6000, 64, 16, "fine", None, False, "hit-ulp", id="mma_split-min_ulp_below_a_hit"),
]


@pytest.mark.parametrize("storage,n,d,b,pre,mask,ties_low,ms_kind", DYADIC)
def test_dyadic_corpus_every_query(storage, n, d, b, pre, mask, ties_low, ms_kind):
    amp, exp = preset(pre, d)
    v, q, dots = dyadic_corpus(n, d, b, amp, exp, seed=n + d + b)
    allowed = row_mask(mask, n, seed=n)
    ms = min_score_for(ms_kind, dots, max(2, n // 8))
    base = make_base(v, storage, "scan")
    got = base.search_range(q, ms, allowed=allowed, ties_low_first=ties_low)
    assert_same_range(got, expected_range(dots, ms, allowed, ties_low), f"{storage} {ms_kind}")
    if ms_kind != "nan":
        t = base.last_timing()
        assert t["path"] == "scan", t


@pytest.mark.parametrize("storage,n,d,b,pre,mask,ties_low,ms_kind", DYADIC_MMA)
def test_dyadic_corpus_tensor_cores_every_query(storage, n, d, b, pre, mask, ties_low, ms_kind):
    amp, exp = preset(pre, d)
    v, q, dots = dyadic_corpus(n, d, b, amp, exp, seed=n + d + b + 1)
    allowed = row_mask(mask, n, seed=n)
    ms = min_score_for(ms_kind, dots, max(2, n // 8))
    base = make_base(v, storage, "mma")
    got = base.search_range(q, ms, allowed=allowed, ties_low_first=ties_low)
    assert_same_range(got, expected_range(dots, ms, allowed, ties_low), f"{storage} {ms_kind}")
    t = base.last_timing()
    assert t["path"] == ("mma_split" if storage == "float32" else "mma"), t
    assert main_kernels(base) == 1, t  # the default regions hold these hits: no re-pass
    # an unforced batch of >= 16 queries on >= 4096 rows takes the tensor cores too
    base.force_path = None
    if n >= 4096:
        assert_same_range(base.search_range(q, ms, allowed=allowed, ties_low_first=ties_low),
                          expected_range(dots, ms, allowed, ties_low), "unforced")
        assert base.last_timing()["path"] == t["path"]


@pytest.mark.parametrize("storage", ["bfloat16", "float32"])
def test_tensor_core_overflow_repass_equals_exact_hint(storage):
    amp, exp = preset("coarse", 64)
    v, q, dots = dyadic_corpus(7000, 64, 20, amp, exp, seed=77)
    want = expected_range(dots, -2.0)
    base = make_base(v, storage, "mma")
    base._range_hint = 1  # segments of ~34 keys: every segment of every query overflows
    assert_same_range(base.search_range(q, -2.0), want, "tiny hint")
    assert main_kernels(base) == 2, base.last_timing()  # one MAIN, one MAIN over the overflowed queries
    assert base._range_hint == want[0][-1]
    assert_same_range(base.search_range(q, -2.0), want, "exact hint")
    assert main_kernels(base) == 1, base.last_timing()


def test_split_form_beyond_fp16_range_goes_to_the_row_scan():
    amp, exp = preset("fine", 64)
    v, q, _ = dyadic_corpus(5000, 64, 16, amp, exp, seed=65)
    v = v.copy()
    v[5] = 70000.0  # beyond the fp16 range: the two-plane form cannot carry this row
    dots = (q.astype(np.float64) @ v.astype(np.float64).T).astype(np.float32)  # exact but for row 5's clipped sign
    base = make_base(v, "float32", "mma")
    assert_same_range(base.search_range(q, 0.0), expected_range(dots, 0.0), "split overflow")
    assert base.last_timing()["path"] == "scan"


@pytest.mark.parametrize("b", [1, 3])
def test_overflow_repass_equals_exact_hint(b):
    amp, exp = preset("fine", 64)
    v, q, dots = dyadic_corpus(7000, 64, b, amp, exp, seed=5 + b)
    want = expected_range(dots, 0.0)
    base = make_base(v, "bfloat16", "scan")
    base._range_hint = 1  # a region of 33 keys per query: every query overflows
    assert_same_range(base.search_range(q, 0.0), want, "tiny hint")
    assert main_kernels(base) == 2, base.last_timing()  # one scan, one re-pass of the overflowed queries
    base._range_hint = int(np.diff(want[0]).max()) * b  # exact: every query fits its region
    assert_same_range(base.search_range(q, 0.0), want, "exact hint")
    assert main_kernels(base) == 1, base.last_timing()
    assert base._range_hint == want[0][-1]


@pytest.mark.parametrize("storage,n,b,ms,mask,ties_low", [
    P("float32", 8192, 4, 0.0, None, False, id="f32-N8192"),
    P("bfloat16", 5000, 6, 0.52, None, False, id="bf16-min0.52"),
    P("float16", 3000, 3, 0.0, "half", False, id="fp16-mask_half"),
    P("float32", 2500, 2, 0.5, None, True, id="f32-ties_low"),
])
def test_equals_the_paged_top_k(storage, n, b, ms, mask, ties_low):
    """Random (not exact-arithmetic) rows: both forms compute the same float32 dots in the same kernel."""
    v, q = O.make_corpus(n, 96, seed=n + b, n_queries=b)
    allowed = row_mask(mask, n, seed=b)
    base = make_base(v, storage, "scan2")
    offsets, items, scores = base.search_range(q, ms, allowed=allowed, ties_low_first=ties_low)
    pi, ps, pc = base.search_arrays(q, n, ms, allowed=allowed, ties_low_first=ties_low)
    np.testing.assert_array_equal(np.diff(offsets), pc)
    for i in range(b):
        np.testing.assert_array_equal(items[offsets[i]:offsets[i + 1]], pi[i, :pc[i]])
        np.testing.assert_array_equal(scores[offsets[i]:offsets[i + 1]].view(np.uint32), ps[i, :pc[i]].view(np.uint32))


def test_fuzzy_lookup_max_hits_0_reads_the_rows_once():
    amp, exp = preset("fine", 64)
    v, q, dots = dyadic_corpus(20000, 64, 3, amp, exp, seed=20000)
    base = make_base(v, "float32", None)
    for ms in (0.0, float(np.float32(0.55))):
        got = base.fuzzy_lookup_embedding(q[0], max_hits=0, min_score=ms)
        _, wi, ws = expected_range(dots[:1], ms)
        assert [h.item for h in got] == wi.tolist()
        assert np.array_equal(np.array([h.score for h in got], np.float32).view(np.uint32), ws.view(np.uint32))
        assert main_kernels(base) == 1, base.last_timing()  # the paged form ran 10 scans (k = 20000)
    batch = base.fuzzy_lookup_embeddings(q, max_hits=0, min_score=0.5)
    wo, wi, ws = expected_range(dots, 0.5)
    for i in range(3):
        assert [h.item for h in batch[i]] == wi[wo[i]:wo[i + 1]].tolist()
        assert [h.score for h in batch[i]] == ws[wo[i]:wo[i + 1]].tolist()


def test_fetch_after_a_routed_lookup():
    """A max_hits=0 lookup on a fresh index leaves its hits fetchable like a threshold search's."""
    amp, exp = preset("fine", 32)
    v, q, dots = dyadic_corpus(9000, 32, 1, amp, exp, seed=90)
    base = make_base(v, "float32", None)
    got = base.fuzzy_lookup_embedding(q[0], max_hits=0, min_score=0.5)
    lib, ix = base._ensure_device()
    n = len(got)
    items, scores = np.empty(n, np.int64), np.empty(n, np.float32)
    _capi.check(lib.tav_range_fetch(ix, 0, n, items.ctypes.data_as(C.c_void_p), scores.ctypes.data_as(C.c_void_p),
                                    0, None))
    assert items.tolist() == [h.item for h in got] and scores.tolist() == [h.score for h in got]
    assert_same_range((np.array([0, n]), items, scores), expected_range(dots, 0.5), "routed")


def test_fuzzy_lookup_in_subset_max_hits_0():
    amp, exp = preset("fine", 48)
    v, q, dots = dyadic_corpus(12000, 48, 1, amp, exp, seed=9000)
    rng = np.random.default_rng(9)
    sub = rng.integers(-12000, 12000, size=9000)
    sub[100:200] = sub[0]  # duplicates
    sub = sub.tolist()
    base = make_base(v, "bfloat16", None)
    got = base.fuzzy_lookup_embedding_in_subset(q[0], sub, max_hits=0, min_score=0.5)
    assert main_kernels(base) == 1, base.last_timing()
    cols = np.asarray(sub) % 12000
    _, wi, ws = expected_range(dots[:, cols], 0.5, positions=sub)
    assert [h.item for h in got] == wi.tolist()
    assert [h.score for h in got] == ws.tolist()
    assert_hits_match(got, O.lookup_in_subset(v, q[0], sub, 0, 0.5), min_score=0.5)
    offsets, items, scores = base.search_range(q, 0.5, subset=sub)
    assert items.tolist() == wi.tolist() and scores.tolist() == ws.tolist()


@pytest.mark.parametrize("ties_low", [False, True])
def test_one_large_segment_heavy_ties(ties_low):
    amp, exp = preset("coarse", 16)
    v, q, dots = dyadic_corpus(300_000, 16, 1, amp, exp, seed=300)
    base = make_base(v, "bfloat16", "scan")
    got = base.search_range(q, -2.0, ties_low_first=ties_low)
    want = expected_range(dots, -2.0, ties_low=ties_low)
    assert want[0][-1] == 300_000 and len(np.unique(want[2])) < 1000  # every row, few distinct scores
    assert_same_range(got, want, "radix")


def test_edge_cases():
    amp, exp = preset("fine", 32)
    v, q, dots = dyadic_corpus(5000, 32, 2, amp, exp, seed=77)
    v = v.copy()
    v[[3, 4096, 4999]] = np.nan
    base = make_base(v, "float32", "scan")
    with np.errstate(invalid="ignore"):
        want = expected_range(q @ v.T, -2.0)
    got = base.search_range(q, -2.0)
    assert_same_range(got, want, "nan rows")
    assert not np.isin(got[1], [3, 4096, 4999]).any() and got[0][-1] == 2 * 4997
    # item_offset, offsets on the host, hits fetched in two pieces
    lib, ix = base._ensure_device()
    qq = np.ascontiguousarray(q)
    offsets = np.zeros(3, np.int64)
    _capi.check(lib.tav_range_search(ix, qq.ctypes.data_as(C.c_void_p), 2, C.c_float(0.5), 0, None, 0, 1000, 0,
                                     offsets.ctypes.data_as(C.c_void_p), None))
    total = int(offsets[-1])
    items, scores = np.empty(total, np.int64), np.empty(total, np.float32)
    for lo, hi in ((0, total // 3), (total // 3, total)):
        _capi.check(lib.tav_range_fetch(ix, lo, hi - lo, items[lo:].ctypes.data_as(C.c_void_p),
                                        scores[lo:].ctypes.data_as(C.c_void_p), 0, None))
    with np.errstate(invalid="ignore"):
        assert_same_range((offsets, items, scores), expected_range(q @ v.T, 0.5, item_offset=1000), "item_offset")
    with pytest.raises(IndexError):
        _capi.check(lib.tav_range_fetch(ix, total - 1, 2, items.ctypes.data_as(C.c_void_p),
                                        scores.ctypes.data_as(C.c_void_p), 0, None))
    # NaN min_score in the library itself: all-zero offsets, nothing to fetch
    offsets[:] = 7
    _capi.check(lib.tav_range_search(ix, qq.ctypes.data_as(C.c_void_p), 2, C.c_float(float("nan")), 0, None, 0, 0, 0,
                                     offsets.ctypes.data_as(C.c_void_p), None))
    assert (offsets == 0).all()
    with pytest.raises(IndexError):
        _capi.check(lib.tav_range_fetch(ix, 0, 1, items.ctypes.data_as(C.c_void_p),
                                        scores.ctypes.data_as(C.c_void_p), 0, None))
    # B = 0, an empty subset, FORCE_MMA with a subset refused
    _capi.check(lib.tav_range_search(ix, qq.ctypes.data_as(C.c_void_p), 0, C.c_float(0.0), 0, None, 0, 0, 0,
                                     offsets.ctypes.data_as(C.c_void_p), None))
    assert offsets[0] == 0
    empty = np.zeros(1, np.int64)
    offsets[:] = 7
    _capi.check(lib.tav_range_search(ix, qq.ctypes.data_as(C.c_void_p), 2, C.c_float(0.0), 0,
                                     empty.ctypes.data_as(C.c_void_p), 0, 0, 0, offsets.ctypes.data_as(C.c_void_p), None))
    assert (offsets == 0).all()
    with pytest.raises(ValueError):
        _capi.check(lib.tav_range_search(ix, qq.ctypes.data_as(C.c_void_p), 2, C.c_float(0.0), _capi.TAV_FORCE_MMA,
                                         empty.ctypes.data_as(C.c_void_p), 1, 0, 0,
                                         offsets.ctypes.data_as(C.c_void_p), None))
    got = base.search_range(q[:0], 0.0)
    assert got[0].tolist() == [0] and len(got[1]) == 0


def test_device_outputs():
    import torch

    amp, exp = preset("fine", 64)
    v, q, dots = dyadic_corpus(6000, 64, 3, amp, exp, seed=61)
    base = make_base(v, "float16", "scan")
    lib, ix = base._ensure_device()
    dq = torch.from_numpy(q).cuda()
    offs = torch.empty(4, dtype=torch.int64, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    flags = _capi.TAV_QUERIES_ON_DEVICE | _capi.TAV_OUTPUTS_ON_DEVICE
    _capi.check(lib.tav_range_search(ix, C.c_void_p(dq.data_ptr()), 3, C.c_float(0.0), flags, None, 0, 0, 0,
                                     C.c_void_p(offs.data_ptr()), C.c_void_p(stream)))
    want = expected_range(dots, 0.0)
    total = int(want[0][-1])
    items = torch.empty(total, dtype=torch.int64, device="cuda")
    scores = torch.empty(total, dtype=torch.float32, device="cuda")
    _capi.check(lib.tav_range_fetch(ix, 0, total, C.c_void_p(items.data_ptr()), C.c_void_p(scores.data_ptr()),
                                    _capi.TAV_OUTPUTS_ON_DEVICE, C.c_void_p(stream)))
    torch.cuda.synchronize()
    assert_same_range((offs.cpu().numpy(), items.cpu().numpy(), scores.cpu().numpy()), want, "device outputs")


def test_reference_parity_golden():
    """Recorded outputs of the unmodified reference: its max_hits=0 case whole, and on the Episode-53 excerpt the
    recorded top-k lists as the head of the every-passing-row lists."""
    golden = GC.load_golden()["cases"]
    checked = 0
    for case in GC.CASES:
        vectors, queries = GC.build_inputs(case)
        base = make_base(vectors, "float32", None)
        for (kind, kw), per_query in zip(case["lookups"], golden[case["name"]]):
            if kind != "lookup" or (kw.get("max_hits") != 0 and case["name"] != "episode53"):
                continue
            ms = kw.get("min_score") or 0.0
            got_all = base.fuzzy_lookup_embeddings(queries, max_hits=0, min_score=ms)
            for qi, (q, want) in enumerate(zip(queries, per_query)):
                got = base.fuzzy_lookup_embedding(q, max_hits=0, min_score=ms)
                assert [(h.item, h.score) for h in got] == [(h.item, h.score) for h in got_all[qi]]
                head = got[:len(want["items"])]
                assert_hits_match(head, want, score_tol=1e-4, min_score=ms, what=f"{case['name']}/{kw}/q{qi}")
                assert all(h.score >= np.float32(ms) for h in got)
                if kw.get("max_hits") == 0:
                    assert len(got) == len(want["items"])
                checked += 1
    assert checked >= 7 * 3 + 1
