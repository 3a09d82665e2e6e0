"""Per-query subsets from device tensors (``search_device`` / ``search_range_device`` with ``subsets=``,
``tav_search_subsets_into`` / ``tav_range_search_subsets_into``), bit for bit, no tolerances.

(1) every row equals ``search_arrays(subsets=)`` / ``search_range(subsets=)`` on the same index: three storages,
    widths 64, 768 and 67, subsets of 0 .. 100k entries with duplicates, negatives, one row repeated 10k times, empty
    subsets between non-empty ones and the planner's tile edges (255, 256, 257, 512 entries), k from 1 to beyond the
    longest subset, min_score at a hit's score and one ulp either side, NaN, both tie orders, flat positions;
(2) dyadic corpora: every query equals numpy's exact top-k / threshold set over its subset;
(3) a skewed batch: one query with 1M entries and 255 with 10;
(4) threshold capacity 0, below the total and exactly the total: complete offsets, untouched slots after it;
(5) no host synchronisation: a deferred call returns while the stream is held, and one finish completes deferred
    subset searches together with a deferred tensor-core ``search_device`` and ``search_range_device``;
(6) refused input (an ordinal N or -N-1, offsets[0] != 0, decreasing offsets, offsets[B] != n_ordinals),
    synchronous and deferred: the documented exception and outputs, exact valid searches, a usable index;
(7) CSR tensors made by torch kernels just before the call, a normalising index, row changes between calls;
(8) deliberately broken builds (``TAV_SUBSETS_DEVICE_MUTANT``), each caught by the checks here.
"""

from __future__ import annotations

import contextlib
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from tests.test_gpu_subsets import (STORAGES, WIDTHS, assert_bits, corpus, dyadic, exact_subset_topk, make_base,
                                    mixed_subsets, unit_corpus)
from typeagent_py_b200 import _capi

pytestmark = pytest.mark.gpu

N = 120_000  # the rows of tests/test_gpu_subsets.corpus


def cuda(a, dtype=None):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a, dtype)).cuda()


def dev_csr(subsets):
    """B host subsets -> (offsets, ordinals) int64 CUDA tensors."""
    lens = [len(s) for s in subsets]
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    ordinals = np.concatenate([np.asarray(s, np.int64).reshape(-1) for s in subsets]) if subsets else np.empty(0)
    return cuda(offsets, np.int64), cuda(ordinals, np.int64)


def edge_subsets(n, seed):
    """mixed_subsets plus empty subsets between non-empty ones and the planner's tile edges."""
    rng = np.random.default_rng(seed)
    out = []
    for s in mixed_subsets(n, seed):
        out += [s, np.empty(0, np.int64)]
    for m in (255, 256, 257, 512):
        out.append(rng.integers(-n, n, size=m))
    return out


def np3(ts):
    return tuple(t.cpu().numpy() for t in ts)


def host_topk(base, q, k, ms, subsets, tl=False):
    return base.search_arrays(q, k, ms, subsets=subsets, ties_low_first=tl)


def assert_topk_equal(got, want, k, what):
    items, scores, counts = got
    wi, ws, wc = want
    kk = wi.shape[1]
    assert items.shape == (len(wc), k), what
    assert_bits(counts, wc, what + " counts")
    m = min(k, kk)
    assert_bits(items[:, :m], wi[:, :m], what + " items")
    assert_bits(scores[:, :m], ws[:, :m], what + " scores")
    assert (items[:, m:] == -1).all() and (scores[:, m:] == 0).all(), what + " padding"


def assert_range_prefix(got, want, cap, what):
    offs, items, scores = got
    wo, wi, ws = want
    assert_bits(offs, wo, what + " offsets")
    n = min(cap, int(wo[-1]))
    assert_bits(items[:n], wi[:n], what + " items")
    assert_bits(scores[:n], ws[:n], what + " scores")


# ---- the C ABI on torch tensors -------------------------------------------------------------------------------
def ptr(t):
    return C.c_void_p(t.data_ptr() if t is not None else 0)


def c_topk(lib, ix, qd, k, ms, flags, off, ords, n_ord=None):
    import torch

    b = qd.shape[0]
    items = torch.full((b, k), -7, dtype=torch.int64, device=qd.device)
    scores = torch.full((b, k), 7.0, dtype=torch.float32, device=qd.device)
    counts = torch.full((b,), -7, dtype=torch.int32, device=qd.device)
    rc = lib.tav_search_subsets_into(ix, ptr(qd), b, k, C.c_float(ms), flags, ptr(off), ptr(ords),
                                     ords.numel() if n_ord is None else n_ord, ptr(items), ptr(scores), ptr(counts),
                                     C.c_void_p(torch.cuda.current_stream().cuda_stream))
    return rc, (items, scores, counts)


def c_range(lib, ix, qd, ms, flags, off, ords, cap):
    import torch

    b = qd.shape[0]
    offsets = torch.full((b + 1,), -7, dtype=torch.int64, device=qd.device)
    items = torch.full((max(cap, 1),), -7, dtype=torch.int64, device=qd.device)
    scores = torch.full((max(cap, 1),), 7.0, dtype=torch.float32, device=qd.device)
    rc = lib.tav_range_search_subsets_into(ix, ptr(qd), b, C.c_float(ms), flags, ptr(off), ptr(ords), ords.numel(),
                                           cap, ptr(offsets), ptr(items), ptr(scores),
                                           C.c_void_p(torch.cuda.current_stream().cuda_stream))
    return rc, (offsets, items, scores)


# ---------------------------------------------------------------- (1) equal to the host form
def equal_host_checks(base, q, subsets, what, ks=(1, 10, 100, 2049, 200_000)):
    lib, ix = base._ensure_device()
    qd = cuda(q)
    off, ords = dev_csr(subsets)
    for k in ks:
        got = np3(base.search_device(qd, k, 0.0, subsets=(off, ords)))
        assert_topk_equal(got, host_topk(base, q, k, 0.0, subsets), k, f"{what} k={k}")
        rc, got = c_topk(lib, ix, qd, k, 0.0, _capi.TAV_TIES_LOW_FIRST, off, ords)
        assert rc == 0
        assert_topk_equal(np3(got), host_topk(base, q, k, 0.0, subsets, True), k, f"{what} k={k} ties low")
    items, scores, counts = host_topk(base, q, 100, 0.0, subsets)
    s0 = np.float32(scores[6, 40])  # a hit of the 4096-entry query
    for ms in (s0, np.nextafter(s0, np.float32(-1)), np.nextafter(s0, np.float32(2)), float("nan")):
        ms = float(ms)
        got = np3(base.search_device(qd, 100, ms, subsets=(off, ords)))
        assert_topk_equal(got, host_topk(base, q, 100, ms, subsets), 100, f"{what} ms={ms!r}")
        for tl in (False, True):
            want = base.search_range(q, ms, subsets=subsets, ties_low_first=tl)
            cap = int(want[0][-1])
            got = np3(base.search_range_device(qd, ms, cap, subsets=(off, ords), ties_low_first=tl))
            assert_range_prefix(got, want, cap, f"{what} range ms={ms!r} ties_low={tl}")


@pytest.mark.parametrize("d", WIDTHS)
@pytest.mark.parametrize("storage", STORAGES)
def test_each_row_equals_the_host_form(storage, d):
    v, q8 = corpus(d)
    subsets = edge_subsets(N, seed=d)
    q = np.ascontiguousarray(np.resize(q8, (len(subsets), d)))
    base = make_base(v, storage)
    equal_host_checks(base, q, subsets, f"{storage} d={d}")
    base.enable_timing()
    off, ords = dev_csr(subsets)
    base.search_device(cuda(q), 10, 0.0, subsets=(off, ords))
    t = base.last_timing()
    assert t["path"] == "scan" and t["scan_ms"] > 0


def test_positions_through_the_c_abi():
    v, q = unit_corpus(5000, 64, 4, seed=31)
    base = make_base(v)
    lib, ix = base._ensure_device()
    subsets = [np.array([3, -2, 3, 4999]), np.arange(0, 5000, 7), np.empty(0, np.int64), np.full(300, -17)]
    offsets, ordinals = base._subsets_csr(subsets, 4)
    qd = cuda(q)
    off, ords = dev_csr(subsets)
    for tl in (0, _capi.TAV_TIES_LOW_FIRST):
        flags = tl | _capi.TAV_ITEMS_AS_POSITIONS
        want = np.zeros((4, 50), np.int64), np.zeros((4, 50), np.float32), np.zeros(4, np.int32)
        assert lib.tav_search_subsets(ix, q.ctypes.data_as(C.c_void_p), 4, 50, C.c_float(0.0), flags,
                                      offsets.ctypes.data_as(C.c_void_p), ordinals.ctypes.data_as(C.c_void_p),
                                      *[w.ctypes.data_as(C.c_void_p) for w in want], None) == 0
        rc, got = c_topk(lib, ix, qd, 50, 0.0, flags, off, ords)
        assert rc == 0
        for j in range(3):
            assert_bits(np3(got)[j], want[j], f"positions top-k ties={tl}")
        w_off = np.zeros(5, np.int64)
        assert lib.tav_range_search_subsets(ix, q.ctypes.data_as(C.c_void_p), 4, C.c_float(0.4), flags,
                                            offsets.ctypes.data_as(C.c_void_p), ordinals.ctypes.data_as(C.c_void_p),
                                            w_off.ctypes.data_as(C.c_void_p), None) == 0
        w_i, w_s = np.empty(w_off[-1], np.int64), np.empty(w_off[-1], np.float32)
        assert lib.tav_range_fetch(ix, 0, w_off[-1], w_i.ctypes.data_as(C.c_void_p), w_s.ctypes.data_as(C.c_void_p),
                                   0, None) == 0
        rc, got = c_range(lib, ix, qd, 0.4, flags, off, ords, int(w_off[-1]))
        assert rc == 0
        assert_range_prefix(np3(got), (w_off, w_i, w_s), int(w_off[-1]), f"positions range ties={tl}")
        # the device form replaced the range hits: nothing to fetch until the next tav_range_search
        assert lib.tav_range_fetch(ix, 0, 1, w_i.ctypes.data_as(C.c_void_p), w_s.ctypes.data_as(C.c_void_p), 0,
                                   None) == _capi.TAV_ERR_STATE
    for f in (_capi.TAV_FORCE_SCAN, _capi.TAV_FORCE_MMA, _capi.TAV_USE_ROW_MASK, _capi.TAV_USE_QUERY_MASKS,
              _capi.TAV_NO_FUSED_SCAN):
        assert c_topk(lib, ix, qd, 5, 0.0, f, off, ords)[0] == _capi.TAV_ERR_INVALID, f
        assert c_range(lib, ix, qd, 0.0, f, off, ords, 10)[0] == _capi.TAV_ERR_INVALID, f
    both = _capi.TAV_QUERIES_ON_DEVICE | _capi.TAV_OUTPUTS_ON_DEVICE
    rc, got = c_topk(lib, ix, qd, 50, 0.0, both, off, ords)
    assert rc == 0
    assert_topk_equal(np3(got), host_topk(base, q, 50, 0.0, subsets), 50, "_ON_DEVICE flags change nothing")
    assert c_topk(lib, ix, qd, 0, 0.0, 0, off, ords)[0] == _capi.TAV_ERR_INVALID
    assert c_topk(lib, ix, qd, 5, 0.0, 0, off, ords, n_ord=1 << 32)[0] == _capi.TAV_ERR_INVALID
    assert c_range(lib, ix, qd, 0.0, 0, off, ords, -1)[0] == _capi.TAV_ERR_INVALID
    import torch

    torch.cuda.synchronize()


# ---------------------------------------------------------------- (2) exact arithmetic, (3) skew
@pytest.mark.parametrize("storage", STORAGES)
def test_exact_topk_and_threshold_sets(storage):
    v, q, dots = dyadic(20_000, 64, 8, seed=5)
    base = make_base(v, storage)
    subsets = mixed_subsets(20_000, seed=6)
    subsets[5] = subsets[5][:30_000]
    qd = cuda(q)
    off, ords = dev_csr(subsets)
    lib, ix = base._ensure_device()
    for tl in (False, True):
        for k in (1, 10, 300, 5000, 40_000):
            want, _ = exact_subset_topk(dots, subsets, k, 0.0, tl)
            rc, got = c_topk(lib, ix, qd, k, 0.0, _capi.TAV_TIES_LOW_FIRST if tl else 0, off, ords)
            assert rc == 0
            assert_topk_equal(np3(got), want, k, f"exact top-k {storage} k={k} ties_low={tl}")
        for ms in (0.0, 0.55, 0.75):
            _, want = exact_subset_topk(dots, subsets, 1, ms, tl)
            got = np3(base.search_range_device(qd, ms, int(want[0][-1]), subsets=(off, ords), ties_low_first=tl))
            assert_range_prefix(got, want, int(want[0][-1]), f"exact range {storage} ms={ms} ties_low={tl}")


def test_one_huge_subset_and_many_tiny_ones():
    v, q, dots = dyadic(50_000, 64, 256, seed=9)
    rng = np.random.default_rng(10)
    subsets = [rng.integers(-50_000, 50_000, size=1_000_000)] + [rng.integers(50_000, size=10) for _ in range(255)]
    base = make_base(v, "bfloat16")
    qd = cuda(q)
    off, ords = dev_csr(subsets)
    for k in (10, 100):
        want, csr = exact_subset_topk(dots, subsets, k, 0.5)
        assert_topk_equal(np3(base.search_device(qd, k, 0.5, subsets=(off, ords))), want, k, f"skew top-k k={k}")
    got = np3(base.search_range_device(qd, 0.5, int(csr[0][-1]), subsets=(off, ords)))
    assert_range_prefix(got, csr, int(csr[0][-1]), "skew range")


# ---------------------------------------------------------------- (4) capacity
def test_capacity_prefix_and_untouched_slots():
    import torch

    v, q, dots = dyadic(20_000, 64, 8, seed=41)
    subsets = mixed_subsets(20_000, seed=42)
    base = make_base(v, "float16")
    _, want = exact_subset_topk(dots, subsets, 1, 0.5)
    total = int(want[0][-1])
    assert total > 1000
    qd = cuda(q)
    off, ords = dev_csr(subsets)
    for cap in (0, 1, total // 3, total - 1, total):
        room = cap + 50
        out = (torch.full((9,), -7, dtype=torch.int64, device="cuda"),
               torch.full((room,), -7, dtype=torch.int64, device="cuda"),
               torch.full((room,), 7.0, dtype=torch.float32, device="cuda"))
        for defer in (False, True):
            base.search_range_device(qd, 0.5, cap, out=out, subsets=(off, ords), defer_check=defer)
            if defer:
                assert base.finish_search() == 0
            o, i, s = np3(out)
            assert_range_prefix((o, i, s), want, cap, f"capacity {cap} defer={defer}")
            assert (i[cap:] == -7).all() and (s[cap:] == 7.0).all(), f"capacity {cap}: slots from cap written"


# ---------------------------------------------------------------- (5) no host synchronisation
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


def test_deferred_calls_do_not_synchronise_and_finish_together(hold_cycles):
    import torch

    from tests.exact import expected_topk

    v, q, dots = dyadic(6000, 64, 16, seed=51)
    base = make_base(v, "bfloat16")
    base.force_path = "mma"  # the plain search_device below runs on the tensor cores
    subsets = mixed_subsets(6000, seed=52) * 2
    subsets[5] = subsets[5][:20_000]
    subsets[13] = subsets[13][:7000]
    qd = cuda(q)
    off, ords = dev_csr(subsets)
    want_t, want_r = exact_subset_topk(dots, subsets, 100, 0.45)
    cap = int(want_r[0][-1])
    # warm-up: buffers of these shapes
    base.search_device(qd, 100, 0.45, subsets=(off, ords), defer_check=True)
    base.search_range_device(qd, 0.45, cap, subsets=(off, ords), defer_check=True)
    base.finish_search()
    stream = torch.cuda.current_stream()
    torch.cuda._sleep(hold_cycles)
    t1 = base.search_device(qd, 100, 0.45, subsets=(off, ords), defer_check=True)
    r1 = base.search_range_device(qd, 0.45, cap, subsets=(off, ords), defer_check=True)
    assert not stream.query(), "a deferred subsets call waited for the stream"
    plain = base.search_device(qd, 50, 0.0, defer_check=True)
    rng_all = base.search_range_device(qd, 0.45, 200_000, defer_check=True)
    t2 = base.search_device(qd, 3000, 0.0, subsets=(off, ords), defer_check=True)
    r2 = base.search_range_device(qd, 0.0, 10, subsets=(off, ords), defer_check=True, ties_low_first=True)
    assert base.finish_search() == 0
    torch.cuda.synchronize()
    assert_topk_equal(np3(t1), want_t, 100, "deferred top-k")
    assert_range_prefix(np3(r1), want_r, cap, "deferred range")
    assert_topk_equal(np3(t2), exact_subset_topk(dots, subsets, 3000, 0.0)[0], 3000, "deferred top-k 3000")
    assert_range_prefix(np3(r2), exact_subset_topk(dots, subsets, 1, 0.0, True)[1], 10, "deferred range cap 10")
    wi, ws, wc = expected_topk(dots, 50, 0.0)
    for j, w in enumerate((wi, ws, wc)):
        assert_bits(np3(plain)[j], w, "deferred tensor-core search_device")
    o, i, s = np3(rng_all)
    from tests.test_gpu_range_device import expected_range

    wo, wi2, ws2 = expected_range(dots, 0.45)
    assert_range_prefix((o, i, s), (wo, wi2, ws2), 200_000, "deferred search_range_device")


# ---------------------------------------------------------------- (6) refused input
def refusals(n, offsets, ordinals):
    """(what, offsets, ordinals, exception) of every documented refusal of a valid CSR."""
    bad_hi, bad_lo = ordinals.copy(), ordinals.copy()
    bad_hi[len(ordinals) // 2] = n
    bad_lo[-1] = -n - 1
    first = offsets.copy()
    first[0] = 1
    dec = offsets.copy()
    dec[2] = dec[1] - 1
    last = offsets.copy()
    last[-1] -= 1
    return [("ordinal N", offsets, bad_hi, IndexError), ("ordinal -N-1", offsets, bad_lo, IndexError),
            ("offsets[0] != 0", first, ordinals, ValueError), ("decreasing offsets", dec, ordinals, ValueError),
            ("offsets[B] != n_ordinals", last, ordinals, ValueError)]


def test_refused_input_sync_and_deferred():
    import torch

    v, q, dots = dyadic(20_000, 64, 6, seed=61)
    base = make_base(v, "bfloat16")
    subsets = [np.arange(0, 20_000, 9), np.array([4, -4, 4]), np.empty(0, np.int64), np.arange(-300, 0),
               np.full(600, 7), np.arange(256)]
    offsets, ordinals = base._subsets_csr(subsets, 6)
    qd = cuda(q)
    good = dev_csr(subsets)
    want_t, want_r = exact_subset_topk(dots, subsets, 20, 0.5)
    cap = int(want_r[0][-1])

    def sentinel_out(room):
        return (torch.full((7,), -7, dtype=torch.int64, device="cuda"),
                torch.full((room,), -7, dtype=torch.int64, device="cuda"),
                torch.full((room,), 7.0, dtype=torch.float32, device="cuda"))

    def assert_refused(t, r, what):
        items, scores, counts = np3(t)
        assert (counts == 0).all() and (items == -1).all() and (scores == 0).all(), what + " top-k outputs"
        o, i, s = np3(r)
        assert (o == 0).all() and (i == -7).all() and (s == 7.0).all(), what + " threshold outputs"

    for what, bad_off, bad_ord, exc in refusals(20_000, offsets, ordinals):
        bad = (cuda(bad_off, np.int64), cuda(bad_ord, np.int64))
        t = tuple(torch.full(shape, 5, dtype=dt, device="cuda")
                  for shape, dt in (((6, 20), torch.int64), ((6, 20), torch.float32), ((6,), torch.int32)))
        with pytest.raises(exc):
            base.search_device(qd, 20, 0.5, subsets=bad, out=t)
        r = sentinel_out(cap)
        with pytest.raises(exc):
            base.search_range_device(qd, 0.5, cap, out=r, subsets=bad)
        assert_refused(t, r, what + " (synchronous)")
        # deferred, between valid searches: one finish completes them all, then raises
        v1 = base.search_device(qd, 20, 0.5, subsets=good, defer_check=True)
        t = base.search_device(qd, 20, 0.5, subsets=bad, defer_check=True)
        r = sentinel_out(cap)
        base.search_range_device(qd, 0.5, cap, out=r, subsets=bad, defer_check=True)
        v2 = base.search_range_device(qd, 0.5, cap, subsets=good, defer_check=True)
        with pytest.raises(exc):
            base.finish_search()
        assert base._pending == []
        assert base.finish_search() == 0  # nothing left
        torch.cuda.synchronize()
        assert_refused(t, r, what + " (deferred)")
        assert_topk_equal(np3(v1), want_t, 20, what + ": valid deferred top-k")
        assert_range_prefix(np3(v2), want_r, cap, what + ": valid deferred range")
        # the index is still usable, synchronously and on the host path
        assert_topk_equal(np3(base.search_device(qd, 20, 0.5, subsets=good)), want_t, 20, what + ": afterwards")
        got = base.search_arrays(q, 20, 0.5, subsets=subsets)
        assert_topk_equal(tuple(np.asarray(g) for g in got), want_t, got[0].shape[1], what + ": host form afterwards")


def test_empty_cases_do_no_work():
    import torch

    v, q = unit_corpus(1000, 64, 3, seed=71)
    base = make_base(v)
    qd = cuda(q)
    empty = (cuda(np.zeros(4), np.int64), cuda(np.empty(0), np.int64))
    items, scores, counts = np3(base.search_device(qd, 5, 0.0, subsets=empty))
    assert (items == -1).all() and (scores == 0).all() and (counts == 0).all()
    nan_csr = dev_csr([[1, 2], [3], [5000]])  # not looked at: NaN admits nothing
    items, scores, counts = np3(base.search_device(qd, 5, float("nan"), subsets=nan_csr))
    assert (counts == 0).all() and (items == -1).all()
    o, _, _ = np3(base.search_range_device(qd, float("nan"), 4, subsets=nan_csr))
    assert (o == 0).all()
    o, _, _ = np3(base.search_range_device(qd[:0], 0.0, 4, subsets=(cuda([0], np.int64), cuda(np.empty(0), np.int64))))
    assert o.tolist() == [0]
    torch.cuda.synchronize()


# ---------------------------------------------------------------- (7) torch-made CSR, normalisation, row changes
def test_csr_made_by_torch_kernels_just_before_the_call():
    import torch

    v, q, dots = dyadic(30_000, 64, 8, seed=81)
    base = make_base(v, "float32")
    subsets = mixed_subsets(30_000, seed=82)
    want_t, want_r = exact_subset_topk(dots, subsets, 50, 0.5)
    lens_h = np.array([len(s) for s in subsets], np.int64)
    flat_h = np.concatenate([np.asarray(s, np.int64) for s in subsets])
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        lens = cuda(lens_h)
        flat = cuda(flat_h)
        torch.cuda._sleep(2_000_000)  # the kernels below run late on this stream
        off = torch.cat([torch.zeros(1, dtype=torch.int64, device="cuda"), torch.cumsum(lens, 0)])
        ords = (flat + 30_000) - 30_000  # a fresh tensor from an elementwise kernel
        t = base.search_device(cuda(q), 50, 0.5, subsets=(off, ords))
        r = base.search_range_device(cuda(q), 0.5, int(want_r[0][-1]), subsets=(off, ords))
    side.synchronize()
    assert_topk_equal(np3(t), want_t, 50, "torch-made CSR top-k")
    assert_range_prefix(np3(r), want_r, int(want_r[0][-1]), "torch-made CSR range")


@pytest.mark.parametrize("storage", ["float32", "bfloat16"])
def test_normalising_index(storage):
    rng = np.random.default_rng(12)
    v = rng.standard_normal((30_000, 96), dtype=np.float32) * np.float32(7.0)
    q = rng.standard_normal((8, 96), dtype=np.float32) * np.float32(3.0)
    base = make_base(v, storage, normalize=True)
    subsets = mixed_subsets(30_000, seed=13)
    subsets[5] = subsets[5][:20_000]
    equal_host_checks(base, q, subsets, f"normalize {storage}", ks=(1, 100, 50_000))
    # deferred: the normalised queries are the search's own until the finish
    qd, (off, ords) = cuda(q), dev_csr(subsets)
    # (power-of-two multiples of a query normalise to the same query, exactly)
    got = [base.search_device(qd * 2.0 ** i, 100, 0.0, subsets=(off, ords), defer_check=True) for i in range(3)]
    base.finish_search()
    for g in got:
        assert_topk_equal(np3(g), host_topk(base, q, 100, 0.0, subsets), 100, f"normalize {storage} deferred")


def test_row_changes_between_calls():
    v, q = unit_corpus(40_000, 64, 8, seed=14)
    base = make_base(v, "bfloat16")
    subsets = mixed_subsets(40_000, seed=15)
    subsets[5] = subsets[5][:30_000]
    qd = cuda(q)
    base.search_device(qd, 10, 0.0, subsets=dev_csr(subsets))  # rows on the device before they change
    extra, _ = unit_corpus(1000, 64, 1, seed=16)
    base.add_embeddings(None, extra)
    base.remove_embeddings(np.arange(100, 1100))
    base.set_embeddings_at(500, extra[:200])
    n = len(base)
    subsets = [np.asarray(s, np.int64) % n - (n if i % 2 else 0) for i, s in enumerate(mixed_subsets(n, seed=17))]
    off, ords = dev_csr(subsets)
    for k in (10, 3000):
        got = np3(base.search_device(qd, k, 0.0, subsets=(off, ords)))
        assert_topk_equal(got, host_topk(base, q, k, 0.0, subsets), k, f"after row changes k={k}")
    want = base.search_range(q, 0.55, subsets=subsets)
    got = np3(base.search_range_device(qd, 0.55, int(want[0][-1]), subsets=(off, ords)))
    assert_range_prefix(got, want, int(want[0][-1]), "range after row changes")


# ---------------------------------------------------------------- (8) broken builds
MUTANTS = {1: "planner drops the last tile of a whole-tile query", 2: "deferred finish ignores the status word",
           3: "sort plan ignores the status word"}


@pytest.fixture(scope="module")
def mutant_libs():
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc) and not shutil.which(nvcc):
        pytest.skip("nvcc is needed to build the broken variants")
    from typeagent_py_b200 import build as B

    tmp = tempfile.mkdtemp(prefix="tav_subsets_device_mutants_")
    procs = {}
    for m in MUTANTS:
        out = os.path.join(tmp, f"libtavec_mutant{m}.so")
        cmd = [nvcc, *[f for f in B.NVCC_FLAGS if f != "-Xptxas=-v"], f"-DTAV_SUBSETS_DEVICE_MUTANT={m}", "-o", out,
               *[os.path.join(B.CSRC, s) for s in B.SOURCES]]
        procs[m] = (subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True), out)
    libs = {}
    for m, (proc, out) in procs.items():
        log = proc.communicate()[0]
        assert proc.returncode == 0, log
        lib = C.CDLL(out)
        for name, (restype, argtypes) in _capi.SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = restype, argtypes
        libs[m] = lib
    yield libs
    shutil.rmtree(tmp, ignore_errors=True)


@contextlib.contextmanager
def library(lib):
    saved = _capi._lib
    _capi._lib = lib
    try:
        yield
    finally:
        _capi._lib = saved


def mutant_checks():
    """The checks above, condensed: (AssertionError messages of) what fails."""
    import torch

    v, q = unit_corpus(20_000, 64, 8, seed=20)
    subsets = [np.arange(256), np.arange(-512, 0), np.arange(3, 20_000, 41), np.full(1024, 9), np.arange(257),
               np.empty(0, np.int64), np.arange(100, 355), np.arange(600)]
    caught = []
    base = make_base(v, "bfloat16")
    qd = cuda(q)
    good = dev_csr(subsets)
    offsets, ordinals = base._subsets_csr(subsets, 8)
    bad = (cuda(offsets, np.int64), cuda(np.where(np.arange(len(ordinals)) == 5, 20_000, ordinals), np.int64))
    try:
        assert_topk_equal(np3(base.search_device(qd, 100, 0.0, subsets=good)), host_topk(base, q, 100, 0.0, subsets),
                          100, "mutant check top-k")
        want = base.search_range(q, 0.5, subsets=subsets)
        got = np3(base.search_range_device(qd, 0.5, int(want[0][-1]), subsets=good))
        assert_range_prefix(got, want, int(want[0][-1]), "mutant check range")
    except AssertionError as e:
        caught.append(str(e)[:200])
    try:
        with pytest.raises(IndexError):
            base.search_range_device(qd, 0.5, 100, subsets=bad)
        r = base.search_range_device(qd, 0.5, 100, subsets=bad, defer_check=True)
        try:
            base.finish_search()
            caught.append("a deferred refusal was not reported")
        except IndexError:
            pass
        torch.cuda.synchronize()
        assert (r[0].cpu().numpy() == 0).all(), "a refused search left offsets"
    except (AssertionError, pytest.fail.Exception) as e:
        caught.append(str(e)[:200])
    return caught


@pytest.mark.parametrize("m", sorted(MUTANTS), ids=[MUTANTS[m].replace(" ", "_") for m in sorted(MUTANTS)])
def test_broken_build_is_caught(mutant_libs, m):
    with library(mutant_libs[m]):
        caught = mutant_checks()
    assert caught, f"the checks did not catch: {MUTANTS[m]}"


def test_checks_pass_on_the_real_build():
    assert mutant_checks() == []
