"""Stream order: every call on an index must see exactly the state that the calls before it left, whatever
stream each call names (include/tavec.h, "Threading").

All the other GPU tests run on the legacy default stream. There the device runs the calls one after the other,
whatever the library does. This file moves work to other streams, as a serving process does. The work under
test is queued on a side stream behind a hold: a ``torch.cuda._sleep`` of about 200 ms. The racing call is then
made from the host while the hold still runs, on another stream or on the legacy stream. torch's pool streams
are non-blocking, so the legacy stream does not wait for them either.

If the library did not order the calls itself, the racing call would run first. It would change the mask, the
rows or the hits under the queued call, or finish a deferred search before that search ran. The queued work and
the racing work still never run at the same time, so such a mistake shows up as a wrong result. Each scenario
runs once. A window that closed before the racing call fails as "hold too short" instead of passing. Every
expectation is exact: dyadic corpora (tests/exact.py), or identical rows whose exact answer is rows
n-1, n-2, ... Every query is compared bit for bit."""

from __future__ import annotations

import ctypes as C
import threading

import numpy as np
import pytest

import typeagent_py_b200 as tab
from oracle import vectorbase_oracle as O
from tests.exact import dyadic_corpus, expected_topk, preset, round_to, scores_of, unit_rows
from tests.test_gpu_exact import assert_equal_results, row_mask
from tests.test_gpu_ingest import assert_same_values
from tests.test_gpu_range import assert_same_range, expected_range
from typeagent_py_b200 import _capi

pytestmark = pytest.mark.gpu

HOLD_MS = 200.0


# ------------------------------------------------------------------ the race window
@pytest.fixture(scope="session")
def hold_cycles():
    """Clock cycles of torch.cuda._sleep that last about HOLD_MS, measured once with CUDA events."""
    import torch

    torch.cuda._sleep(1000)  # loads the kernel
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    cycles = 20_000_000
    start.record()
    torch.cuda._sleep(cycles)
    end.record()
    end.synchronize()
    return int(cycles * HOLD_MS / start.elapsed_time(end))


@pytest.fixture
def hold(hold_cycles):
    """hold(stream): delay everything queued on `stream` after this by about HOLD_MS."""
    import torch

    def enqueue(stream):
        with torch.cuda.stream(stream):
            torch.cuda._sleep(hold_cycles)

    return enqueue


def window_open(stream):
    assert not stream.query(), "hold too short: the queued work ended before the racing call was made"


# ------------------------------------------------------------------ data and plumbing
def dyadic(n, d, b, seed, pre="fine"):
    amp, exp = preset(pre, d)
    return dyadic_corpus(n, d, b, amp, exp, seed)


def exact_dots(q, v):
    """float32 dots of dyadic queries and rows: every product and partial sum is exact in float64."""
    return (np.asarray(q, np.float64) @ np.asarray(v, np.float64).T).astype(np.float32)


def identical_rows(n, d, b, seed):
    """n copies of one dyadic row, and b dyadic queries. Every score of a query ties, which overflows the
    tensor-core search's candidates and flags every query. The exact answer is rows n-1, n-2, ..."""
    v, q, _ = dyadic(1, d, b, seed)
    rows = np.repeat(v, n, axis=0)
    return rows, q, exact_dots(q, rows)


def cuda(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def device_out(b, k):
    """Result tensors, allocated on the current stream."""
    import torch

    return (torch.empty((b, k), dtype=torch.int64, device="cuda"), torch.empty((b, k), dtype=torch.float32, device="cuda"),
            torch.empty(b, dtype=torch.int32, device="cuda"))


def host(res):
    return tuple(t.cpu().numpy() for t in res)


def hits_as_arrays(lists, k):
    items, scores = np.full((len(lists), k), -1, np.int64), np.zeros((len(lists), k), np.float32)
    counts = np.array([len(h) for h in lists], np.int32)
    for b, hits in enumerate(lists):
        items[b, :len(hits)] = [h.item for h in hits]
        scores[b, :len(hits)] = [h.score for h in hits]
    return items, scores, counts


def vbase(v, storage, path, normalize=False):
    base = tab.VectorBase(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()), storage_dtype=storage,
                          normalize=normalize)
    base.add_embeddings(None, v)
    base.force_path = path
    return base


def sp(stream):
    return None if stream is None else C.c_void_p(stream.cuda_stream)


class Raw:
    """A bare libtavec index, driven through the C ABI with explicit streams (None: the legacy stream)."""

    def __init__(self, storage, d, reserve):
        self.lib, self.h, self.d = _capi.load(), C.c_void_p(), d
        _capi.check(self.lib.tav_create(0, d, _capi.DTYPE_CODES[storage], 0, reserve, C.byref(self.h)))

    def append(self, rows, stream=None):
        """float32 rows from host memory (numpy) or device memory (a CUDA tensor)."""
        if isinstance(rows, np.ndarray):
            rows = np.ascontiguousarray(rows, np.float32)
            ptr, n, on_device = rows.ctypes.data_as(C.c_void_p), len(rows), 0
        else:
            ptr, n, on_device = C.c_void_p(rows.data_ptr()), rows.shape[0], 1
        _capi.check(self.lib.tav_append(self.h, ptr, n, self.d, _capi.TAV_F32, on_device, sp(stream)))

    def search(self, q, k, ms, flags=0, stream=None):
        """Host queries, host outputs."""
        q = np.ascontiguousarray(q, np.float32)
        items, scores, counts = np.empty((len(q), k), np.int64), np.empty((len(q), k), np.float32), np.empty(len(q), np.int32)
        _capi.check(self.lib.tav_search(self.h, q.ctypes.data_as(C.c_void_p), len(q), k, ms, flags, None, 0, 0,
                                        items.ctypes.data_as(C.c_void_p), scores.ctypes.data_as(C.c_void_p),
                                        counts.ctypes.data_as(C.c_void_p), sp(stream)))
        return items, scores, counts

    def search_device(self, qd, k, ms, out, flags, stream):
        flags |= _capi.TAV_QUERIES_ON_DEVICE | _capi.TAV_OUTPUTS_ON_DEVICE
        _capi.check(self.lib.tav_search(self.h, C.c_void_p(qd.data_ptr()), qd.shape[0], k, ms, flags, None, 0, 0,
                                        *(C.c_void_p(t.data_ptr()) for t in out), sp(stream)))

    def finish(self, stream):
        redone = C.c_int(0)
        _capi.check(self.lib.tav_finish_search(self.h, sp(stream), C.byref(redone)))
        return redone.value

    def read(self, stream=None):
        out = np.empty((self.lib.tav_size(self.h), self.d), np.float32)
        _capi.check(self.lib.tav_read_rows(self.h, 0, len(out), out.ctypes.data_as(C.c_void_p), sp(stream)))
        return out

    def set_mask(self, bits, n, stream=None):
        """Packed uint32 words from host memory (numpy) or device memory (a CUDA tensor)."""
        if isinstance(bits, np.ndarray):
            ptr, on_device = np.ascontiguousarray(bits).ctypes.data_as(C.c_void_p), 0
        else:
            ptr, on_device = C.c_void_p(bits.data_ptr()), 1
        _capi.check(self.lib.tav_set_row_mask(self.h, ptr, n, on_device, sp(stream)))

    def range_search(self, q, ms, stream=None):
        q = np.ascontiguousarray(q, np.float32)
        offsets = np.empty(len(q) + 1, np.int64)
        _capi.check(self.lib.tav_range_search(self.h, q.ctypes.data_as(C.c_void_p), len(q), ms, _capi.TAV_FORCE_SCAN,
                                              None, 0, 0, 0, offsets.ctypes.data_as(C.c_void_p), sp(stream)))
        return offsets

    def range_fetch(self, n, items, scores, flags=0, stream=None):
        _capi.check(self.lib.tav_range_fetch(self.h, 0, n, items, scores, flags, sp(stream)))

    def close(self):
        self.lib.tav_destroy(self.h)


def raw_with_decoys(storage, v0, v1, warm_up):
    """A bare index that holds v0, with capacity for v1 as well. The storage rows after v0 hold decoys, -v1, so
    a search or a read that ran before v1's append would see them rather than stale copies of v1. They were
    written by an append of v0 and the decoys and then dropped by tav_clear. ``warm_up(ix)`` runs at full size
    in between, so the racing call allocates nothing."""
    ix = Raw(storage, v0.shape[1], len(v0) + len(v1))
    ix.append(np.concatenate([v0, -v1]))
    warm_up(ix)
    _capi.check(ix.lib.tav_clear(ix.h))
    ix.append(v0)
    return ix


# ------------------------------------------------------------------ scenarios through the Python class
def py_mask_swap(hold, path):
    """Two masked searches in one `with torch.cuda.stream(side)` block: the masks are uploaded on the legacy
    stream, the searches run on `side`."""
    import torch

    storage, defer = ("float32", False) if path == "scan" else ("bfloat16", True)
    n, d, b, k = 6000, 64, 16, 10
    v, q, dots = dyadic(n, d, b, seed=101)
    m1, m2 = row_mask("half", n, seed=1), row_mask("half", n, seed=2)
    base = vbase(v, storage, "scan" if path == "scan" else "mma")
    qd = cuda(q)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        out1, out2 = device_out(b, k), device_out(b, k)
        base.search_device(qd, k, 0.0, out=out1, defer_check=defer, allowed=row_mask("half", n, seed=3))
        base.finish_search()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        hold(side)
        base.search_device(qd, k, 0.0, out=out1, defer_check=defer, allowed=m1)
        window_open(side)
        base.search_device(qd, k, 0.0, out=out2, defer_check=defer, allowed=m2)
    base.finish_search()
    torch.cuda.synchronize()
    assert_equal_results(host(out1), expected_topk(dots, k, 0.0, m1), "the first search (mask m1)")
    assert_equal_results(host(out2), expected_topk(dots, k, 0.0, m2), "the second search (mask m2)")


def py_corpus_replaced(hold):
    """A search queued on `side`, then deserialize() and a search: the new rows are cleared and appended on the
    legacy stream."""
    import torch

    n, d, b, k = 6000, 64, 8, 10
    v, q, dots = dyadic(n, d, b, seed=102)
    v2 = dyadic(n, d, 1, seed=103)[0]
    base = vbase(v, "float32", "scan")
    qd = cuda(q)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        out1, out2 = device_out(b, k), device_out(b, k)
        base.search_device(qd, k, 0.0, out=out1)
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        hold(side)
        base.search_device(qd, k, 0.0, out=out1)
        window_open(side)
        base.deserialize(v2)
        base.search_device(qd, k, 0.0, out=out2)
    torch.cuda.synchronize()
    assert_equal_results(host(out1), expected_topk(dots, k, 0.0), "the search on the first corpus")
    assert_equal_results(host(out2), expected_topk(exact_dots(q, v2), k, 0.0), "the search on the second corpus")


def py_defer_then(hold, racing):
    """A deferred tensor-core search on `side` that flags every query, then a call that finishes it on the legacy
    stream: a mask upload before a masked search, or a batched host lookup."""
    import torch

    n, d, b, k = 30000, 64, 5, 9
    rows, q, dots = identical_rows(n, d, b, seed=104)
    allowed = row_mask("half", n, seed=5)
    base = vbase(rows, "bfloat16", "mma")
    qd = cuda(q)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        out1, out2 = device_out(b, k), device_out(b, k)
        base.search_device(qd, k, 0.0, out=out1, defer_check=True)
        assert base.finish_search() == b
        if racing == "mask":
            base.search_device(qd, k, 0.0, out=out2, allowed=row_mask("half", n, seed=6))
        else:
            base.fuzzy_lookup_embeddings(q, max_hits=k, min_score=0.0)
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        hold(side)
        base.search_device(qd, k, 0.0, out=out1, defer_check=True)
        window_open(side)
        if racing == "mask":
            base.search_device(qd, k, 0.0, out=out2, allowed=allowed)
        else:
            got = hits_as_arrays(base.fuzzy_lookup_embeddings(q, max_hits=k, min_score=0.0), k)
    base.finish_search()
    torch.cuda.synchronize()
    assert_equal_results(host(out1), expected_topk(dots, k, 0.0), "the deferred search")
    if racing == "mask":
        assert_equal_results(host(out2), expected_topk(dots, k, 0.0, allowed), "the masked search")
    else:
        assert_equal_results(got, expected_topk(dots, k, 0.0), "the host lookup")


def py_defer_normalize(hold):
    """Deferred searches on a normalising index (each keeps its normalised queries in a region of its own): one
    on A behind the hold, one on B, then finish_search() on B."""
    import torch

    d, n, b, k = 64, 30000, 16, 7
    v, a, m, _ = unit_rows(1, d, 255, seed=3)
    qs, qi, mq, _ = unit_rows(2 * b, d, 255, seed=4)
    unit, qunit = a[0] * 2.0 ** -m, qi * 2.0 ** -mq  # the exact normalised forms
    base = vbase(np.repeat(v, n, axis=0), "bfloat16", "mma", normalize=True)
    qa, qb = cuda(qs[:b]), cuda(qs[b:])
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(sa):
        out_a = device_out(b, k)
        base.search_device(qa, k, -2.0, out=out_a, defer_check=True)
    with torch.cuda.stream(sb):
        out_b = device_out(b, k)
        base.search_device(qb, k, -2.0, out=out_b, defer_check=True)
    torch.cuda.synchronize()
    assert base.finish_search() == 2 * b
    with torch.cuda.stream(sa):
        hold(sa)
        base.search_device(qa, k, -2.0, out=out_a, defer_check=True)
    with torch.cuda.stream(sb):
        window_open(sa)
        base.search_device(qb, k, -2.0, out=out_b, defer_check=True)
    redone = base.finish_search()
    torch.cuda.synchronize()
    for what, out, qn in (("A", out_a, qunit[:b]), ("B", out_b, qunit[b:])):
        s = np.repeat(scores_of((qn @ unit).astype(np.float32))[:, None], k, axis=1)
        want = (np.tile(np.arange(n - 1, n - 1 - k, -1), (b, 1)), s, np.full(b, k, np.int32))
        assert_equal_results(host(out), want, f"deferred search {what}")
    assert redone == 2 * b, "finish_search must redo every query of both searches"


# ------------------------------------------------------------------ scenarios through the C ABI
def abi_append_then_search(hold, where):
    """An append queued on A, then a search with host outputs on B (host source: float32 rows, B the legacy
    stream; device source: conversion to bf16, B a second stream)."""
    import torch

    storage, seed = ("float32", 105) if where == "host" else ("bfloat16", 106)
    n0, n1, d, b, k = 3000, 1000, 64, 4, 16
    v, q, dots = dyadic(n0 + n1, d, b, seed=seed)
    sa = torch.cuda.Stream()
    sb = None if where == "host" else torch.cuda.Stream()
    ix = raw_with_decoys(storage, v[:n0], v[n0:], lambda ix: ix.search(q, k, 0.0, stream=sb))
    try:
        src = v[n0:] if where == "host" else cuda(v[n0:])
        torch.cuda.synchronize()
        hold(sa)
        ix.append(src, stream=sa)
        window_open(sa)
        got = ix.search(q, k, 0.0, stream=sb)
        assert_equal_results(got, expected_topk(dots, k, 0.0), f"search after a {where} append")
    finally:
        torch.cuda.synchronize()
        ix.close()


def abi_append_then_reserve(hold):
    """A host append queued on A (float32 -> bf16), then tav_reserve to twice the capacity and a read of the rows."""
    import torch

    n0, n1, d = 3000, 1000, 100
    rng = np.random.default_rng(110)
    v = (rng.standard_normal((n0 + n1, d)) * 3).astype(np.float32)
    sa = torch.cuda.Stream()
    ix = raw_with_decoys("bfloat16", v[:n0], v[n0:], lambda ix: ix.read())
    try:
        hold(sa)
        ix.append(v[n0:], stream=sa)
        window_open(sa)
        _capi.check(ix.lib.tav_reserve(ix.h, 2 * (n0 + n1)))
        assert_same_values(ix.read(), round_to(v, "bfloat16"), "rows after the reserve")
    finally:
        torch.cuda.synchronize()
        ix.close()


def abi_mask_device_then_search(hold):
    """A row mask from device memory set on A, then a masked search with host outputs on B."""
    import torch

    n, d, b, k = 4000, 64, 4, 16
    v, q, dots = dyadic(n, d, b, seed=107)
    m1, m2 = row_mask("half", n, seed=8), row_mask("half", n, seed=9)
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    ix = Raw("float32", d, n)
    try:
        ix.append(v)
        ix.set_mask(tab.VectorBase.pack_row_mask(m1), n)
        bits = cuda(tab.VectorBase.pack_row_mask(m2).view(np.int32))
        ix.search(q, k, 0.0, _capi.TAV_USE_ROW_MASK, stream=sb)
        torch.cuda.synchronize()
        hold(sa)
        ix.set_mask(bits, n, stream=sa)
        window_open(sa)
        got = ix.search(q, k, 0.0, _capi.TAV_USE_ROW_MASK, stream=sb)
        assert_equal_results(got, expected_topk(dots, k, 0.0, m2), "search under the new mask")
    finally:
        torch.cuda.synchronize()
        ix.close()


def abi_read_rows_after_append(hold):
    """A host append queued on A (float32 -> fp16), then tav_read_rows on B."""
    import torch

    n0, n1, d = 2000, 700, 100
    rng = np.random.default_rng(111)
    v = (rng.standard_normal((n0 + n1, d)) * 3).astype(np.float32)
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    ix = raw_with_decoys("float16", v[:n0], v[n0:], lambda ix: ix.read(stream=sb))
    try:
        hold(sa)
        ix.append(v[n0:], stream=sa)
        window_open(sa)
        assert_same_values(ix.read(stream=sb), round_to(v, "float16"), "rows read after the append")
    finally:
        torch.cuda.synchronize()
        ix.close()


def abi_fetch_then_range_search(hold):
    """A fetch of a threshold search's hits into device memory queued on A, then a threshold search with another
    min_score on B (fewer hits: nothing is reallocated)."""
    import torch

    n, d, b = 4000, 64, 3
    v, q, dots = dyadic(n, d, b, seed=108)
    lo, hi = 0.5, 0.6
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    ix = Raw("float32", d, n)
    try:
        ix.append(v)
        ix.range_search(q, hi, stream=sb)
        off_lo = ix.range_search(q, lo, stream=sb)
        total = int(off_lo[-1])
        with torch.cuda.stream(sa):
            items = torch.empty(total, dtype=torch.int64, device="cuda")
            scores = torch.empty(total, dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        hold(sa)
        ix.range_fetch(total, C.c_void_p(items.data_ptr()), C.c_void_p(scores.data_ptr()),
                       _capi.TAV_OUTPUTS_ON_DEVICE, stream=sa)
        window_open(sa)
        off_hi = ix.range_search(q, hi, stream=sb)
        torch.cuda.synchronize()
        assert_same_range((off_lo, items.cpu().numpy(), scores.cpu().numpy()), expected_range(dots, lo),
                          "the fetched hits of the first search")
        n_hi = int(off_hi[-1])
        items_hi, scores_hi = np.empty(n_hi, np.int64), np.empty(n_hi, np.float32)
        ix.range_fetch(n_hi, items_hi.ctypes.data_as(C.c_void_p), scores_hi.ctypes.data_as(C.c_void_p))
        assert_same_range((off_hi, items_hi, scores_hi), expected_range(dots, hi), "the second search")
    finally:
        torch.cuda.synchronize()
        ix.close()


def abi_finish_on_other_stream(hold):
    """Two deferred tensor-core searches queued on A that flag every query, then tav_finish_search on B."""
    import torch

    n, d, b, k = 30000, 64, 5, 9
    rows, q, dots = identical_rows(n, d, 2 * b, seed=109)
    flags = _capi.TAV_DEFER_RETRY | _capi.TAV_FORCE_MMA
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    ix = Raw("bfloat16", d, n)
    try:
        ix.append(rows)
        q1, q2 = cuda(q[:b]), cuda(q[b:])
        with torch.cuda.stream(sa):
            out1, out2 = device_out(b, k), device_out(b, k)
        ix.search_device(q1, k, 0.0, out1, flags, sa)
        assert ix.finish(sa) == b
        torch.cuda.synchronize()
        hold(sa)
        ix.search_device(q1, k, 0.0, out1, flags, sa)
        ix.search_device(q2, k, 0.0, out2, flags, sa)
        window_open(sa)
        redone = ix.finish(sb)
        torch.cuda.synchronize()
        assert_equal_results(host(out1), expected_topk(dots[:b], k, 0.0), "the first deferred search")
        assert_equal_results(host(out2), expected_topk(dots[b:], k, 0.0), "the second deferred search")
        assert redone == 2 * b, "tav_finish_search must redo every query of both searches"
    finally:
        torch.cuda.synchronize()
        ix.close()


SCENARIOS = {
    "py-mask-swap-scan": lambda h: py_mask_swap(h, "scan"),
    "py-mask-swap-mma_defer": lambda h: py_mask_swap(h, "mma_defer"),
    "py-corpus-replaced": py_corpus_replaced,
    "py-defer-then-mask": lambda h: py_defer_then(h, "mask"),
    "py-defer-then-mma_host_lookup": lambda h: py_defer_then(h, "mma_host_lookup"),
    "py-defer-normalize": py_defer_normalize,
    "abi-append-host-then-search": lambda h: abi_append_then_search(h, "host"),
    "abi-append-device-then-search": lambda h: abi_append_then_search(h, "device"),
    "abi-append-then-reserve": abi_append_then_reserve,
    "abi-mask-device-then-search": abi_mask_device_then_search,
    "abi-read-rows-after-append": abi_read_rows_after_append,
    "abi-fetch-then-range-search": abi_fetch_then_range_search,
    "abi-finish-on-other-stream": abi_finish_on_other_stream,
}


@pytest.mark.parametrize("scenario", list(SCENARIOS))
def test_calls_on_other_streams_run_in_call_order(scenario, hold):
    SCENARIOS[scenario](hold)


# ------------------------------------------------------------------ host threads
def run_threads(jobs):
    errors = []

    def run(job):
        try:
            job()
        except BaseException as e:  # re-raised in the main thread
            errors.append(e)

    threads = [threading.Thread(target=run, args=(job,)) for job in jobs]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if errors:
        raise errors[0]


def searches_on_own_stream(base, batches, k, outs):
    """A job: every batch searched with device outputs on a stream of the thread's own, nothing synchronised."""
    import torch

    def job():
        stream = torch.cuda.Stream()
        with torch.cuda.stream(stream):
            for qd, out in zip(batches, outs):
                base.search_device(qd, k, 0.0, out=out)

    return job


def test_two_indexes_two_threads_each_on_its_own_stream():
    """Indexes are independent: two threads, each searching its own index on its own stream."""
    import torch

    n, d, b, k, m = 6000, 64, 16, 10, 6
    jobs, checks = [], []
    for storage, path, seed in (("float32", "scan", 120), ("bfloat16", "mma", 121)):
        v, q, dots = dyadic(n, d, m * b, seed=seed)
        base = vbase(v, storage, path)
        batches = [cuda(q[i * b:(i + 1) * b]) for i in range(m)]
        outs = [device_out(b, k) for _ in range(m)]
        base.search_device(batches[0], k, 0.0, out=outs[0])
        torch.cuda.synchronize()
        jobs.append(searches_on_own_stream(base, batches, k, outs))
        checks.append((storage, dots, outs))
    run_threads(jobs)
    torch.cuda.synchronize()
    for storage, dots, outs in checks:
        for i, out in enumerate(outs):
            assert_equal_results(host(out), expected_topk(dots[i * b:(i + 1) * b], k, 0.0), f"{storage} batch {i}")


def test_one_index_two_threads_each_on_its_own_stream():
    """One index, two threads, each searching on its own stream with device outputs: the library orders the
    searches, which share the index's workspace."""
    import torch

    n, d, b, k, m = 6000, 64, 16, 10, 6
    v, q, dots = dyadic(n, d, 2 * m * b, seed=122)
    base = vbase(v, "float32", "scan")
    batches = [cuda(q[i * b:(i + 1) * b]) for i in range(2 * m)]
    outs = [device_out(b, k) for _ in range(2 * m)]
    base.search_device(batches[0], k, 0.0, out=outs[0])
    torch.cuda.synchronize()
    run_threads([searches_on_own_stream(base, batches[:m], k, outs[:m]),
                 searches_on_own_stream(base, batches[m:], k, outs[m:])])
    torch.cuda.synchronize()
    for i, out in enumerate(outs):
        assert_equal_results(host(out), expected_topk(dots[i * b:(i + 1) * b], k, 0.0), f"batch {i}")
