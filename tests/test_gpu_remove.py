"""Removing and overwriting rows on the device (``tav_remove_rows`` / ``tav_write_rows``).

The oracle: after any sequence of appends, removals and overwrites, every result must equal, bit for bit, what
a fresh index built from the surviving rows returns — the rows read back, ``serialize()``, and every search
path: the single-launch row scan, the two-kernel scan, the tensor cores on bf16 / fp16, the float32 split form,
the threshold search, subsets, masks set after the removal, ties-low, and deferred searches finished
afterwards.  The corpora are dyadic (tests/exact.py), so every search must also equal the exact top-k.

Removal patterns: none, the first, the last, all rows, every other row, one long run, a long run that begins
inside a warp's destinations, random 1%, 50% and 99%, on row counts that are not tile multiples; each through the out-of-place compaction and through the in-place
one with a window buffer of a few rows (many windows).  Then: searches racing on other streams, invalid calls
that must leave the index bit-identical, the fp16-range flag of the split form after the offending row is
removed or overwritten, row widths that are not a multiple of 16 bytes, and one rank of ``ShardedVectorBase``.
"""

from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import typeagent_py_b200 as tab
from oracle import vectorbase_oracle as O
from tests.exact import dyadic_corpus, expected_topk, preset
from tests.test_gpu_exact import assert_equal_results, row_mask
from tests.test_gpu_range import assert_same_range
from tests.test_gpu_streams import Raw, cuda, device_out, exact_dots, hold, hold_cycles, host, window_open  # noqa: F401
from typeagent_py_b200 import _capi

pytestmark = pytest.mark.gpu

OUT_OF_PLACE, IN_PLACE = 1, 2


def internal(name, argtypes):
    fn = getattr(_capi.load(), name)
    fn.argtypes, fn.restype = argtypes, C.c_int
    return fn


def set_policy(h, mode, scratch_bytes=0):
    _capi.check(internal("tav_internal_compact_policy", [C.c_void_p, C.c_int, C.c_int64])(h, mode, scratch_bytes))


def last_compaction(h):
    path, windows = C.c_int(0), C.c_int64(0)
    _capi.check(internal("tav_internal_compact_stats", [C.c_void_p, C.c_void_p, C.c_void_p])(
        h, C.byref(path), C.byref(windows)))
    return path.value, windows.value


def read_rows(h, d):
    lib = _capi.load()
    out = np.empty((lib.tav_size(h), d), np.float32)
    _capi.check(lib.tav_read_rows(h, 0, len(out), out.ctypes.data_as(C.c_void_p), None))
    return out


def settings():
    return tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel())


def vbase(rows, storage):
    base = tab.VectorBase(settings(), storage_dtype=storage)
    base.add_embeddings(None, rows)
    base.search_arrays(rows[:1], 1)  # the device copy exists
    return base


def dyadic(n, d, b, seed):
    amp, exp = preset("fine", d)
    return dyadic_corpus(n, d, b, amp, exp, seed)


def removal(pattern, n, seed):
    rng = np.random.default_rng(seed)
    pick = lambda frac: rng.choice(n, max(1, int(round(frac * n))), replace=False)  # noqa: E731
    return {
        "none": np.zeros(0, np.int64),
        "first": np.array([0]),
        "last": np.array([-1]),
        "all": np.arange(n),
        "every-other": np.arange(1, n, 2),
        "run": np.arange(n // 5, n // 5 + 1237),
        "random-1%": pick(0.01),
        "random-50%": pick(0.5),
        "random-99%": pick(0.99),
        "repeated-negative": np.array([-3, 17, 17, -3, 2 * n // 3]),
        # a short run, then a long one that begins inside a warp's 16 destinations: equal keys to gallop over
        "runs-mid-warp": np.concatenate([np.arange(10, 20), np.arange(1003, 4000)]),
    }[pattern]


PATHS = ("scan1", "scan2", "scan", "mma", "range", "range-mma", "subset", "mask", "ties-low", "defer")


def results(base, path, q, k):
    """One search form on `base` -> comparable numpy arrays."""
    import torch

    n = len(base)
    if path == "scan1":  # one host query per call: the single-launch form
        base.force_path = None
        out = [base.search_arrays(q[i:i + 1], k, 0.0) for i in range(4)]
        return tuple(np.concatenate([o[j] for o in out]) for j in range(3))
    base.force_path = {"scan2": "scan2", "scan": "scan", "mma": "mma", "range-mma": "mma", "defer": "mma"}.get(path)
    try:
        if path in ("range", "range-mma"):
            return base.search_range(q, 0.55)
        if path == "subset":
            sub = np.random.default_rng(1).choice(n, min(n, 700), replace=True)
            return base.search_arrays(q, k, 0.0, subset=sub)
        if path == "mask":
            return base.search_arrays(q, k, 0.0, allowed=row_mask("half", n, seed=4))
        if path == "ties-low":
            return base.search_arrays(q, k, 0.0, ties_low_first=True)
        if path == "defer":
            res = base.search_device(torch.from_numpy(q).cuda(), k, 0.0, defer_check=True)
            base.finish_search()
            torch.cuda.synchronize()
            return tuple(t.cpu().numpy() for t in res)
        return base.search_arrays(q, k, 0.0)
    finally:
        base.force_path = None


def assert_same_as_fresh(base, rows, q, storage, what, k=12):
    """`base` holds `rows` (float32 host values): equal to a fresh index of them, bit for bit, on every path."""
    d = rows.shape[1]
    np.testing.assert_array_equal(base.serialize(), rows, err_msg=f"{what}: serialize()")
    fresh = vbase(rows, storage) if len(rows) else tab.VectorBase(settings(), storage_dtype=storage)
    if len(rows) == 0:
        assert len(base) == 0 and base.fuzzy_lookup_embedding(q[0]) == []
        return
    base.search_arrays(q[:1], 1)  # sync the device copy (appends after a removal)
    got_rows, want_rows = read_rows(base._ix, d), read_rows(fresh._ix, d)
    np.testing.assert_array_equal(got_rows.view(np.uint32), want_rows.view(np.uint32), err_msg=f"{what}: rows")
    dots = exact_dots(q, rows)
    kk = min(k, len(rows))
    for path in PATHS:
        if path in ("mma", "range-mma", "defer") and len(rows) < 8:
            continue
        got, want = results(base, path, q, kk), results(fresh, path, q, kk)
        if path.startswith("range"):
            assert_same_range(got, want, f"{what}: {path}")
            continue
        assert_equal_results(got, want, f"{what}: {path} against a fresh index")
        if path in ("scan1",):
            assert_equal_results(got, expected_topk(dots[:4], kk, 0.0), f"{what}: {path} against the exact top-k")
        elif path in ("scan2", "scan", "mma", "defer"):
            assert_equal_results(got, expected_topk(dots, kk, 0.0), f"{what}: {path} against the exact top-k")


PATTERNS = ("none", "first", "last", "all", "every-other", "run", "random-1%", "random-50%", "random-99%",
            "repeated-negative", "runs-mid-warp")


@pytest.mark.parametrize("mode", ["out-of-place", "in-place"])
@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("storage", ["float32", "bfloat16", "float16"])
def test_every_search_equals_a_fresh_index_after_removal(storage, pattern, mode):
    n, d, b = 4999, 64, 20  # not a multiple of any tile
    v, q, _ = dyadic(n, d, b, seed=7)
    base = vbase(v, storage)
    window = 37  # rows per in-place window: many windows
    set_policy(base._ix, OUT_OF_PLACE if mode == "out-of-place" else IN_PLACE,
               window * d * (4 if storage == "float32" else 2))
    gone = removal(pattern, n, seed=3)
    gen = base._generation
    base.remove_embeddings(gone)
    rows = np.delete(v, gone, axis=0)
    assert base._generation == gen and len(base) == len(rows)
    path, windows = last_compaction(base._ix)
    first = int(np.min(np.where(gone < 0, gone + n, gone))) if len(gone) else n
    moving = len(rows) - first
    if moving > 0:
        assert path == (1 if mode == "out-of-place" else 2), "the compaction took the other path"
        if mode == "in-place":
            assert windows == -(-moving // window)
    assert_same_as_fresh(base, rows, q, storage, f"{storage} {pattern} {mode}")


@pytest.mark.parametrize("storage", ["float32", "bfloat16"])
def test_a_sequence_of_appends_removals_and_overwrites(storage):
    n, d, b = 3001, 64, 16
    v, q, _ = dyadic(n + 900, d, b, seed=8)
    w = dyadic(600, d, 1, seed=9)[0]
    base = vbase(v[:n], storage)
    rows = v[:n].copy()
    rng = np.random.default_rng(10)
    for step in range(4):
        gone = rng.choice(len(rows), 97 * (step + 1), replace=False)
        base.remove_embeddings(gone)
        rows = np.delete(rows, gone, axis=0)
        first = int(rng.integers(0, len(rows) - 150))
        new = w[150 * step: 150 * step + 150]
        base.set_embeddings_at(first, new)
        rows[first:first + 150] = new
        extra = v[n + 225 * step: n + 225 * (step + 1)]
        base.add_embeddings(None, extra)
        rows = np.concatenate([rows, extra])
        base.set_embedding_at(len(rows) - 1, w[-1 - step])  # a row appended on the host only so far
        rows[-1] = w[-1 - step]
        assert_same_as_fresh(base, rows, q, storage, f"{storage} step {step}")


def test_remove_back_to_the_old_size_then_masked_search():
    n, d, b, k = 5000, 64, 8, 10
    v, q, _ = dyadic(n + 1, d, b, seed=11)
    base = vbase(v[:n], "bfloat16")
    allowed = row_mask("half", n, seed=5)
    base.search_arrays(q, k, 0.0, allowed=allowed)
    base.remove_embeddings([0])
    base.add_embeddings(None, v[n:])
    rows = np.concatenate([v[1:n], v[n:]])
    for path in ("scan", "mma"):
        base.force_path = path
        got = base.search_arrays(q, k, 0.0, allowed=allowed)
        assert_equal_results(got, expected_topk(exact_dots(q, rows), k, 0.0, allowed), f"masked {path}")


@pytest.mark.parametrize("d", [1, 3, 5, 13, 100])
@pytest.mark.parametrize("storage", ["float32", "bfloat16", "float16"])
def test_row_widths_the_vector_loads_cannot_take_whole(storage, d):
    """Widths whose rows are not a multiple of 16 bytes: the compaction falls back to narrower vectors."""
    n = 2003
    v, q, _ = dyadic(n, d, 8, seed=12)
    for mode in (OUT_OF_PLACE, IN_PLACE):
        base = vbase(v, storage)
        set_policy(base._ix, mode, 29 * d * 4)
        gone = removal("random-50%", n, seed=13)
        base.remove_embeddings(gone)
        rows = np.delete(v, gone, axis=0)
        fresh = vbase(rows, storage)
        np.testing.assert_array_equal(read_rows(base._ix, d).view(np.uint32), read_rows(fresh._ix, d).view(np.uint32))
        base.force_path = "scan"
        assert_equal_results(base.search_arrays(q, 9, 0.0), expected_topk(exact_dots(q, rows), 9, 0.0),
                             f"{storage} d={d} mode {mode}")


def test_the_default_compaction_is_in_place():
    n, d = 6000, 64
    v = dyadic(n, d, 1, seed=14)[0]
    base = vbase(v, "bfloat16")
    base.remove_embeddings([10])  # nearly every row moves, in one window
    assert last_compaction(base._ix) == (2, 1)
    base.remove_embeddings([len(base) - 100])  # 99 rows move
    assert last_compaction(base._ix) == (2, 1)
    base.remove_embeddings([-1])  # nothing moves
    assert last_compaction(base._ix)[0] == 0
    np.testing.assert_array_equal(base.serialize(), np.delete(v, [10, n - 100, n - 1], axis=0))


@pytest.mark.parametrize("change", ["remove", "overwrite"])
def test_split_form_flag_follows_the_offending_row(change):
    """A float32 value beyond the fp16 range sends every split-form search to the exact redo; once that row is
    removed or overwritten, the planes are rebuilt and the flag cleared."""
    import torch

    n, d, b, k = 5000, 64, 16, 8
    v, q, _ = dyadic(n, d, b, seed=15)
    big = v.copy()
    big[1234, 5] = 1e6
    base = vbase(big, "float32")
    base.force_path = "mma"
    qd = torch.from_numpy(q).cuda()
    base.search_device(qd, k, 0.0, defer_check=True)
    assert base.finish_search() == b, "the row beyond the fp16 range must send every query to the redo"
    if change == "remove":
        base.remove_embeddings([1234])
        rows = np.delete(v, 1234, axis=0)
    else:
        base.set_embedding_at(1234, v[1234])
        rows = v
    res = base.search_device(qd, k, 0.0, defer_check=True)
    assert base.finish_search() < b, "the flag must be recomputed once the row is gone"
    torch.cuda.synchronize()
    assert_equal_results(host(res), expected_topk(exact_dots(q, rows), k, 0.0), f"split form after {change}")


def test_deferred_search_before_a_removal_sees_the_old_rows():
    """A deferred search that flags every query, then a removal: the removal finishes it first, on the old rows."""
    import torch

    n, d, b, k = 30000, 64, 5, 9
    one, q, _ = dyadic(1, d, b, seed=16)
    rows = np.repeat(one, n, axis=0)
    base = vbase(rows, "bfloat16")
    base.force_path = "mma"
    qd = torch.from_numpy(q).cuda()
    res = base.search_device(qd, k, 0.0, defer_check=True)
    base.remove_embeddings(np.arange(n - 40, n))  # the top rows of every query go
    torch.cuda.synchronize()
    want = expected_topk(exact_dots(q, rows), k, 0.0)
    assert_equal_results(host(res), want, "the deferred search issued before the removal")
    assert base.finish_search() == 0
    res = base.search_device(qd, k, 0.0, defer_check=True)
    base.finish_search()
    torch.cuda.synchronize()
    assert_equal_results(host(res), expected_topk(exact_dots(q, rows[:-40]), k, 0.0), "a deferred search after")


# ------------------------------------------------------------------ streams
def raw_index(storage, v):
    ix = Raw(storage, v.shape[1], 2 * len(v))
    ix.append(v)
    return ix


def remove(ix, ordinals, stream=None):
    o = np.ascontiguousarray(ordinals, np.int64)
    return ix.lib.tav_remove_rows(ix.h, o.ctypes.data_as(C.c_void_p), len(o),
                                  None if stream is None else C.c_void_p(stream.cuda_stream))


def write(ix, first, rows, stream=None):
    if isinstance(rows, np.ndarray):
        rows = np.ascontiguousarray(rows, np.float32)
        ptr, n, on_device = rows.ctypes.data_as(C.c_void_p), len(rows), 0
    else:
        ptr, n, on_device = C.c_void_p(rows.data_ptr()), rows.shape[0], 1
    return ix.lib.tav_write_rows(ix.h, first, ptr, n, ix.d, _capi.TAV_F32, on_device,
                                 None if stream is None else C.c_void_p(stream.cuda_stream))


@pytest.mark.parametrize("scenario", ["search-then-remove", "search-then-overwrite", "overwrite-then-search",
                                      "remove-then-search"])
@pytest.mark.parametrize("storage", ["float32", "bfloat16"])
def test_changes_racing_on_other_streams_keep_call_order(scenario, storage, hold):
    import torch

    n, d, b, k = 6000, 64, 8, 12
    v, q, _ = dyadic(n, d, b, seed=17)
    w = dyadic(300, d, 1, seed=18)[0]
    gone = removal("random-50%", n, seed=19)
    after = np.delete(v, gone, axis=0) if "remove" in scenario else np.concatenate([v[:100], w, v[400:]])
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    ix = raw_index(storage, v)
    qd, wd = cuda(q), cuda(w)
    try:
        out = device_out(b, k)
        ix.search(q, k, 0.0, stream=sb)
        torch.cuda.synchronize()
        change = (lambda s: remove(ix, gone, s)) if "remove" in scenario else (lambda s: write(ix, 100, wd, s))
        if scenario.startswith("search"):
            hold(sa)
            ix.search_device(qd, k, 0.0, out, _capi.TAV_FORCE_SCAN, sa)
            window_open(sa)
            _capi.check(change(sb))
            got_after = ix.search(q, k, 0.0, stream=sb)
            torch.cuda.synchronize()
            assert_equal_results(host(out), expected_topk(exact_dots(q, v), k, 0.0), "the search queued before")
        else:
            hold(sa)
            if scenario == "overwrite-then-search":
                _capi.check(change(sa))
                window_open(sa)
            else:
                _capi.check(change(sa))  # a removal that moves rows waits for its stream
            got_after = ix.search(q, k, 0.0, stream=sb)
        assert_equal_results(got_after, expected_topk(exact_dots(q, after), k, 0.0), "the search made after")
        np.testing.assert_array_equal(ix.read(), after)  # dyadic values are exact in bf16 too
    finally:
        torch.cuda.synchronize()
        ix.close()


# ------------------------------------------------------------------ invalid calls
def test_invalid_calls_leave_the_index_bit_identical():
    import torch

    n, d = 3000, 64
    v = dyadic(n, d, 1, seed=20)[0]
    ix = raw_index("bfloat16", v)
    try:
        before = ix.read()
        for bad in ([n], [-n - 1], [0, 5, n + 7]):
            assert remove(ix, bad) == _capi.TAV_ERR_RANGE
        assert write(ix, n - 1, v[:2]) == _capi.TAV_ERR_RANGE
        assert write(ix, -1, v[:1]) == _capi.TAV_ERR_RANGE
        assert ix.lib.tav_write_rows(ix.h, 0, v.ctypes.data_as(C.c_void_p), 1, d + 1, _capi.TAV_F32, 0,
                                     None) == _capi.TAV_ERR_INVALID
        assert ix.lib.tav_size(ix.h) == n
        np.testing.assert_array_equal(ix.read().view(np.uint32), before.view(np.uint32))
    finally:
        ix.close()
    # adopted memory
    t = torch.from_numpy(v).cuda().to(torch.bfloat16)
    base = tab.VectorBase.from_device_tensor(settings(), t)
    snapshot = t.clone()
    o = np.array([0], np.int64)
    lib = _capi.load()
    assert lib.tav_remove_rows(base._ix, o.ctypes.data_as(C.c_void_p), 1, None) == _capi.TAV_ERR_STATE
    assert lib.tav_write_rows(base._ix, 0, v.ctypes.data_as(C.c_void_p), 1, d, _capi.TAV_F32, 0,
                              None) == _capi.TAV_ERR_STATE
    with pytest.raises(RuntimeError):
        base.remove_embeddings([0])
    with pytest.raises(RuntimeError):
        base.set_embeddings_at(0, v[:1])
    torch.cuda.synchronize()
    assert torch.equal(t.view(torch.int16), snapshot.view(torch.int16)) and len(base) == n
    # the Python class: errors before anything changes
    base = vbase(v, "float32")
    with pytest.raises(IndexError):
        base.remove_embeddings([1, n])
    np.testing.assert_array_equal(read_rows(base._ix, d), v)


# ------------------------------------------------------------------ sharding
def test_sharded_one_rank_equals_vectorbase_after_removals():
    import socket

    import torch.distributed as dist

    from typeagent_py_b200.sharded import ShardedVectorBase

    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    dist.init_process_group("gloo", rank=0, world_size=1, init_method=f"tcp://127.0.0.1:{port}")
    try:
        n = 10000
        v, q, _ = dyadic(n, 64, 20, seed=21)
        for storage in ("float32", "bfloat16"):
            one = tab.VectorBase(settings(), storage_dtype=storage)
            one.add_embeddings(None, v)
            sh = ShardedVectorBase(settings(), device=0, storage_dtype=storage)
            sh.deserialize(v)
            for gone in (removal("random-1%", n, 22), removal("run", n - 100, 0), [-1, 0, 5]):
                one.remove_embeddings(gone)
                sh.remove_embeddings(gone)
                assert len(sh) == len(one)
                for k in (10, 300):
                    gi, gs, gc = sh.search_arrays(q, k, 0.0)
                    wi, ws, wc = one.search_arrays(q, k, 0.0)
                    np.testing.assert_array_equal(gc, wc)
                    np.testing.assert_array_equal(gi, wi)
                    np.testing.assert_array_equal(gs.view(np.uint32), ws.view(np.uint32))
                assert_same_range(sh.search_range(q, 0.6), one.search_range(q, 0.6), f"{storage} range")
    finally:
        dist.destroy_process_group()


def test_sharded_deferred_lookup_before_a_removal_equals_the_old_rows():
    """A deferred sharded lookup that flags every query (identical rows), then remove_embeddings and finish():
    the lookup's result is the top-k of the rows it was issued on."""
    import socket

    import torch
    import torch.distributed as dist

    from typeagent_py_b200.sharded import ShardedVectorBase

    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    dist.init_process_group("gloo", rank=0, world_size=1, init_method=f"tcp://127.0.0.1:{port}")
    try:
        n, d, b, k = 30000, 64, 5, 9
        one, q, _ = dyadic(1, d, b, seed=23)
        rows = np.repeat(one, n, axis=0)
        sh = ShardedVectorBase(settings(), device=0, storage_dtype="bfloat16")
        sh.deserialize(rows)
        sh._engine.base.force_path = "mma"
        out = sh.search_tensors(q, k, 0.0, defer_check=True)
        sh.remove_embeddings(np.arange(n - 40, n))  # the top rows of every query go
        sh.finish()
        torch.cuda.synchronize()
        assert_equal_results(host(out), expected_topk(exact_dots(q, rows), k, 0.0), "the deferred lookup")
        after = sh.search_tensors(q, k, 0.0)
        assert_equal_results(host(after), expected_topk(exact_dots(q, rows[:-40]), k, 0.0), "a lookup after")
    finally:
        dist.destroy_process_group()
