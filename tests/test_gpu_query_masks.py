"""Per-query row masks (``allowed=`` 2-D, ``TAV_USE_QUERY_MASKS``), bit for bit, without tolerances.

(1) the same mask on every query equals the shared (1-D) mask, on every path and in both tie orders;
(2) dyadic corpora (tests/exact.py) with random masks per query at densities 1 .. 1e-3, one row and none:
    every query equals numpy's exact top-k / threshold set of its own allowed rows;
(3) row b of a masked batch equals a one-query search with ``allowed=mask[b]`` on the same path;
(4) the exact redo, a deferred search finished after later calls, the threshold search's re-pass over
    gathered queries, and a batch of more than one tensor-core slab;
(5) lifecycle (append, remove, overwrite), argument errors and a racing upload on another stream;
(6) deliberately broken builds (``TAV_QUERY_MASK_MUTANT``), each caught by the checks above.
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

import typeagent_py_b200 as tab
from oracle import vectorbase_oracle as O
from tests.exact import dyadic_corpus, expected_topk, preset, scores_of
from typeagent_py_b200 import _capi

pytestmark = pytest.mark.gpu

N, D = 70_000, 64   # large enough for the tensor-core sample pass (N > 16384 and 8 * target < N)
PATHS = ["scan", "scan2", "mma"]
STORAGES = ["float32", "bfloat16", "float16"]
DENSITIES = [1.0, 0.5, 0.01, 1e-3, "one", "none"]


def make_base(v, storage="float32", path=None):
    base = tab.VectorBase(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()), storage_dtype=storage)
    base.add_embeddings(None, v)
    base.force_path = path
    return base


def dyadic(n, d, b, seed):
    amp, exp = preset("fine", d)
    return dyadic_corpus(n, d, b, amp, exp, seed)


def masks_for(b, n, seed, densities=DENSITIES):
    """bool [b, n]: query i gets densities[i % len(densities)] ("one": a single row, "none": empty)."""
    rng = np.random.default_rng(seed)
    m = np.zeros((b, n), bool)
    for i in range(b):
        dens = densities[i % len(densities)]
        if dens == "one":
            m[i, rng.integers(n)] = True
        elif dens != "none":
            m[i] = rng.random(n) < dens
    return m


def expected_masked(dots, k, ms, masks):
    rows = [expected_topk(dots[b:b + 1], k, ms, allowed=masks[b]) for b in range(len(dots))]
    return tuple(np.concatenate([r[j] for r in rows]) for j in range(3))


def expected_range_masked(dots, ms, masks, ties_low=False):
    """CSR (offsets, items, scores) of every allowed row >= ms per query, in the library's order."""
    offs, items, scores = [0], [], []
    for b in range(len(dots)):
        s = scores_of(dots[b])
        with np.errstate(invalid="ignore"):
            ok = (s >= np.float32(ms)) & masks[b]
        rows = np.flatnonzero(ok)
        order = np.lexsort((rows if ties_low else -rows, -s[rows].astype(np.float64)))
        items.append(rows[order])
        scores.append(s[rows][order])
        offs.append(offs[-1] + len(rows))
    return np.array(offs, np.int64), np.concatenate(items).astype(np.int64), np.concatenate(scores).astype(np.float32)


def assert_same(got, want, what):
    for j, (g, w) in enumerate(zip(got, want)):
        g, w = np.asarray(g), np.asarray(w)
        if g.dtype == np.float32:
            g, w = g.view(np.uint32), w.view(np.uint32)
        if g.shape != w.shape or not np.array_equal(g, w):
            bad = np.argwhere(g != w)[:3] if g.shape == w.shape else f"shapes {g.shape} vs {w.shape}"
            raise AssertionError(f"{what}: array {j} differs at {bad}")


def hit_score(dots, k):
    s = scores_of(dots[0])
    return float(np.sort(s[(s > 0) & (s < 1)])[-max(1, k // 2)])


@pytest.fixture(scope="module")
def corpus():
    v, q, dots = dyadic(N, D, 36, seed=11)
    return v, q, dots


# ---------------------------------------------------------------- (1) one mask on every query
@pytest.mark.parametrize("storage", STORAGES)
@pytest.mark.parametrize("path", PATHS)
def test_same_mask_on_every_query_equals_the_shared_mask(corpus, storage, path):
    v, q, _ = corpus
    base = make_base(v, storage, path)
    shared = np.random.default_rng(3).random(N) < 0.3
    tiled = np.tile(shared, (len(q), 1))
    for k in (10, 200):
        assert_same(base.search_arrays(q, k, 0.0, allowed=tiled), base.search_arrays(q, k, 0.0, allowed=shared),
                    f"top-k {path} {storage} k={k}")
    assert_same(base.search_range(q, 0.6, allowed=tiled), base.search_range(q, 0.6, allowed=shared),
                f"range {path} {storage}")
    if path != "mma":  # the lower-row-first tie order is a row-scan order
        assert_same(base.search_arrays(q, 50, 0.0, allowed=tiled, ties_low_first=True),
                    base.search_arrays(q, 50, 0.0, allowed=shared, ties_low_first=True), f"ties low {path} {storage}")
        assert_same(base.search_range(q, 0.6, allowed=tiled, ties_low_first=True),
                    base.search_range(q, 0.6, allowed=shared, ties_low_first=True), f"range ties low {path} {storage}")


# ---------------------------------------------------------------- (2) exact corpora
@pytest.mark.parametrize("storage", STORAGES)
@pytest.mark.parametrize("path", PATHS)
def test_every_query_equals_numpy_over_its_own_rows(corpus, storage, path):
    v, q, dots = corpus
    base = make_base(v, storage, path)
    masks = masks_for(len(q), N, seed=7)
    for k, ms in ((10, 0.0), (200, 0.0), (100, hit_score(dots, 100))):
        assert_same(base.search_arrays(q, k, ms, allowed=masks), expected_masked(dots, k, ms, masks),
                    f"top-k {path} {storage} k={k} ms={ms}")
    for ms in (0.6, hit_score(dots, 40)):
        assert_same(base.search_range(q, ms, allowed=masks), expected_range_masked(dots, ms, masks),
                    f"range {path} {storage} ms={ms}")
    if path != "mma":
        assert_same(base.search_range(q, 0.6, allowed=masks, ties_low_first=True),
                    expected_range_masked(dots, 0.6, masks, ties_low=True), f"range ties low {path} {storage}")


def test_packed_words_and_bools_give_the_same_search(corpus):
    v, q, _ = corpus
    base = make_base(v, "bfloat16")
    masks = masks_for(len(q), N, seed=9)
    assert_same(base.search_arrays(q, 20, 0.0, allowed=base.pack_query_masks(masks)),
                base.search_arrays(q, 20, 0.0, allowed=masks), "packed vs bool")


# ---------------------------------------------------------------- (3) row b == a one-query search
@pytest.mark.parametrize("path", PATHS)
def test_row_of_a_batch_equals_a_one_query_search(path):
    v, q = O.make_corpus(N, D, seed=21, n_queries=24)
    v = v.astype(np.float32)
    base = make_base(v, "bfloat16", path)
    masks = masks_for(len(q), N, seed=4, densities=[0.3, 0.02, 1.0])
    got = base.search_arrays(q, 30, 0.0, allowed=masks)
    for b in range(len(q)):
        one = base.search_arrays(q[b:b + 1], 30, 0.0, allowed=masks[b])
        assert_same(tuple(x[b:b + 1] for x in got), one, f"{path} row {b}")


# ---------------------------------------------------------------- (4) redo, deferred, re-pass, slabs
def identical_rows(n, d, b, seed):
    """n copies of one dyadic row: every score of a query ties, which overflows the tensor-core search's
    candidates and sends every query to the exact redo."""
    v, q, _ = dyadic(1, d, b, seed)
    rows = np.repeat(v, n, axis=0)
    return rows, q, (q.astype(np.float64) @ rows.astype(np.float64).T).astype(np.float32)


def test_exact_redo_uses_each_querys_own_mask():
    import torch

    v, q, dots = identical_rows(N, D, 20, seed=5)
    base = make_base(v, "bfloat16", "mma")
    masks = masks_for(len(q), N, seed=6, densities=[0.5, 0.1, 1.0])
    res = base.search_device(torch.from_numpy(q).cuda(), 40, 0.0, defer_check=True, allowed=masks)
    redone = base.finish_search()
    torch.cuda.synchronize()
    print(f"queries redone exactly: {redone} of {len(q)}")
    assert redone > 0
    assert_same(tuple(t.cpu().numpy() for t in res), expected_masked(dots, 40, 0.0, masks), "redo")


def test_deferred_search_finished_after_later_calls_keeps_its_masks():
    import torch

    v, q, dots = identical_rows(N, D, 20, seed=8)
    base = make_base(v, "bfloat16", "mma")
    m1 = masks_for(len(q), N, seed=1, densities=[0.5, 0.05])
    m2 = masks_for(len(q), N, seed=2, densities=[0.05, 0.5])
    first = base.search_device(torch.from_numpy(q).cuda(), 30, 0.0, defer_check=True, allowed=m1)
    plain = base.search_arrays(q, 30, 0.0)                        # a later call without masks
    second = base.search_arrays(q, 30, 0.0, allowed=m2)          # a later upload of other masks
    base.finish_search()
    torch.cuda.synchronize()
    assert_same(tuple(t.cpu().numpy() for t in first), expected_masked(dots, 30, 0.0, m1), "deferred")
    assert_same(plain, expected_topk(dots, 30, 0.0), "plain")
    assert_same(second, expected_masked(dots, 30, 0.0, m2), "second")


@pytest.mark.parametrize("path", ["scan", "mma"])
def test_range_repass_over_gathered_queries_keeps_their_masks(corpus, path):
    v, q, dots = corpus
    base = make_base(v, "float16", path)
    # even queries allow few rows (no re-pass), odd ones many (re-passed): gathered query i is not query i
    masks = masks_for(len(q), N, seed=12, densities=[1e-3, 0.8])
    base._range_hint = 1   # a tiny capacity hint: the dense queries overflow their regions
    got = base.search_range(q, 0.55, allowed=masks)
    assert_same(got, expected_range_masked(dots, 0.55, masks), f"re-pass {path}")


def test_batch_larger_than_one_tensor_core_slab():
    n, b = 4096, 32768 + 300
    v, q, _ = dyadic(n, D, b, seed=13)
    base = make_base(v, "bfloat16", "mma")
    masks = np.random.default_rng(14).random((b, n)) < 0.5
    got = base.search_arrays(q, 5, 0.0, allowed=masks)
    picks = list(range(40)) + list(range(32760, b))
    dots = (q[picks].astype(np.float64) @ v.astype(np.float64).T).astype(np.float32)
    want = expected_masked(dots, 5, 0.0, masks[picks])
    assert_same(tuple(x[picks] for x in got), want, "slabs")


# ---------------------------------------------------------------- (5) lifecycle and errors
def set_masks_abi(base, masks):
    lib, ix = base._ensure_device()
    words = base.pack_query_masks(masks)
    _capi.check(lib.tav_set_query_masks(ix, words.ctypes.data_as(C.c_void_p), len(words), masks.shape[1],
                                        words.shape[1], 0, None))
    base._qmask_key = None  # the Python cache does not know about this upload


def search_abi(base, q, k, flags):
    lib, ix = base._ensure_device()
    q = np.ascontiguousarray(q, np.float32)
    items = np.empty((len(q), k), np.int64)
    scores = np.empty((len(q), k), np.float32)
    counts = np.empty(len(q), np.int32)
    rc = lib.tav_search(ix, q.ctypes.data_as(C.c_void_p), len(q), k, C.c_float(0.0), flags, None, 0, 0,
                        items.ctypes.data_as(C.c_void_p), scores.ctypes.data_as(C.c_void_p),
                        counts.ctypes.data_as(C.c_void_p), None)
    return rc, (items, scores, counts)


def test_lifecycle_append_remove_overwrite():
    v, q, dots = dyadic(5000, D, 6, seed=15)
    base = make_base(v[:4000], "float32", "scan")
    masks = masks_for(len(q), 4000, seed=16, densities=[0.5, 0.1])
    set_masks_abi(base, masks)
    assert search_abi(base, q, 10, _capi.TAV_USE_QUERY_MASKS)[0] == 0
    base.add_embeddings(None, v[4000:])                              # an append invalidates the masks
    base._ensure_device()
    assert search_abi(base, q, 10, _capi.TAV_USE_QUERY_MASKS)[0] == _capi.TAV_ERR_STATE
    masks = masks_for(len(q), 5000, seed=17, densities=[0.5, 0.1])
    set_masks_abi(base, masks)
    base.set_embeddings_at(10, v[20:30])                             # an overwrite keeps them
    new_v = v.copy()
    new_v[10:20] = v[20:30]
    new_dots = (q.astype(np.float64) @ new_v.astype(np.float64).T).astype(np.float32)
    rc, got = search_abi(base, q, 10, _capi.TAV_USE_QUERY_MASKS)
    assert rc == 0
    assert_same(got, expected_masked(new_dots, 10, 0.0, masks), "after overwrite")
    base.remove_embeddings([3])                                      # a removal drops them
    base._ensure_device()
    assert search_abi(base, q, 10, _capi.TAV_USE_QUERY_MASKS)[0] == _capi.TAV_ERR_STATE
    # through the Python forms: a mask of the new size is uploaded and used
    masks = masks_for(len(q), 4999, seed=18, densities=[0.5, 0.1])
    dots = np.delete(new_dots, 3, axis=1)
    assert_same(base.search_arrays(q, 10, 0.0, allowed=masks), expected_masked(dots, 10, 0.0, masks), "after removal")


def test_argument_errors():
    v, q, _ = dyadic(3000, D, 4, seed=19)
    base = make_base(v, "bfloat16")
    masks = masks_for(4, 3000, seed=20, densities=[0.5])
    with pytest.raises(ValueError, match="rows for 4 queries"):
        base.search_arrays(q, 5, 0.0, allowed=masks[:3])
    with pytest.raises(ValueError, match="entries for 3000 rows"):
        base.search_arrays(q, 5, 0.0, allowed=masks[:, :2999])
    with pytest.raises(ValueError, match="bits for 3000 rows"):
        base.search_arrays(q, 5, 0.0, allowed=base.pack_query_masks(masks)[:, :-1])
    with pytest.raises(ValueError, match="cannot be combined"):
        base.search_arrays(q, 5, 0.0, allowed=masks, subset=[1, 2, 3])
    set_masks_abi(base, masks)
    assert search_abi(base, q[:3], 5, _capi.TAV_USE_QUERY_MASKS)[0] == _capi.TAV_ERR_INVALID        # count
    assert search_abi(base, q, 5, _capi.TAV_USE_QUERY_MASKS | _capi.TAV_USE_ROW_MASK)[0] == _capi.TAV_ERR_INVALID
    lib, ix = base._ensure_device()
    sub = np.arange(10, dtype=np.int64)
    out = (np.empty((4, 5), np.int64), np.empty((4, 5), np.float32), np.empty(4, np.int32))
    qq = np.ascontiguousarray(q, np.float32)
    assert lib.tav_search(ix, qq.ctypes.data_as(C.c_void_p), 4, 5, C.c_float(0.0), _capi.TAV_USE_QUERY_MASKS,
                          sub.ctypes.data_as(C.c_void_p), len(sub), 0, *(a.ctypes.data_as(C.c_void_p) for a in out),
                          None) == _capi.TAV_ERR_INVALID                                            # with a subset
    offsets = np.empty(5, np.int64)
    assert lib.tav_range_search(ix, qq.ctypes.data_as(C.c_void_p), 4, C.c_float(0.5), _capi.TAV_USE_QUERY_MASKS,
                                sub.ctypes.data_as(C.c_void_p), len(sub), 0, 0, offsets.ctypes.data_as(C.c_void_p),
                                None) == _capi.TAV_ERR_INVALID
    lib, ix = base._ensure_device()
    assert lib.tav_set_query_masks(ix, None, 0, 0, 0, 0, None) == 0                                     # clears
    assert search_abi(base, q, 5, _capi.TAV_USE_QUERY_MASKS)[0] == _capi.TAV_ERR_STATE


def test_single_upload_per_mask_object(corpus):
    v, q, _ = corpus
    base = make_base(v, "bfloat16")
    masks = masks_for(len(q), N, seed=22)
    lib, _ = base._ensure_device()
    calls = []
    real = lib.tav_set_query_masks

    class Counting:
        def __getattr__(self, name):
            return getattr(lib, name)

        def tav_set_query_masks(self, *a):
            calls.append(1)
            return real(*a)

    base._ensure_device = lambda: (Counting(), base._ix)
    for _ in range(3):
        base.search_arrays(q, 10, 0.0, allowed=masks)
    base.search_range(q, 0.6, allowed=masks)
    assert len(calls) == 1


def test_racing_mask_upload_on_another_stream_waits_for_the_search():
    """A search queued behind a ~200 ms hold on stream A, then a mask upload on stream B: the search must see
    the masks it was issued with."""
    import torch

    v, q, dots = dyadic(20_000, D, 32, seed=23)
    base = make_base(v, "bfloat16", "mma")
    m1 = masks_for(len(q), 20_000, seed=24, densities=[0.5, 0.02])
    m2 = masks_for(len(q), 20_000, seed=25, densities=[0.02, 0.5])
    qd = torch.from_numpy(q).cuda()
    base.search_device(qd, 10, 0.0, allowed=m1)  # warm-up
    torch.cuda.synchronize()
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda._sleep(1000)
    start.record()
    torch.cuda._sleep(20_000_000)
    end.record()
    end.synchronize()
    cycles = int(20_000_000 * 200.0 / start.elapsed_time(end))
    # everything allocated before the hold: an allocation inside the window may synchronise the device
    words = torch.from_numpy(base.pack_query_masks(m2).view(np.int32)).cuda()
    outs = [(torch.empty((len(q), 10), dtype=torch.int64, device="cuda"),
             torch.empty((len(q), 10), dtype=torch.float32, device="cuda"),
             torch.empty(len(q), dtype=torch.int32, device="cuda")) for _ in range(2)]
    torch.cuda.synchronize()
    with torch.cuda.stream(a):
        torch.cuda._sleep(cycles)
        res = base.search_device(qd, 10, 0.0, allowed=m1, defer_check=True, out=outs[0])
    with torch.cuda.stream(b):
        assert not a.query(), "hold too short"
        base.search_device(qd, 10, 0.0, allowed=words, defer_check=True, out=outs[1])
    base.finish_search()
    torch.cuda.synchronize()
    assert_same(tuple(t.cpu().numpy() for t in res), expected_masked(dots, 10, 0.0, m1), "held search")
    assert_same(tuple(t.cpu().numpy() for t in outs[1]), expected_masked(dots, 10, 0.0, m2), "racing search")


# ---------------------------------------------------------------- (6) broken builds
MUTANTS = {1: "MAIN epilogue reads the other query's mask", 2: "exact redo uses mask 0",
           3: "range re-pass drops the mask map"}


@pytest.fixture(scope="module")
def mutant_libs():
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc) and not shutil.which(nvcc):
        pytest.skip("nvcc is needed to build the broken variants")
    from typeagent_py_b200 import build as B

    tmp = tempfile.mkdtemp(prefix="tav_qmask_mutants_")
    procs = {}
    for m in MUTANTS:
        out = os.path.join(tmp, f"libtavec_mutant{m}.so")
        cmd = [nvcc, *[f for f in B.NVCC_FLAGS if f != "-Xptxas=-v"], f"-DTAV_QUERY_MASK_MUTANT={m}", "-o", out,
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


def mutant_checks(corpus):
    caught = []
    checks = [
        lambda: test_every_query_equals_numpy_over_its_own_rows(corpus, "bfloat16", "mma"),
        test_exact_redo_uses_each_querys_own_mask,
        lambda: test_range_repass_over_gathered_queries_keeps_their_masks(corpus, "scan"),
        lambda: test_range_repass_over_gathered_queries_keeps_their_masks(corpus, "mma"),
    ]
    for check in checks:
        try:
            check()
        except AssertionError as e:
            caught.append(str(e)[:200])
    return caught


@pytest.mark.parametrize("m", sorted(MUTANTS), ids=[MUTANTS[m].replace(" ", "_") for m in sorted(MUTANTS)])
def test_broken_build_is_caught(mutant_libs, corpus, m):
    with library(mutant_libs[m]):
        caught = mutant_checks(corpus)
    assert caught, f"the exact checks did not catch: {MUTANTS[m]}"


def test_checks_pass_on_the_real_build(corpus):
    assert mutant_checks(corpus) == []
