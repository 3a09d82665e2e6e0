"""Per-query subsets (``subsets=``, ``tav_search_subsets`` / ``tav_range_search_subsets``), bit for bit.

(1) row b of a batch equals the one-query search with ``subset=subsets[b]`` (items, float32 score bits, counts,
    order): float32 / bf16 / fp16 storage, widths 64, 768 and an odd one, subsets of 0 .. 100k entries with
    duplicates, negatives and one row repeated 10k times, k from 1 to beyond the longest subset, min_score at a
    hit's score and one ulp either side, NaN, both tie orders;
(2) dyadic corpora (tests/exact.py): every query equals numpy's exact top-k / threshold set over its subset, and
    ``fuzzy_lookup_embeddings_in_subsets`` equals the oracle's ``fuzzy_lookup_embedding_in_subset`` per query;
(3) a skewed batch: one query with 1M entries and 255 with 10;
(4) the C ABI: flat positions, flags, offsets and ordinals that are refused, and an index left as it was;
(5) a normalising index; (6) appends, removals and overwrites; (7) call order across streams;
(8) deliberately broken builds (``TAV_SUBSETS_MUTANT``), each caught by the checks above.
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
from tests.exact import dyadic_corpus, preset, scores_of
from typeagent_py_b200 import _capi

pytestmark = pytest.mark.gpu

STORAGES = ["float32", "bfloat16", "float16"]
WIDTHS = [64, 768, 67]  # 67: rows that are not a multiple of 16 bytes take the scalar loop
N = 120_000


def make_base(v, storage="float32", normalize=False):
    base = tab.VectorBase(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()), storage_dtype=storage,
                          normalize=normalize)
    base.add_embeddings(None, v)
    return base


def unit_corpus(n, d, b, seed):
    rng = np.random.default_rng(seed)
    v = rng.standard_normal((n, d), dtype=np.float32)
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    q = v[rng.integers(n, size=b)] + np.float32(0.3) * rng.standard_normal((b, d), dtype=np.float32)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    return v, np.ascontiguousarray(q, np.float32)


def mixed_subsets(n, seed):
    """Eight subsets: lengths 0, 1, 7, 4096, 4097 and 100k, one row repeated 10k times, and a short mix; with
    duplicates and negative ordinals."""
    rng = np.random.default_rng(seed)

    def some(m, neg=0.3):
        s = rng.integers(n, size=m)
        flip = rng.random(m) < neg
        s[flip] -= n
        return s

    tied = np.concatenate([np.full(10_000, rng.integers(n)), some(50)])
    rng.shuffle(tied)
    return [np.empty(0, np.int64), some(1), np.array([5, 5, -1, n - 1, 0, -n, 5]), some(4096), some(4097),
            some(100_000), tied, some(257).tolist()]


def assert_bits(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    if got.dtype == np.float32:
        got, want = got.view(np.uint32), want.view(np.uint32)
    if got.shape != want.shape or not np.array_equal(got, want):
        bad = np.argwhere(got != want)[:3] if got.shape == want.shape else f"shapes {got.shape} vs {want.shape}"
        raise AssertionError(f"{what}: differs at {bad}")


def assert_rows_equal_loop(base, q, subsets, k, ms, ties_low, what=""):
    items, scores, counts = base.search_arrays(q, k, ms, subsets=subsets, ties_low_first=ties_low)
    longest = max(len(s) for s in subsets)
    assert items.shape == (len(q), max(1, min(k, longest)))
    for b in range(len(q)):
        i1, s1, c1 = base.search_arrays(q[b:b + 1], k, ms, subset=np.asarray(subsets[b], np.int64),
                                        ties_low_first=ties_low)
        kb = i1.shape[1]
        tag = f"{what} k={k} ms={ms!r} ties_low={ties_low} query {b}"
        assert counts[b] == c1[0], f"{tag}: count {counts[b]} != {c1[0]}"
        assert_bits(items[b, :kb], i1[0], tag + " items")
        assert_bits(scores[b, :kb], s1[0], tag + " scores")
        assert (items[b, kb:] == -1).all() and (scores[b, kb:] == 0).all(), tag + " padding"


def assert_range_equal_loop(base, q, subsets, ms, ties_low, what=""):
    offs, items, scores = base.search_range(q, ms, subsets=subsets, ties_low_first=ties_low)
    for b in range(len(q)):
        o1, i1, s1 = base.search_range(q[b:b + 1], ms, subset=np.asarray(subsets[b], np.int64), ties_low_first=ties_low)
        tag = f"{what} range ms={ms!r} ties_low={ties_low} query {b}"
        assert offs[b + 1] - offs[b] == o1[1], f"{tag}: {offs[b + 1] - offs[b]} hits != {o1[1]}"
        assert_bits(items[offs[b]:offs[b + 1]], i1, tag + " items")
        assert_bits(scores[offs[b]:offs[b + 1]], s1, tag + " scores")


_CORPORA: dict = {}


def corpus(d):
    if d not in _CORPORA:
        _CORPORA.clear()
        _CORPORA[d] = unit_corpus(N, d, 8, seed=d)
    return _CORPORA[d]


def loop_checks(base, q, subsets, what, ks=(1, 10, 100, 2048, 2049, 200_000)):
    for ties_low in (False, True):
        for k in ks:
            assert_rows_equal_loop(base, q, subsets, k, 0.0, ties_low, what)
    items, scores, counts = base.search_arrays(q, 100, 0.0, subsets=subsets)
    s0 = np.float32(scores[3, 40])  # a hit of the 4096-entry query
    for ms in (s0, np.nextafter(s0, np.float32(-1)), np.nextafter(s0, np.float32(2)), float("nan")):
        for ties_low in (False, True):
            assert_rows_equal_loop(base, q, subsets, 100, float(ms), ties_low, what)
            assert_range_equal_loop(base, q, subsets, float(ms), ties_low, what)


# ---------------------------------------------------------------- (1) equal to a loop of one-query searches
@pytest.mark.parametrize("d", WIDTHS)
@pytest.mark.parametrize("storage", STORAGES)
def test_each_row_equals_the_one_query_search(storage, d):
    v, q = corpus(d)
    base = make_base(v, storage)
    loop_checks(base, q, mixed_subsets(N, seed=d), f"{storage} d={d}")
    base.enable_timing()
    base.search_arrays(q, 10, 0.0, subsets=mixed_subsets(N, seed=1))
    t = base.last_timing()
    assert t["path"] == "scan" and t["scan_ms"] > 0


# ---------------------------------------------------------------- (2) exact arithmetic
def exact_subset_topk(dots, subsets, k, ms, ties_low=False):
    b_n = len(subsets)
    kk = max(1, min(k, max(len(s) for s in subsets)))
    items, scores, counts = np.full((b_n, kk), -1, np.int64), np.zeros((b_n, kk), np.float32), np.zeros(b_n, np.int32)
    offs, all_i, all_s = [0], [], []
    for b, sub in enumerate(subsets):
        sub = np.asarray(sub, np.int64)
        s = scores_of(dots[b])[sub]
        pos = np.arange(len(sub))
        with np.errstate(invalid="ignore"):
            keep = np.flatnonzero(s >= np.float32(ms))
        order = keep[np.lexsort((pos[keep] if ties_low else -pos[keep], -s[keep].astype(np.float64)))]
        all_i.append(sub[order])
        all_s.append(s[order])
        offs.append(offs[-1] + len(order))
        c = min(kk, len(order))
        items[b, :c], scores[b, :c], counts[b] = sub[order[:c]], s[order[:c]], c
    csr = (np.array(offs, np.int64), np.concatenate(all_i).astype(np.int64), np.concatenate(all_s).astype(np.float32))
    return (items, scores, counts), csr


def dyadic(n, d, b, seed):
    amp, exp = preset("fine", d)
    return dyadic_corpus(n, d, b, amp, exp, seed)


@pytest.mark.parametrize("storage", STORAGES)
def test_exact_topk_and_threshold_sets(storage):
    v, q, dots = dyadic(20_000, 64, 8, seed=5)
    base = make_base(v, storage)
    subsets = mixed_subsets(20_000, seed=6)
    subsets[5] = subsets[5][:30_000]
    for ties_low in (False, True):
        for k in (1, 10, 300, 5000, 40_000):
            (want, _) = exact_subset_topk(dots, subsets, k, 0.0, ties_low)
            got = base.search_arrays(q, k, 0.0, subsets=subsets, ties_low_first=ties_low)
            for j in range(3):
                assert_bits(got[j], want[j], f"exact top-k {storage} k={k} ties_low={ties_low}")
        for ms in (0.0, 0.55, 0.75):
            _, want = exact_subset_topk(dots, subsets, 1, ms, ties_low)
            got = base.search_range(q, ms, subsets=subsets, ties_low_first=ties_low)
            for j in range(3):
                assert_bits(got[j], want[j], f"exact range {storage} ms={ms} ties_low={ties_low}")


def test_fuzzy_lookup_embeddings_in_subsets_equals_the_oracle():
    v, q, dots = dyadic(20_000, 64, 6, seed=7)
    rng = np.random.default_rng(8)
    subsets = []
    for b in range(len(q)):  # no tied scores inside a subset: the reference orders ties arbitrarily
        cand = rng.permutation(20_000)[:3000]
        _, first = np.unique(scores_of(dots[b])[cand], return_index=True)
        sub = cand[np.sort(first)][: [0, 1, 9, 500, 2000, 3000][b]]
        sub = np.where(rng.random(len(sub)) < 0.3, sub - 20_000, sub)
        subsets.append(sub.tolist())
    base = make_base(v)
    ref = O.OracleVectorBase(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()))
    ref.add_embeddings(None, v)
    for max_hits in (None, 0, 5):
        for ms in (None, 0.6):
            got = base.fuzzy_lookup_embeddings_in_subsets(q, subsets, max_hits, ms)
            for b in range(len(q)):
                want = ref.fuzzy_lookup_embedding_in_subset(q[b], subsets[b], max_hits, ms)
                one = base.fuzzy_lookup_embedding_in_subset(q[b], subsets[b], max_hits, ms)
                assert [(h.item, np.float32(h.score)) for h in got[b]] == \
                       [(h.item, np.float32(h.score)) for h in want], f"max_hits={max_hits} ms={ms} query {b}"
                assert [(h.item, h.score) for h in got[b]] == [(h.item, h.score) for h in one]
    index = tab.EmbeddingIndex(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()), v)
    got = index.get_indexes_of_nearest_in_subsets_batch(q, subsets, 5, 0.6)
    assert [[(h.item, h.score) for h in r] for r in got] == \
           [[(h.item, h.score) for h in r] for r in base.fuzzy_lookup_embeddings_in_subsets(q, subsets, 5, 0.6)]
    with pytest.raises(ValueError):
        base.fuzzy_lookup_embeddings_in_subsets(q, subsets, -1)


# ---------------------------------------------------------------- (3) skew
def test_one_huge_subset_and_many_tiny_ones():
    v, q, dots = dyadic(50_000, 64, 256, seed=9)
    rng = np.random.default_rng(10)
    subsets = [rng.integers(-50_000, 50_000, size=1_000_000)] + [rng.integers(50_000, size=10) for _ in range(255)]
    base = make_base(v, "bfloat16")
    for k in (10, 100):
        want, csr = exact_subset_topk(dots, subsets, k, 0.5)
        got = base.search_arrays(q, k, 0.5, subsets=subsets)
        for j in range(3):
            assert_bits(got[j], want[j], f"skew top-k k={k}")
    got = base.search_range(q, 0.5, subsets=subsets)
    for j in range(3):
        assert_bits(got[j], csr[j], "skew range")
    assert_rows_equal_loop(base, q[:3], subsets[:3], 100, 0.5, False, "skew")


# ---------------------------------------------------------------- (4) the C ABI
def c_search(lib, ix, q, k, ms, flags, offsets, ordinals):
    b = len(q)
    items, scores, counts = np.zeros((b, k), np.int64), np.zeros((b, k), np.float32), np.zeros(b, np.int32)
    offsets = np.ascontiguousarray(offsets, np.int64)
    ordinals = np.ascontiguousarray(ordinals, np.int64)
    rc = lib.tav_search_subsets(ix, q.ctypes.data_as(C.c_void_p), b, k, C.c_float(ms), flags,
                                offsets.ctypes.data_as(C.c_void_p), ordinals.ctypes.data_as(C.c_void_p),
                                items.ctypes.data_as(C.c_void_p), scores.ctypes.data_as(C.c_void_p),
                                counts.ctypes.data_as(C.c_void_p), None)
    return rc, items, scores, counts


def c_range(lib, ix, q, ms, flags, offsets, ordinals):
    out = np.zeros(len(q) + 1, np.int64)
    offsets = np.ascontiguousarray(offsets, np.int64)
    ordinals = np.ascontiguousarray(ordinals, np.int64)
    rc = lib.tav_range_search_subsets(ix, q.ctypes.data_as(C.c_void_p), len(q), C.c_float(ms), flags,
                                      offsets.ctypes.data_as(C.c_void_p), ordinals.ctypes.data_as(C.c_void_p),
                                      out.ctypes.data_as(C.c_void_p), None)
    return rc, out


def test_c_abi_positions_flags_and_errors():
    v, q = unit_corpus(5000, 64, 4, seed=11)
    base = make_base(v)
    lib, ix = base._ensure_device()
    subsets = [np.array([3, -2, 3, 4999]), np.arange(0, 5000, 7), np.empty(0, np.int64), np.full(300, -17)]
    offsets, ordinals = base._subsets_csr(subsets, 4)

    rc, items, scores, counts = c_search(lib, ix, q, 50, 0.0, 0, offsets, ordinals)
    assert rc == 0
    for tl in (0, _capi.TAV_TIES_LOW_FIRST):
        rc, it0, sc0, c0 = c_search(lib, ix, q, 50, 0.0, tl, offsets, ordinals)
        rc2, pos, sc1, c1 = c_search(lib, ix, q, 50, 0.0, tl | _capi.TAV_ITEMS_AS_POSITIONS, offsets, ordinals)
        assert rc == rc2 == 0
        assert_bits(c1, c0, "positions counts")
        assert_bits(sc1, sc0, "positions scores")
        for b in range(4):
            p = pos[b, :c0[b]]
            assert ((p >= offsets[b]) & (p < offsets[b + 1])).all()
            assert_bits(ordinals[p], it0[b, :c0[b]], "positions map back")
        rc, r_off = c_range(lib, ix, q, 0.4, tl | _capi.TAV_ITEMS_AS_POSITIONS, offsets, ordinals)
        assert rc == 0
        pos_r = np.empty(r_off[-1], np.int64)
        sc_r = np.empty(r_off[-1], np.float32)
        assert lib.tav_range_fetch(ix, 0, r_off[-1], pos_r.ctypes.data_as(C.c_void_p), sc_r.ctypes.data_as(C.c_void_p),
                                   0, None) == 0
        o2, i2, s2 = base.search_range(q, 0.4, subsets=subsets, ties_low_first=bool(tl))
        assert_bits(r_off, o2, "range positions offsets")
        assert_bits(ordinals[pos_r], i2, "range positions map back")

    # a range result to fetch afterwards: refused calls must leave it (and the rows) as they were
    rc, keep_off = c_range(lib, ix, q, 0.4, 0, offsets, ordinals)
    assert rc == 0
    bad_flags = [_capi.TAV_FORCE_MMA, _capi.TAV_FORCE_SCAN, _capi.TAV_USE_ROW_MASK, _capi.TAV_USE_QUERY_MASKS,
                 _capi.TAV_DEFER_RETRY, _capi.TAV_NO_FUSED_SCAN]
    for f in bad_flags:
        assert c_search(lib, ix, q, 10, 0.0, f, offsets, ordinals)[0] == _capi.TAV_ERR_INVALID, f
        assert c_range(lib, ix, q, 0.0, f, offsets, ordinals)[0] == _capi.TAV_ERR_INVALID, f
    for bad in ([1, 4, 10, 10, 310], [0, 4, 3, 10, 310], [0, 4, 10, 10, 1 << 32]):
        assert c_search(lib, ix, q, 10, 0.0, 0, bad, ordinals)[0] == _capi.TAV_ERR_INVALID, bad
        assert c_range(lib, ix, q, 0.0, 0, bad, ordinals)[0] == _capi.TAV_ERR_INVALID, bad
    for o in (5000, -5001):
        wrong = ordinals.copy()
        wrong[7] = o
        assert c_search(lib, ix, q, 10, 0.0, 0, offsets, wrong)[0] == _capi.TAV_ERR_RANGE
        assert _capi.last_error() == f"index {o} is out of bounds for axis 0 with size 5000"
        assert c_range(lib, ix, q, 0.0, 0, offsets, wrong)[0] == _capi.TAV_ERR_RANGE
    got_i = np.empty(keep_off[-1], np.int64)
    got_s = np.empty(keep_off[-1], np.float32)
    assert lib.tav_range_fetch(ix, 0, keep_off[-1], got_i.ctypes.data_as(C.c_void_p), got_s.ctypes.data_as(C.c_void_p),
                               0, None) == 0
    o2, i2, s2 = base.search_range(q, 0.4, subsets=subsets)
    assert_bits(keep_off, o2, "kept offsets")
    assert_bits(got_i, i2, "kept items")
    assert_bits(got_s, s2, "kept scores")
    again = c_search(lib, ix, q, 50, 0.0, 0, offsets, ordinals)
    for j in range(3):
        assert_bits(again[j + 1], (items, scores, counts)[j], "unchanged after refused calls")

    # Python surface: errors before any work
    with pytest.raises(ValueError, match="3 subsets for 4 queries"):
        base.search_arrays(q, 5, subsets=subsets[:3])
    with pytest.raises(ValueError, match="cannot be combined"):
        base.search_arrays(q, 5, subsets=subsets, subset=[1])
    with pytest.raises(ValueError, match="cannot be combined"):
        base.search_range(q, 0.0, subsets=subsets, allowed=np.ones(5000, bool))
    with pytest.raises(IndexError, match="integer"):
        base.search_arrays(q, 5, subsets=[[1], [2.5], [], [3]])
    with pytest.raises(IndexError, match="index 5000 is out of bounds"):
        base.search_arrays(q, 5, subsets=[[1], [5000], [], [3]])
    with pytest.raises(IndexError, match="index -5001 is out of bounds"):
        base.search_range(q, 0.0, subsets=[[1], [-5001], [], [3]])


# ---------------------------------------------------------------- (5) normalisation, (6) row changes
@pytest.mark.parametrize("storage", ["float32", "bfloat16"])
def test_normalising_index(storage):
    rng = np.random.default_rng(12)
    v = rng.standard_normal((30_000, 96), dtype=np.float32) * np.float32(7.0)
    q = rng.standard_normal((8, 96), dtype=np.float32) * np.float32(3.0)
    base = make_base(v, storage, normalize=True)
    subsets = mixed_subsets(30_000, seed=13)
    subsets[5] = subsets[5][:20_000]
    loop_checks(base, q, subsets, f"normalize {storage}", ks=(1, 100, 2049, 50_000))


def test_row_changes_equal_a_fresh_index():
    v, q = unit_corpus(40_000, 64, 8, seed=14)
    base = make_base(v, "bfloat16")
    subsets = mixed_subsets(40_000, seed=15)
    subsets[5] = subsets[5][:30_000]
    base.search_arrays(q, 10, 0.0, subsets=subsets)  # rows on the device before they change
    extra, _ = unit_corpus(1000, 64, 1, seed=16)
    base.add_embeddings(None, extra)
    base.remove_embeddings(np.arange(100, 1100))
    base.set_embeddings_at(500, extra[:200])
    n = len(base)
    subsets = [np.asarray(s, np.int64) % n - (n if i % 2 else 0) for i, s in enumerate(mixed_subsets(n, seed=17))]
    fresh = make_base(np.array(base.serialize()), "bfloat16")
    for k in (10, 3000):
        for tl in (False, True):
            got = base.search_arrays(q, k, 0.0, subsets=subsets, ties_low_first=tl)
            want = fresh.search_arrays(q, k, 0.0, subsets=subsets, ties_low_first=tl)
            for j in range(3):
                assert_bits(got[j], want[j], f"after row changes k={k} ties_low={tl}")
    for j, (g, w) in enumerate(zip(base.search_range(q, 0.55, subsets=subsets), fresh.search_range(q, 0.55, subsets=subsets))):
        assert_bits(g, w, "range after row changes")


# ---------------------------------------------------------------- (7) call order
def test_call_on_another_stream_sees_the_rows_written_before_it():
    import torch

    v, q = unit_corpus(20_000, 64, 4, seed=18)
    new_rows, _ = unit_corpus(5000, 64, 1, seed=19)
    base = make_base(v)
    lib, ix = base._ensure_device()
    subsets = [np.arange(0, 6000, 3), np.arange(-20_000, -15_000), np.arange(100, 200), np.full(50, 1234)]
    offsets, ordinals = base._subsets_csr(subsets, 4)
    after = v.copy()
    after[:5000] = new_rows
    want = make_base(after).search_arrays(q, 100, 0.0, subsets=subsets)

    torch.cuda._sleep(1000)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    torch.cuda._sleep(20_000_000)
    end.record()
    end.synchronize()
    cycles = int(20_000_000 * 200.0 / start.elapsed_time(end))

    held, racing = torch.cuda.Stream(), torch.cuda.Stream()
    rows_dev = torch.from_numpy(new_rows).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(held):
        torch.cuda._sleep(cycles)
    assert lib.tav_write_rows(ix, 0, C.c_void_p(rows_dev.data_ptr()), 5000, 64, _capi.TAV_F32, 1,
                              C.c_void_p(held.cuda_stream)) == 0
    assert not held.query(), "hold too short"
    b = len(q)
    items, scores, counts = np.zeros((b, 100), np.int64), np.zeros((b, 100), np.float32), np.zeros(b, np.int32)
    assert lib.tav_search_subsets(ix, q.ctypes.data_as(C.c_void_p), b, 100, C.c_float(0.0), 0,
                                  offsets.ctypes.data_as(C.c_void_p), ordinals.ctypes.data_as(C.c_void_p),
                                  items.ctypes.data_as(C.c_void_p), scores.ctypes.data_as(C.c_void_p),
                                  counts.ctypes.data_as(C.c_void_p), C.c_void_p(racing.cuda_stream)) == 0
    for j, got in enumerate((items, scores, counts)):
        assert_bits(got, want[j], "racing subsets search")
    torch.cuda.synchronize()


# ---------------------------------------------------------------- (8) broken builds
MUTANTS = {1: "later tiles start one entry late", 2: "negative ordinals come back wrapped", 3: "ties-low ignored"}


@pytest.fixture(scope="module")
def mutant_libs():
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc) and not shutil.which(nvcc):
        pytest.skip("nvcc is needed to build the broken variants")
    from typeagent_py_b200 import build as B

    tmp = tempfile.mkdtemp(prefix="tav_subsets_mutants_")
    procs = {}
    for m in MUTANTS:
        out = os.path.join(tmp, f"libtavec_mutant{m}.so")
        cmd = [nvcc, *[f for f in B.NVCC_FLAGS if f != "-Xptxas=-v"], f"-DTAV_SUBSETS_MUTANT={m}", "-o", out,
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
    v, q = unit_corpus(20_000, 64, 8, seed=20)
    subsets = mixed_subsets(20_000, seed=21)
    subsets[5] = subsets[5][:10_000]
    caught = []
    for tl in (False, True):
        base = make_base(v, "bfloat16")
        try:
            assert_rows_equal_loop(base, q, subsets, 100, 0.0, tl, "mutant check")
            assert_range_equal_loop(base, q, subsets, 0.5, tl, "mutant check")
        except AssertionError as e:
            caught.append(str(e)[:200])
    return caught


@pytest.mark.parametrize("m", sorted(MUTANTS), ids=[MUTANTS[m].replace(" ", "_") for m in sorted(MUTANTS)])
def test_broken_build_is_caught(mutant_libs, m):
    with library(mutant_libs[m]):
        caught = mutant_checks()
    assert caught, f"the exact checks did not catch: {MUTANTS[m]}"


def test_checks_pass_on_the_real_build():
    assert mutant_checks() == []
