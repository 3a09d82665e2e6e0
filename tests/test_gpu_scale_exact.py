"""Every query, bit for bit, at the benchmark's sizes and past 2^24 rows (tests/exact_torch.py).

The small exact tests (test_gpu_exact, _range, _subsets, _query_masks) stop at 120k rows, where each tensor-core
unit walks a few tiles.  Here dyadic corpora (tests/exact.py, preset "scale": dots spread to std ~0.15, so the
top 2048 of 10M rows stay below the clip at score 1.0) are built on the device, and every search is compared
with the exact device reference for every query of the batch: items, float32 score bits and counts, no
tolerances.  The plan make_plan (tav_mma.cu) picks for 10M x 768 bf16, B = 256: 2 query chunks, 66 units per
chunk of ~592 tiles, 264 candidate segments of at most 125 keys per query, 128-row sample blocks, target 2048.

  * 10M x 768 bf16: the benchmark's plan (k = 100), small-k targets (k = 1, 8), the streaming finalize after
    sampling (k = 600, 2048), a ragged second chunk (B = 129) and one query on the tensor cores, min_score at
    a rank-50 score and one ulp either side, row masks (0.5, 1e-3, the last 37 rows), per-query masks (320 MB),
    the row scan (one host query, device queries, three paging passes, ties-low), the threshold search on the
    tensor cores (the default collect region overflows: one re-pass) and on the row scan (radix sort of ~5M-key
    segments, both tie orders), per-query subsets (256 x 4096 ordinals and one of 4M), segment overflow from
    100k copies of one row (flagged, redone exactly, synchronous and deferred), and a library-owned copy of
    the corpus with 1% of its rows removed in place (~57 windows of 256 MB), then 1M rows overwritten;
  * 2^24 + 2^20 + 37 rows x 64 bf16: row positions float32 cannot hold exactly, 69k tiles: top-k on the tensor
    cores and the row scan with item_offset = 2^32 + 5, the threshold search on both, subsets with ordinals
    above 2^24 and one query of 2^24 + 5 entries (flat index j above 2^24), per-query masks;
  * config 4's shard (1.25M x 1536 fp16, B = 1024: eight query chunks), config 5 (50k x 384 bf16, B = 1000,
    k = 5), and the float32 split form (4M x 768 float32: path mma_split);
  * deliberately broken builds (``TAV_SCALE_MUTANT``: 24-bit row keys in the tensor-core epilogue, a 24-bit flat
    index in the subset gather, the radix sort's position byte 3 skipped): each passes the small exact tests and
    test_gpu_fullsize, and is caught here.

One anchor ties the device reference to the numpy one the rest of the suite trusts: two queries of the 10M
corpus, their dots computed by numpy in float64 from the corpus read back, through ``exact.expected_topk``.
Each corpus is freed before the next is built; a device with too little free memory skips with the bytes needed.
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
from tests import exact_torch as T
from tests.exact import expected_topk, preset
from tests.test_gpu_exact import assert_equal_results
from tests.test_gpu_range import assert_same_range, main_kernels
from typeagent_py_b200 import _capi

pytestmark = pytest.mark.gpu

GB = 1 << 30
N_LONG = (1 << 24) + (1 << 20) + 37
OFFSET = (1 << 32) + 5


# ---------------------------------------------------------------- corpora, one at a time
class Corpus:
    def __init__(self, name, n, d, dtype, b_max, seed):
        import torch

        self.name, self.n, self.d = name, n, d
        self.amp, self.exp = preset("scale", d)
        dev = torch.device("cuda", 0)
        gen = torch.Generator(device=dev).manual_seed(seed)
        self.t = self._dyadic(n, d, dtype, gen, dev)
        self.q = self._dyadic(b_max, d, torch.float32, gen, dev)
        self.gen = gen
        self.base = self.wrap()

    def _dyadic(self, n, d, dtype, gen, dev):
        import torch

        out = torch.empty((n, d), dtype=dtype, device=dev)
        step = max(1, (1 << 28) // d)
        for r0 in range(0, n, step):
            r1 = min(n, r0 + step)
            out[r0:r1] = torch.randint(-self.amp, self.amp + 1, (r1 - r0, d), generator=gen, device=dev,
                                       dtype=torch.int16).to(dtype)
        return out.mul_(2.0 ** -self.exp)  # a power of two: exact

    def wrap(self):
        base = tab.VectorBase.from_device_tensor(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()), self.t)
        base.enable_timing()
        return base

    def dots(self, q):
        return T.dyadic_dots(self.t, q, self.exp)


_CORPORA: dict = {}
SPECS = {  # name: (rows, width, dtype, queries drawn, seed)
    "10M": (10_000_000, 768, "bfloat16", 1024, 1),
    "long": (N_LONG, 64, "bfloat16", 256, 2),
    "c4": (1_250_000, 1536, "float16", 1024, 3),
    "c5": (50_000, 384, "bfloat16", 1000, 4),
    "split": (4_000_000, 768, "float32", 256, 5),
}


def corpus(name) -> Corpus:
    import torch

    if name not in _CORPORA:
        _CORPORA.clear()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        n, d, dt, b, seed = SPECS[name]
        dtype = getattr(torch, dt)
        elem = torch.tensor([], dtype=dtype).element_size()
        # the corpus (and a float32 index's two fp16 planes), plus the reference's blocks and the masks
        need = n * d * elem * (2 if dt == "float32" else 1) + 8 * GB
        free = torch.cuda.mem_get_info()[0]
        if free < need:
            pytest.skip(f"corpus {name} needs {need} bytes of free device memory, {free} are free")
        _CORPORA[name] = Corpus(name, n, d, dtype, b, seed)
    return _CORPORA[name]


def teardown_module(module):
    import torch

    _CORPORA.clear()
    torch.cuda.empty_cache()


# ---------------------------------------------------------------- searches and expectations
def np3(res):
    return tuple(x.cpu().numpy() for x in res)


def search(c, q, k, ms, path, allowed=None, item_offset=0):
    """-> ((items, scores, counts) numpy, queries redone, last_timing() of the search itself).  mma / defer /
    scan: search_device on device queries (synchronous, deferred + finish_search, row scan); scan1 / scan2:
    search_arrays on host queries (single launch, scan + select kernels); ties_low: search_arrays with
    ties_low_first.  ``allowed``: a bool CUDA tensor [N] (row mask) or packed int32 words [B, W] (query masks)."""
    import torch

    base = c.base
    base.force_path = {"mma": "mma", "defer": "mma", "scan": "scan", "scan1": "scan", "scan2": "scan2",
                       "ties_low": "scan"}[path]
    if allowed is not None and allowed.dtype == torch.bool:
        allowed = allowed.cpu().numpy()
    if path in ("mma", "defer", "scan"):
        res = base.search_device(q, k, ms, item_offset=item_offset, defer_check=path == "defer", allowed=allowed)
        timing = base.last_timing()  # before finish_search: the search's own launches
        redone = base.finish_search()
        torch.cuda.synchronize()
        return np3(res), redone, timing
    got = base.search_arrays(q.cpu().numpy(), k, ms, allowed=allowed, ties_low_first=path == "ties_low")
    return got, 0, base.last_timing()


def assert_plan(t, split=False, launches=None):
    """The tensor-core path with its sample pass (every corpus here is large enough to be sampled)."""
    assert t["path"] == ("mma_split" if split else "mma"), t
    assert sum(1 for name, _ in t["kernels"] if name == "sample") == 1, t
    if launches is not None:
        assert t["launches"] == launches, t  # query prep, sample, main, finalize


def pack_words(allowed):
    """bool [B, N] CUDA tensor -> int32 [B, ceil(N / 32)] packed words (bit r of word r // 32 = row r)."""
    import torch

    b, n = allowed.shape
    w = (n + 31) // 32
    out = torch.empty((b, w), dtype=torch.int32, device=allowed.device)
    weights = torch.ones(32, dtype=torch.int64, device=allowed.device) << torch.arange(32, device=allowed.device)
    for q0 in range(0, b, 8):
        bits = torch.zeros((min(8, b - q0), w * 32), dtype=torch.int64, device=allowed.device)
        bits[:, :n] = allowed[q0:q0 + 8]
        words = (bits.view(len(bits), w, 32) * weights).sum(-1)
        out[q0:q0 + len(bits)] = torch.where(words >= 1 << 31, words - (1 << 32), words).to(torch.int32)
    return out


def random_masks(c, b, densities):
    """bool [b, N]: query i allows a random share densities[i % len] of the rows; an int density is a number of
    rows (a query that allows fewer rows than k)."""
    import torch

    out = torch.zeros((b, c.n), dtype=torch.bool, device=c.t.device)
    for i in range(b):
        p = densities[i % len(densities)]
        if isinstance(p, int):
            out[i, torch.randint(0, c.n, (int(p),), generator=c.gen, device=c.t.device)] = True
        else:
            out[i] = torch.rand(c.n, generator=c.gen, device=c.t.device) < p
    return out


def row_mask(c, kind):
    import torch

    if kind is None:
        return None
    if kind == "last37":
        m = torch.zeros(c.n, dtype=torch.bool, device=c.t.device)
        m[-37:] = True
        return m
    return torch.rand(c.n, generator=c.gen, device=c.t.device) < {"half": 0.5, "sparse": 1e-3}[kind]


def min_score_for(c, kind):
    """0, or query 0's rank-50 score, or its float32 neighbours."""
    if kind == "0":
        return 0.0
    _, s, _ = T.topk_ref(c.dots(c.q[:1]), 50, 0.0)
    hit = np.float32(s[0, 49].item())
    assert 0 < hit < 1
    step = {"hit": None, "hit+ulp": np.float32(2), "hit-ulp": np.float32(-1)}[kind]
    return float(hit if step is None else np.nextafter(hit, step))


def expect(c, q, k, ms, allowed=None, ties_low=False, item_offset=0):
    return np3(T.topk_ref(c.dots(q), k, ms, allowed, ties_low, item_offset))


def range_c(lib, ix, q, ms, flags, item_offset=0, hint=0):
    """tav_range_search + tav_range_fetch with an item offset -> numpy CSR."""
    qh = np.ascontiguousarray(q.cpu().numpy())
    offsets = np.zeros(len(qh) + 1, np.int64)
    _capi.check(lib.tav_range_search(ix, qh.ctypes.data_as(C.c_void_p), len(qh), C.c_float(ms), flags, None, 0,
                                     item_offset, hint, offsets.ctypes.data_as(C.c_void_p), None))
    total = int(offsets[-1])
    items, scores = np.empty(total, np.int64), np.empty(total, np.float32)
    if total:
        _capi.check(lib.tav_range_fetch(ix, 0, total, items.ctypes.data_as(C.c_void_p),
                                        scores.ctypes.data_as(C.c_void_p), 0, None))
    return offsets, items, scores


def subsets_case(c, sizes, seed):
    """Per-query ordinal lists over all rows (negatives and repeats included) -> (list of numpy, offsets and
    ordinals as CUDA tensors)."""
    import torch

    rng = np.random.default_rng(seed)
    subs = []
    for m in sizes:
        s = rng.integers(-c.n, c.n, size=m)
        if m > 100:
            s[rng.integers(0, m, size=m // 100)] = s[0]  # repeats
        subs.append(s)
    offsets = np.zeros(len(subs) + 1, np.int64)
    offsets[1:] = np.cumsum(sizes)
    ordinals = np.concatenate(subs)
    return subs, torch.from_numpy(offsets).cuda(), torch.from_numpy(ordinals).cuda()


def check_subsets(c, q, subs, offsets, ordinals, k, ms, what):
    want_k, want_r = T.subsets_ref(T.subset_dots(c.t, q, c.exp, offsets, ordinals), offsets, ordinals,
                                   max(1, min(k, max(len(s) for s in subs))), ms)
    got = c.base.search_arrays(q.cpu().numpy(), k, ms, subsets=subs)
    assert_equal_results(got, np3(want_k), f"{what} subsets top-k")
    assert_same_range(c.base.search_range(q.cpu().numpy(), ms, subsets=subs), np3(want_r), f"{what} subsets range")


# ================================================================ 10M x 768 bf16 (BASELINE configs[2])
P = pytest.param
TOPK_10M = [  # (B, k, min_score kind, path, mask)
    P(256, 100, "0", "defer", None, id="bench_plan-B256-k100"),
    P(256, 1, "0", "defer", None, id="k1-small_k_target"),
    P(256, 8, "0", "defer", None, id="k8-small_k_target"),
    P(256, 600, "0", "defer", None, id="k600-streaming_finalize"),
    P(256, 2048, "0", "defer", None, id="k2048-streaming_finalize"),
    P(129, 100, "0", "mma", None, id="B129-ragged_second_chunk"),
    P(1, 100, "0", "mma", None, id="B1-forced_tensor_cores"),
    P(256, 100, "hit", "defer", None, id="min_at_rank50_score"),
    P(256, 100, "hit+ulp", "defer", None, id="min_ulp_above"),
    P(256, 100, "hit-ulp", "defer", None, id="min_ulp_below"),
    P(256, 100, "0", "defer", "half", id="mask_half"),
    P(256, 100, "0", "defer", "sparse", id="mask_1e-3"),
    P(256, 100, "0", "mma", "last37", id="mask_last37_rows-ragged_last_tile"),
    P(1, 50, "0", "scan1", None, id="scan-one_host_query-scan_select"),
    P(8, 100, "0", "scan", None, id="scan-B8-device_queries"),
    P(2, 4097, "0", "scan2", None, id="scan-B2-k4097-three_passes"),
    P(16, 100, "0", "ties_low", None, id="scan-ties_low"),
]


@pytest.mark.parametrize("b,k,ms_kind,path,mask", TOPK_10M)
def test_10m_topk_every_query(b, k, ms_kind, path, mask):
    c = corpus("10M")
    q = c.q[:b].contiguous()
    ms = min_score_for(c, ms_kind)
    allowed = row_mask(c, mask)
    want = expect(c, q, k, ms, allowed, ties_low=path == "ties_low")
    got, redone, t = search(c, q, k, ms, path, allowed)
    assert_equal_results(got, want, f"10M {path} B={b} k={k} ms={ms!r} mask={mask}")
    if path in ("mma", "defer"):
        assert_plan(t, launches=4 if path == "defer" else None)
        if mask in (None, "half"):
            assert redone == 0, redone  # well-mixed rows: the sampled threshold settles every query
    else:
        assert t["path"] == "scan", t
        if path == "scan1":  # 15 GB of rows exceed what the single-launch form takes: scan + select
            assert t["launches"] == 2, t
        if path == "scan2":
            assert t["launches"] % (2 * 3) == 0, t  # scan + select per pass, three passes
    if mask == "last37":
        assert (got[2] == 37).all()


def test_10m_spread_keeps_the_sampled_path_unclipped():
    """The corpus is what the plan is sized for: for nearly every query the top 2048 lie below the clip."""
    c = corpus("10M")
    _, s, counts = np3(T.topk_ref(c.dots(c.q[:256]), 2048, 0.0))
    assert (counts == 2048).all()
    assert (s[:, 0] < 1.0).mean() >= 0.9, (s[:, 0] == 1.0).sum()


def test_10m_per_query_masks():
    """B = 256 masks of 10M rows (320 MB of words), densities 1 / 0.1 / 1e-3 / 10 rows: a query that allows
    fewer rows than k is admitted at the floor."""
    c = corpus("10M")
    q = c.q[:256].contiguous()
    masks = random_masks(c, 256, [1.0, 0.1, 1e-3, 10])
    words = pack_words(masks)
    want = expect(c, q, 100, 0.0, masks)
    for path in ("defer", "mma"):
        got, _, t = search(c, q, 100, 0.0, path, words)
        assert_equal_results(got, want, f"10M per-query masks {path}")
        assert_plan(t)
    assert (want[2][3::4] <= 10).all() and (want[2][::4] == 100).all()
    del masks, words


def test_10m_range_on_the_tensor_cores_repass():
    """B = 16, min_score where the median query has ~30k hits: the default region (16,384 per query)
    overflows and one re-pass collects the rest; the same call with the previous total as the hint."""
    c = corpus("10M")
    q = c.q[:16].contiguous()
    _, s, _ = np3(T.topk_ref(c.dots(q), 30_000, 0.0))
    ms = float(np.median(s[:, -1]))
    want = np3(T.range_ref(c.dots(q), ms))
    assert np.median(np.diff(want[0])) > 16_384
    base = c.base
    base.force_path = "mma"
    base._range_hint = 0
    assert_same_range(base.search_range(q.cpu().numpy(), ms), want, "10M range, default hint")
    assert main_kernels(base) == 2, base.last_timing()
    assert base.last_timing()["path"] == "mma"
    assert base._range_hint == want[0][-1]
    # with the total as the hint each query's region is 1.5x the mean and each segment twice its even share of
    # that: queries within 1.5x the mean fit, and the single collection pass serves the call
    counts = np.diff(want[0])
    assert counts.max() <= 1.5 * counts.mean(), counts
    assert_same_range(base.search_range(q.cpu().numpy(), ms), want, "10M range, previous total as hint")
    assert main_kernels(base) == 1, base.last_timing()


@pytest.mark.parametrize("ties_low", [False, True])
def test_10m_range_on_the_row_scan_radix(ties_low):
    """B = 3, min_score 0.5: ~5M hits per query, each segment radix-sorted."""
    c = corpus("10M")
    q = c.q[:3].contiguous()
    want = np3(T.range_ref(c.dots(q), 0.5, ties_low=ties_low))
    assert (np.diff(want[0]) > 4_000_000).all()
    c.base.force_path = "scan"
    got = c.base.search_range(q.cpu().numpy(), 0.5, ties_low_first=ties_low)
    assert c.base.last_timing()["path"] == "scan"
    assert_same_range(got, want, f"10M range scan ties_low={ties_low}")


def test_10m_subsets():
    """256 queries of 4096 ordinals over all 10M rows and one of 4M (negatives, repeats): top-k and range."""
    c = corpus("10M")
    q = c.q[:257].contiguous()
    subs, offsets, ordinals = subsets_case(c, [4096] * 256 + [4_000_000], seed=10)
    check_subsets(c, q, subs, offsets, ordinals, 100, 0.0, "10M")
    check_subsets(c, q, subs, offsets, ordinals, 100, 0.55, "10M min 0.55")


def test_10m_anchor_to_numpy():
    """Two queries: numpy float64 dots of the corpus read back in 500k-row blocks -> exact.expected_topk equals
    the device reference."""
    c = corpus("10M")
    qh = c.q[:2].cpu().numpy().astype(np.float64)
    dots = np.empty((2, c.n), np.float32)
    for r0 in range(0, c.n, 500_000):
        blk = c.t[r0:r0 + 500_000].float().cpu().numpy()
        dots[:, r0:r0 + len(blk)] = (qh @ blk.astype(np.float64).T).astype(np.float32)
    for k, ms in ((100, 0.0), (2048, 0.6)):
        want = expected_topk(dots, k, ms)
        got = np3(T.topk_ref(c.dots(c.q[:2]), k, ms))
        assert_equal_results(got, want, f"device reference vs numpy k={k}")


def test_10m_segment_overflow_redone_exactly():
    """100k copies of query 0's best row, spread over the corpus (the first row, rows above 2^23, the last):
    query 0's segments overflow, it is flagged and redone exactly; the tie order after the redo is the
    library's (higher row first).  The deferred form shows the flag: before finish_search the flagged queries
    hold no hits.  The synchronous form returns the same batch exact and leaves nothing for tav_finish_search,
    so it redid the flagged queries itself.  The corpus is restored afterwards."""
    import torch

    c = corpus("10M")
    base = c.base
    q = c.q[:256].contiguous()
    best = int(T.topk_ref(c.dots(q[:1]), 1, 0.0)[0][0, 0])
    rng = np.random.default_rng(11)
    rows = np.unique(np.concatenate([[0, (1 << 23) + 1, c.n - 1], rng.choice(c.n, 100_000, replace=False)]))
    rows = torch.from_numpy(rows[rows != best]).cuda()
    saved = c.t[rows].clone()
    try:
        c.t[rows] = c.t[best].clone()
        torch.cuda.synchronize()
        want = expect(c, q, 100, 0.0)
        assert (want[0][0] >= 0).all() and len(np.unique(want[1][0])) == 1  # a tie of copies
        assert want[0][0, 0] == c.n - 1
        base.force_path = "mma"
        res = base.search_device(q, 100, 0.0, defer_check=True)
        torch.cuda.synchronize()
        before = np3(res)
        flagged = np.flatnonzero((before[2] != want[2]) | (before[0] != want[0]).any(1))
        assert 0 in flagged, "query 0 was not flagged"
        assert (before[2][flagged] == 0).all() and (before[0][flagged] == -1).all(), "a wrong query was not flagged"
        redone = base.finish_search()
        torch.cuda.synchronize()
        assert redone >= len(flagged)
        assert_equal_results(np3(res), want, "overflow, deferred, after finish_search")
        got, _, _ = search(c, q, 100, 0.0, "mma")
        assert_equal_results(got, want, "overflow, synchronous")
        lib, ix = base._ensure_device()
        left = C.c_int(-1)
        _capi.check(lib.tav_finish_search(ix, None, C.byref(left)))
        assert left.value == 0, "the synchronous search left flagged queries behind"
    finally:
        c.t[rows] = saved
        torch.cuda.synchronize()


def survivor_dots(c, q, keep, first=0, new=None, step=1 << 18):
    """Dots of an index holding rows ``keep`` of the corpus, in that order (the renumbering of a removal), with
    rows [first, first + len(new)) overwritten by ``new``."""
    for p0 in range(0, len(keep), step):
        rows = c.t[keep[p0:p0 + step]]
        if new is not None:
            lo, hi = max(p0, first), min(p0 + len(rows), first + len(new))
            if lo < hi:
                rows[lo - p0:hi - p0] = new[lo - first:hi - first]
        for _, dots in T.dyadic_dots(rows, q, c.exp, block_rows=len(rows)):
            yield p0, dots


def test_10m_removal_in_place_windows_then_overwrite():
    """A library-owned index appended from the device corpus (tav_append): 1% of the rows removed at random
    (negatives and a repeat among the ordinals) by the default in-place compaction, ~57 windows of 256 MB; then
    1M rows overwritten (tav_write_rows).  Top-k on the tensor cores and the threshold search after each step
    equal the exact result of the surviving rows, renumbered in order."""
    import torch

    c = corpus("10M")
    need = c.n * c.d * 2 + 8 * GB
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip(f"a second copy of the 10M corpus needs {need} bytes of free device memory, {free} are free")
    lib = _capi.load()
    ix = C.c_void_p()
    _capi.check(lib.tav_create(0, c.d, _capi.TAV_BF16, 0, c.n, C.byref(ix)))
    compact_stats = lib.tav_internal_compact_stats
    compact_stats.argtypes, compact_stats.restype = [C.c_void_p, C.c_void_p, C.c_void_p], C.c_int
    q = c.q[:256].contiguous()

    def check(keep, first=0, new=None, what=""):
        assert lib.tav_size(ix) == len(keep)
        b, k = len(q), 100
        out = (torch.empty((b, k), dtype=torch.int64, device="cuda"), torch.empty((b, k), dtype=torch.float32,
                                                                                    device="cuda"),
               torch.empty(b, dtype=torch.int32, device="cuda"))
        flags = _capi.TAV_QUERIES_ON_DEVICE | _capi.TAV_OUTPUTS_ON_DEVICE | _capi.TAV_FORCE_MMA
        _capi.check(lib.tav_search(ix, C.c_void_p(q.data_ptr()), b, k, C.c_float(0.0), flags, None, 0, 0,
                                   *(C.c_void_p(t.data_ptr()) for t in out), None))
        torch.cuda.synchronize()
        scan, total, launches, path = C.c_float(0), C.c_float(0), C.c_int(0), C.c_int(0)
        _capi.check(lib.tav_last_timing(ix, C.byref(scan), C.byref(total), C.byref(launches), C.byref(path)))
        assert path.value == 2, "not the tensor-core path"
        want = np3(T.topk_ref(survivor_dots(c, q, keep, first, new), k, 0.0))
        assert_equal_results(np3(out), want, f"top-k {what}")
        qr = q[:16]
        want = np3(T.range_ref(survivor_dots(c, qr, keep, first, new), 0.7))
        assert_same_range(range_c(lib, ix, qr, 0.7, _capi.TAV_FORCE_MMA), want, f"range {what}")

    try:
        _capi.check(lib.tav_append(ix, C.c_void_p(c.t.data_ptr()), c.n, c.d, _capi.TAV_BF16, 1, None))
        rng = np.random.default_rng(14)
        gone = rng.choice(c.n, c.n // 100, replace=False)
        gone[:10] -= c.n  # the same rows, counted from the end
        gone = np.concatenate([gone, gone[10:11]])  # a repeat removes one row
        _capi.check(lib.tav_remove_rows(ix, np.ascontiguousarray(gone, np.int64).ctypes.data_as(C.c_void_p),
                                        len(gone), None))
        removed = np.unique(np.where(gone < 0, gone + c.n, gone))
        keep_mask = torch.ones(c.n, dtype=torch.bool, device="cuda")
        keep_mask[torch.from_numpy(removed).cuda()] = False
        keep = torch.nonzero(keep_mask).squeeze(1)  # surviving row p of the index: corpus row keep[p]
        del keep_mask
        path, windows = C.c_int(0), C.c_int64(0)
        _capi.check(compact_stats(ix, C.byref(path), C.byref(windows)))
        moving = len(keep) - int(removed[0])
        window_rows = (256 << 20) // (c.d * 2)
        assert path.value == 2, "the compaction was not in place"
        assert windows.value == -(-moving // window_rows), (windows.value, moving)
        assert windows.value >= 50
        check(keep, what="after removing 1%")

        first = 3_000_000
        new = c._dyadic(1_000_000, c.d, torch.bfloat16, c.gen, c.t.device)
        _capi.check(lib.tav_write_rows(ix, first, C.c_void_p(new.data_ptr()), len(new), c.d, _capi.TAV_BF16, 1,
                                       None))
        torch.cuda.synchronize()
        check(keep, first, new, what="after overwriting 1M rows")
    finally:
        lib.tav_destroy(ix)
        torch.cuda.empty_cache()


# ================================================================ 2^24 + 2^20 + 37 rows x 64 bf16
@pytest.mark.parametrize("path", ["defer", "scan"])
def test_long_topk_item_offset(path):
    c = corpus("long")
    b = 256 if path == "defer" else 8
    q = c.q[:b].contiguous()
    want = expect(c, q, 100, 0.0, item_offset=OFFSET)
    assert (want[0] - OFFSET >= 1 << 24).any()
    got, redone, t = search(c, q, 100, 0.0, path, item_offset=OFFSET)
    assert_equal_results(got, want, f"long {path}")
    if path == "defer":
        assert_plan(t, launches=4)
        assert redone == 0
    else:
        assert t["path"] == "scan", t


@pytest.mark.parametrize("flags,b,ties_low", [
    P(_capi.TAV_FORCE_MMA, 16, False, id="mma-B16"),
    P(_capi.TAV_FORCE_SCAN, 3, False, id="scan-B3-radix"),
    P(_capi.TAV_FORCE_SCAN | _capi.TAV_TIES_LOW_FIRST, 3, True, id="scan-B3-radix-ties_low"),
])
def test_long_range_item_offset(flags, b, ties_low):
    c = corpus("long")
    q = c.q[:b].contiguous()
    ms = 0.6 if flags & _capi.TAV_FORCE_MMA else 0.5
    want = np3(T.range_ref(c.dots(q), ms, ties_low=ties_low, item_offset=OFFSET))
    assert (want[1] - OFFSET >= 1 << 24).any() and (np.diff(want[0]) > 4096).all()
    assert_same_range(range_c(*c.base._ensure_device(), q, ms, flags, OFFSET), want, f"long range flags={flags}")


def test_long_subsets_past_2_24_entries():
    """One query of 2^24 + 5 entries (flat index j above 2^24), then queries of ordinals above 2^24."""
    import torch

    c = corpus("long")
    q = c.q[:4].contiguous()
    subs, _, _ = subsets_case(c, [(1 << 24) + 5, 4096, 4096, 300], seed=12)
    rng = np.random.default_rng(13)
    subs[1] = rng.integers(1 << 24, c.n, size=4096)
    subs[3] = np.concatenate([np.full(100, c.n - 1), np.full(100, -1), rng.integers(1 << 24, c.n, size=100)])
    offsets = np.zeros(5, np.int64)
    offsets[1:] = np.cumsum([len(s) for s in subs])
    offsets, ordinals = torch.from_numpy(offsets).cuda(), torch.from_numpy(np.concatenate(subs)).cuda()
    check_subsets(c, q, subs, offsets, ordinals, 100, 0.0, "long")
    check_subsets(c, q, subs, offsets, ordinals, 100, 0.7, "long min 0.7")


def test_long_per_query_masks():
    c = corpus("long")
    q = c.q[:32].contiguous()
    masks = random_masks(c, 32, [0.5, 1e-3, 10, 0.5])
    masks[3::4, :1 << 24] = False  # only rows above 2^24
    words = pack_words(masks)
    want = expect(c, q, 100, 0.0, masks)
    got, _, _ = search(c, q, 100, 0.0, "defer", words)
    assert_equal_results(got, want, "long per-query masks")


# ---------------------------------------------------------------- broken builds
MUTANTS = {1: "tensor-core keys keep 24 bits of the row", 2: "subset gather keeps 24 bits of j",
           3: "radix sort skips position byte 3"}


@pytest.fixture(scope="module")
def mutant_libs():
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc) and not shutil.which(nvcc):
        pytest.skip("nvcc is needed to build the broken variants")
    from typeagent_py_b200 import build as B

    tmp = tempfile.mkdtemp(prefix="tav_scale_mutants_")
    procs = {}
    try:
        for m in MUTANTS:
            out = os.path.join(tmp, f"libtavec_mutant{m}.so")
            cmd = [nvcc, *[f for f in B.NVCC_FLAGS if f != "-Xptxas=-v"], f"-DTAV_SCALE_MUTANT={m}", "-o", out,
                   *[os.path.join(B.CSRC, s) for s in B.SOURCES]]
            procs[m] = (subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True), out)
        logs = {m: proc.communicate()[0] for m, (proc, _) in procs.items()}  # every build ends before any check
        failed = {m: logs[m] for m, (proc, _) in procs.items() if proc.returncode != 0}
        assert not failed, f"broken builds that did not compile: {failed}"
        libs = {}
        for m, (_, out) in procs.items():
            lib = C.CDLL(out)
            for name, (restype, argtypes) in _capi.SIGNATURES.items():
                fn = getattr(lib, name)
                fn.restype, fn.argtypes = restype, argtypes
            libs[m] = lib
        yield libs
    finally:
        for proc, _ in procs.values():  # only left running when the fixture itself was interrupted
            if proc.poll() is None:
                proc.kill()
                proc.wait()
        shutil.rmtree(tmp, ignore_errors=True)


@contextlib.contextmanager
def library(lib):
    saved = _capi._lib
    _capi._lib = lib
    try:
        yield
    finally:
        _capi._lib = saved


@pytest.mark.parametrize("m", sorted(MUTANTS), ids=[MUTANTS[m].replace(" ", "_") for m in sorted(MUTANTS)])
def test_broken_build_is_caught(mutant_libs, m):
    c = corpus("long")
    real = c.base
    caught = []
    with library(mutant_libs[m]):
        c.base = c.wrap()
        try:
            for check in (lambda: test_long_topk_item_offset("defer"),
                          lambda: test_long_subsets_past_2_24_entries(),
                          lambda: test_long_range_item_offset(_capi.TAV_FORCE_SCAN, 3, False)):
                try:
                    check()
                except AssertionError as e:
                    caught.append(str(e)[:200])
        finally:
            c.base = real
    assert caught, f"the exact checks did not catch: {MUTANTS[m]}"


# ================================================================ configs 4 and 5, the float32 split form
def test_config4_shard_eight_query_chunks():
    c = corpus("c4")
    q = c.q[:1024].contiguous()
    want = expect(c, q, 100, 0.0)
    got, redone, t = search(c, q, 100, 0.0, "defer")
    assert_equal_results(got, want, "config 4 shard B=1024")
    assert_plan(t, launches=4)
    assert redone == 0


def test_config5_small_k():
    c = corpus("c5")
    q = c.q[:1000].contiguous()
    want = expect(c, q, 5, 0.0)
    got, redone, t = search(c, q, 5, 0.0, "defer")
    assert_equal_results(got, want, "config 5 B=1000 k=5")
    assert_plan(t, launches=4)
    assert redone == 0


def test_float32_split_form():
    c = corpus("split")
    q = c.q[:256].contiguous()
    want = expect(c, q, 100, 0.0)
    got, redone, t = search(c, q, 100, 0.0, "defer")
    assert_equal_results(got, want, "split form top-k")
    assert_plan(t, split=True)
    assert redone == 0
    want = np3(T.range_ref(c.dots(q[:16]), 0.7))
    c.base.force_path = "mma"
    assert_same_range(c.base.search_range(q[:16].cpu().numpy(), 0.7), want, "split form range")
    assert c.base.last_timing()["path"] == "mma_split"
