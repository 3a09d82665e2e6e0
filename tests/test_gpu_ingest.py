"""What the kernels are fed, bit for bit: append conversion, the scalar row scan, and normalisation.

1. Append conversion (``tav_append`` -> ``tav_read_rows``) for every (source, storage) pair of float32,
   bfloat16 and float16 — the same-type pairs take the plain copy, the others the convert kernel — from
   host and device buffers, against a CPU reference (numpy for float16, ``round_to_bfloat16`` for
   bfloat16; 16-bit sources are upcast exactly and rounded once).  The values cover halfway cases, the
   largest finite value and one ulp past it, the fp16 overflow threshold, subnormals, values that round to
   zero, +-0, +-inf and NaN.  NaN is compared with isnan, everything else by its bits.  Also: a host
   append of several 32 MB pinned staging chunks, and appends that cross capacity doublings.
2. The scalar form of the row scan (rows that are not a multiple of 16 bytes) on dyadic corpora
   (tests/exact.py): every scan form must equal ``expected_topk`` exactly, for every query.
3. Normalisation (``TAV_NORMALIZE``): rows with sum a_i^2 = 4^m times any power of two in [2^-100, 2^64]
   normalise exactly to a / 2^m, so every search path must equal ``expected_topk`` of the exact dots; random
   rows of any scale lie within ``normalize_error_bound``; zero, NaN and inf rows and zero queries keep
   the semantics written in tavec.h.
4. A deferred search redoes its flagged queries with its own queries, whatever searches follow it.
5. ``tav_mma_scores`` normalises as the search does: the search equals top-k of those dots.
"""

from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import typeagent_py_b200 as tab
from oracle import vectorbase_oracle as O
from tests.exact import (conversion_edges, dyadic_corpus, expected_topk, normalize_error_bound,
                         preset, round_to, scores_of, to_bits16, unit_rows)
from tests.test_gpu_exact import assert_dump_within_bound, assert_equal_results, row_mask
from tests.test_gpu_mma import mma_scores
from tests.test_gpu_range import assert_same_range, expected_range
from typeagent_py_b200 import _capi

pytestmark = pytest.mark.gpu

P = pytest.param
SHORT = {"float32": "f32", "bfloat16": "bf16", "float16": "fp16"}
DTYPES = list(SHORT)


# ------------------------------------------------------------------ C ABI plumbing
class Index:
    """A bare libtavec index (no host mirror): appends and reads through the C ABI."""

    def __init__(self, storage, normalize=False):
        self.lib = _capi.load()
        self.h = C.c_void_p()
        _capi.check(self.lib.tav_create(0, 0, _capi.DTYPE_CODES[storage], _capi.TAV_NORMALIZE if normalize else 0,
                                        0, C.byref(self.h)))

    def append(self, values, src, where="host"):
        """values: float32 [n, d] holding values of dtype `src`; sent as `src` from host or device memory."""
        import torch

        n, d = values.shape
        buf = values if src == "float32" else to_bits16(values, src)
        buf = np.ascontiguousarray(buf)
        code = _capi.DTYPE_CODES[src]
        if where == "host":
            _capi.check(self.lib.tav_append(self.h, buf.ctypes.data_as(C.c_void_p), n, d, code, 0, None))
        else:
            t = torch.from_numpy(buf.view(np.int32 if src == "float32" else np.int16)).cuda()
            _capi.check(self.lib.tav_append(self.h, C.c_void_p(t.data_ptr()), n, d, code, 1, None))
            torch.cuda.synchronize()

    def read(self):
        return read_rows(self.lib, self.h)

    def close(self):
        self.lib.tav_destroy(self.h)


def read_rows(lib, h):
    """Every stored row, upcast to float32 on the device (exact)."""
    n, d = lib.tav_size(h), lib.tav_dim(h)
    out = np.empty((n, d), np.float32)
    _capi.check(lib.tav_read_rows(h, 0, n, out.ctypes.data_as(C.c_void_p), None))
    return out


def assert_same_values(got, want, what, classes=None):
    """NaN where NaN, every other value bit for bit (so -0.0 != +0.0)."""
    got, want = np.asarray(got, np.float32).ravel(), np.asarray(want, np.float32).ravel()
    gn, wn = np.isnan(got), np.isnan(want)
    bad = np.flatnonzero((gn != wn) | (~wn & (got.view(np.uint32) != want.view(np.uint32))))
    if len(bad):
        i = bad[0]
        cls = f" ({classes[i]})" if classes is not None else ""
        raise AssertionError(f"{what}: {len(bad)} of {len(got)} values differ, first #{i}{cls}: "
                             f"{got[i]!r} (0x{got.view(np.uint32)[i]:08x}) vs {want[i]!r} (0x{want.view(np.uint32)[i]:08x})")


def as_rows(flat, d, extra_rows=1):
    n = -(-len(flat) // d) + extra_rows
    out = np.zeros(n * d, np.float32)
    out[: len(flat)] = flat
    out[len(flat):] = np.resize(flat, n * d - len(flat))  # the tail repeats the values at other columns
    return out.reshape(n, d)


# ------------------------------------------------------------------ 1. append conversion
PAIRS = [(s, t) for s in DTYPES for t in DTYPES]
PAIR_IDS = [f"{SHORT[s]}_to_{SHORT[t]}" + ("-plain" if s == t else "-convert") for s, t in PAIRS]


def edge_matrix(seed=0):
    """(flat float32 values, class label per value): every edge class plus values of random scales."""
    rng = np.random.default_rng(seed)
    edges = conversion_edges()
    scale = np.exp2(rng.integers(-150, 126, 2000).astype(np.float64))
    rand = (rng.standard_normal(2000) * scale).astype(np.float32)
    flat = np.concatenate([*edges.values(), *(-v for v in edges.values()), rand])
    classes = np.concatenate([np.full(len(v), k) for k, v in edges.items()] * 2 + [np.full(len(rand), "random_scale")])
    return flat, classes


def check_append(src, dst, rows, where, what, classes=None):
    src_vals = round_to(rows, src)  # what a `src` buffer can hold
    ix = Index(dst)
    try:
        ix.append(src_vals, src, where)
        assert_same_values(ix.read(), round_to(src_vals, dst), what, classes)
    finally:
        ix.close()


@pytest.mark.parametrize("where", ["host", "device"])
@pytest.mark.parametrize("d", [1, 3, 5, 7, 8, 9, 100, 1535], ids=lambda d: f"d{d}")
@pytest.mark.parametrize("src,dst", PAIRS, ids=PAIR_IDS)
def test_append_converts_every_edge_value_bit_for_bit(src, dst, d, where):
    flat, classes = edge_matrix(seed=d)
    rows = as_rows(flat, d)
    check_append(src, dst, rows, where, f"{src}->{dst} d={d} {where}", np.resize(classes, rows.size))


@pytest.mark.parametrize("cls", list(conversion_edges()))
@pytest.mark.parametrize("src,dst", PAIRS, ids=PAIR_IDS)
def test_append_edge_class(src, dst, cls):
    vals = conversion_edges()[cls]
    rows = as_rows(np.concatenate([vals, -vals]), 5)
    check_append(src, dst, rows, "host", f"{src}->{dst} {cls}")


@pytest.mark.parametrize("dst", ["bfloat16", "float32"], ids=["convert_f32_to_bf16", "plain_f32"])
def test_host_append_of_several_pinned_chunks(dst):
    """20000 x 1536 float32 = 3.66 chunks of the 32 MB pinned double buffer: both buffers, a partial last one."""
    rng = np.random.default_rng(7)
    rows = rng.standard_normal((20000, 1536), dtype=np.float32)
    rows *= np.exp2(rng.integers(-20, 20, (20000, 1))).astype(np.float32)
    ix = Index(dst)
    try:
        ix.append(rows, "float32", "host")
        got = ix.read()
        assert got.shape == rows.shape
        assert_same_values(got, round_to(rows, dst), f"{dst} chunks")
    finally:
        ix.close()


@pytest.mark.parametrize("src,dst", [("float32", "bfloat16"), ("float32", "float32"), ("float16", "bfloat16")],
                         ids=["f32_to_bf16-convert", "f32_to_f32-plain", "fp16_to_bf16-convert"])
def test_appends_across_capacity_doublings(src, dst):
    """1, 1023, 1, 5000, ... rows: capacity 1024 -> 2048 -> ... ; growth copies the old rows on the device."""
    rng = np.random.default_rng(11)
    d = 100
    ix = Index(dst)
    want = np.empty((0, d), np.float32)
    try:
        for i, n in enumerate([1, 1023, 1, 5000, 3, 9000, 1]):
            rows = round_to((rng.standard_normal((n, d)) * 3).astype(np.float32), src)
            ix.append(rows, src, "host" if i % 2 == 0 else "device")
            want = np.concatenate([want, round_to(rows, dst)])
            assert_same_values(ix.read(), want, f"after append #{i} of {n} rows")
    finally:
        ix.close()


# ------------------------------------------------------------------ 2. the scalar row scan
def make_index(v, storage, path, normalize=False):
    base = tab.VectorBase(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()), storage_dtype=storage,
                          normalize=normalize)
    base.add_embeddings(None, v)
    base.force_path = path
    base.enable_timing()
    return base


SCALAR_WIDTHS = [(s, d) for s in ("bfloat16", "float16") for d in (1, 3, 5, 12, 100, 1001)] + \
                [("float32", d) for d in (1, 3, 5, 17, 101)]
SCAN_FORMS = ["scan1", "scan2", "device", "subset", "mask", "range"]
# k on both sides of the 64 (watched result slots / completion word) and 2048 (one pass) switches
SCAN_KS = {"scan1": (64, 65), "scan2": (64, 2048, 2049), "device": (64, 65), "subset": (65, 2049),
           "mask": (64, 2049), "range": (None,)}


_SMEM_BUDGET, _PASS_K, _FUSED_MAX, _SMS = 160 * 1024, 2048, 8192, 132


def scan_launches(d, b, k, n_scan, fuse=True):
    """Launches of the row-scan search (scan_search in tav_api.cu): queries in blocks of the largest power of
    two whose query rows and candidate lists fit the shared-memory budget; per block and pass of <= 2048 hits a
    scan and a select kernel, or the scan alone when its last CTA merges (one pass of k <= 64 whose grid of
    one CTA per 32-row tile leaves at most 8192 survivors)."""
    pass_k, n_pass = min(k, _PASS_K), -(-k // _PASS_K)
    cap = max(128, 1 << (2 * pass_k - 1).bit_length())
    qb = next(q for q in (8, 4, 2, 1) if (q * d * 4 + 15) // 16 * 16 + q * cap * 8 <= _SMEM_BUDGET)
    qb = 1 << (min(qb, b).bit_length() - 1)
    tiles = -(-n_scan // 32)
    assert tiles <= _SMS  # the grid is one CTA per tile here
    fused = fuse and n_pass == 1 and pass_k <= 64 and tiles * max(pass_k, 32) <= _FUSED_MAX
    return -(-b // qb) * n_pass * (1 if fused else 2)


def collect_launches(d, counts, hint, n_scan):
    """Launches of the row-scan threshold search (range_collect_scan): collect scans over blocks of queries,
    one more for the queries whose hits overflowed their region (sized from the hint, the previous total),
    then one segmented-sort launch when there are hits (every segment here is a small one)."""
    b = len(counts)
    qb = next(q for q in (8, 4, 2, 1) if (q * d * 4 + 15) // 16 * 16 <= _SMEM_BUDGET)
    per = 16384 if hint == 0 else (lambda m: m + m // 2 + 32)(-(-hint // b))
    per = max(1, min(per, n_scan))
    over = int((np.asarray(counts) > per).sum())
    assert max(counts) <= 4096
    return -(-b // qb) + -(-over // qb) + (1 if sum(counts) else 0)


@pytest.mark.parametrize("form", SCAN_FORMS)
@pytest.mark.parametrize("storage,d", SCALAR_WIDTHS, ids=[f"{SHORT[s]}-d{d}-row{d * (4 if s == 'float32' else 2)}B"
                                                           for s, d in SCALAR_WIDTHS])
def test_scalar_row_scan_every_form_bit_for_bit(storage, d, form):
    import torch

    n, b = 4000, 9
    assert (d * (4 if storage == "float32" else 2)) % 16 != 0  # the scalar (non-vector) kernel
    amp, exp = preset("fine", d)
    v, q, dots = dyadic_corpus(n, d, b, amp, exp, seed=n + d)
    base = make_index(v, storage, "scan2" if form == "scan2" else "scan")
    for k in SCAN_KS[form]:
        what = f"{form} {storage} d={d} k={k}"
        if form == "scan1":  # one host query per call: the single-launch form
            for i in range(2):
                got = base.search_arrays(q[i:i + 1], k, 0.0)
                assert_equal_results(got, expected_topk(dots[i:i + 1], k, 0.0), what)
                t = base.last_timing()
                assert t["path"] == "scan" and t["launches"] == 1, t
            continue
        if form == "scan2":
            got = base.search_arrays(q, k, 0.0)
            assert_equal_results(got, expected_topk(dots, k, 0.0), what)
            t = base.last_timing()
            assert t["path"] == "scan" and t["launches"] == scan_launches(d, b, k, n, fuse=False), t
        elif form == "device":
            res = base.search_device(torch.from_numpy(q).cuda(), k, 0.0)
            torch.cuda.synchronize()
            assert_equal_results(tuple(t.cpu().numpy() for t in res), expected_topk(dots, k, 0.0), what)
            t = base.last_timing()
            assert t["path"] == "scan" and t["launches"] == scan_launches(d, b, k, n), t
        elif form == "subset":
            sub = np.sort(np.random.default_rng(d).choice(n, 3000, replace=False))
            got = base.search_arrays(q, k, 0.0, subset=sub)
            wi, ws, wc = expected_topk(dots[:, sub], k, 0.0)
            want = (np.where(wi >= 0, sub[np.maximum(wi, 0)], -1), ws, wc)
            assert_equal_results(got, want, what)
            t = base.last_timing()
            assert t["path"] == "scan" and t["launches"] == scan_launches(d, b, k, len(sub)), t
        elif form == "mask":
            allowed = row_mask("half", n, seed=d)
            got = base.search_arrays(q, k, 0.0, allowed=allowed)
            assert_equal_results(got, expected_topk(dots, k, 0.0, allowed), what)
            t = base.last_timing()
            assert t["path"] == "scan" and t["launches"] == scan_launches(d, b, k, n), t
        else:  # threshold search, collect mode of the row scan
            for ms in (0.0, float(np.sort(scores_of(dots[0]))[-50])):
                hint = base._range_hint  # the previous call's total sizes the regions
                got = base.search_range(q, ms)
                want = expected_range(dots, ms)
                assert_same_range(got, want, f"{what} min_score={ms}")
                t = base.last_timing()
                assert t["path"] == "scan" and t["launches"] == collect_launches(d, np.diff(want[0]), hint, n), t


# ------------------------------------------------------------------ 3. normalisation
def exact_unit_corpus(n, d, b, seed, e_range=(-100, 64)):
    """Rows and queries of any power-of-two scale whose normalised forms a / 2^m are exact, and their
    exact normalised dots (float32)."""
    v, a, m, _ = unit_rows(n, d, 255, seed, e_range)
    q, qa, mq, _ = unit_rows(b, d, 255, seed + 1, e_range)
    dots = ((qa @ a.T).astype(np.float64) * 2.0 ** -(m + mq)).astype(np.float32)
    return v, q, dots, a.astype(np.float32) * np.float32(2.0 ** -m)


NORM_PATHS = [
    P("float32", "scan2", 6000, id="f32-scan2"),
    P("bfloat16", "scan2", 6000, id="bf16-scan2"),
    P("float16", "device", 6000, id="fp16-device_scan"),
    P("float32", "device", 6000, id="f32-device_scan"),
    P("bfloat16", "mma", 6000, id="bf16-mma"),
    P("float16", "mma", 6000, id="fp16-mma"),
    P("bfloat16", "mma", 20000, id="bf16-mma-sampled"),
    P("float32", "mma", 6000, id="f32-mma_split"),
    P("bfloat16", "range_scan", 6000, id="bf16-range_scan"),
    P("float16", "range_mma", 6000, id="fp16-range_mma"),
    P("float32", "range_mma", 6000, id="f32-range_mma_split"),
    P("bfloat16", "defer", 6000, id="bf16-defer_finish"),
    P("float32", "defer", 6000, id="f32-defer_finish"),
]


@pytest.mark.parametrize("storage,path,n", NORM_PATHS)
def test_normalised_search_is_exact_for_rows_of_any_scale(storage, path, n):
    import torch

    d, b, k = 64, 40, 32
    v, q, dots, unit = exact_unit_corpus(n, d, b, seed=n + len(path))
    force = {"scan2": "scan2", "device": "scan", "range_scan": "scan"}.get(path, "mma")
    base = make_index(v, storage, force, normalize=True)
    assert_same_values(read_rows(*base._ensure_device()), unit, "stored rows")  # a / 2^m exactly, whatever 2^e the row came with
    if path.startswith("range"):
        got = base.search_range(q, 0.0)
        assert_same_range(got, expected_range(dots, 0.0), f"{path} {storage}")
    elif path in ("device", "defer"):
        res = base.search_device(torch.from_numpy(q).cuda(), k, 0.0, defer_check=path == "defer")
        base.finish_search()
        torch.cuda.synchronize()
        assert_equal_results(tuple(t.cpu().numpy() for t in res), expected_topk(dots, k, 0.0), f"{path} {storage}")
    else:
        assert_equal_results(base.search_arrays(q, k, 0.0), expected_topk(dots, k, 0.0), f"{path} {storage}")
    want_path = "scan" if force != "mma" else ("mma_split" if storage == "float32" else "mma")
    assert base.last_timing()["path"] == want_path, base.last_timing()


@pytest.mark.parametrize("d", [1, 7, 64, 1536], ids=lambda d: f"d{d}")
@pytest.mark.parametrize("storage", DTYPES, ids=SHORT.get)
def test_normalised_rows_of_random_scale_within_bound(storage, d):
    """Each stored element within the rigorous bound of float64 v / ||v||: scales 2^-140 .. 2^100 per row
    (float32 subnormal inputs included) and a 2^-60 spread inside rows (squares below the normal range)."""
    rng = np.random.default_rng(d)
    n = max(64, 20000 // d)
    v = rng.standard_normal((n, d)) * np.exp2(rng.integers(-140, 101, (n, 1)))
    v *= np.where(rng.random((n, d)) < 0.2, 2.0 ** -60, 1.0)
    v = v.astype(np.float32)
    v = v[np.abs(v).max(1) > 0]
    ix = Index(storage, normalize=True)
    try:
        ix.append(v, "float32")
        got = ix.read().astype(np.float64)
    finally:
        ix.close()
    vv = v.astype(np.float64)
    exact = vv / np.sqrt((vv * vv).sum(1, keepdims=True))
    err = np.abs(got - exact)
    bound = normalize_error_bound(v, storage)
    worst = np.unravel_index(np.argmax(err - bound), err.shape)
    assert (err <= bound).all(), f"row {worst[0]} (max |v| {np.abs(v[worst[0]]).max():.3g}): error {err[worst]:.3g} > bound {bound[worst]:.3g}"


@pytest.mark.parametrize("path", ["scan", "mma"])
@pytest.mark.parametrize("storage", DTYPES, ids=SHORT.get)
def test_normalise_edge_semantics(storage, path):
    """A zero row stays zero (score 0.5); a row with NaN or +-inf is never returned; a zero query returns
    every other row at 0.5."""
    d, n, b = 64, 300, 16
    v, q, _, _ = exact_unit_corpus(n, d, b, seed=5, e_range=(-20, 20))
    zero, nan, pinf, ninf = 10, 20, 30, 40
    v[zero] = 0.0
    v[nan, 3] = np.nan
    v[pinf, 0] = np.inf
    v[ninf, 63] = -np.inf
    q[1] = 0.0
    base = make_index(v, storage, path, normalize=True)
    items, scores, counts = base.search_arrays(q, n, -2.0)
    assert base.last_timing()["path"].startswith(path), base.last_timing()
    bad = {nan, pinf, ninf}
    for i in range(b):
        got = dict(zip(items[i, : counts[i]].tolist(), scores[i, : counts[i]].tolist()))
        assert counts[i] == n - 3 and not bad & set(got), f"q{i}: {counts[i]} hits"
        assert got[zero] == 0.5
        if i == 1:
            assert set(got.values()) == {0.5}
    rows = read_rows(*base._ensure_device())
    assert (rows[zero].view(np.uint32) == 0).all()
    assert np.isnan(rows[[nan, pinf, ninf]]).any(1).all()


def test_tensor_core_query_rounding_on_a_normalising_index():
    """Normalised queries a / 2^m with |a| <= 1023 are exact in float32 but not in bfloat16: the tensor cores
    must see them rounded to nearest even, and at d = 8 every dot of those rounded queries is exact."""
    d, n, b = 8, 3000, 40
    v, a, m, _ = unit_rows(n, d, 255, seed=21)
    q, qa, mq, _ = unit_rows(b, d, 1023, seed=22)
    qn = qa.astype(np.float32) * np.float32(2.0 ** -mq)
    assert (round_to(qn, "bfloat16") != qn).any()
    want = (round_to(qn, "bfloat16").astype(np.float64) @ (a * 2.0 ** -m).T).astype(np.float32)
    base = make_index(v, "bfloat16", "mma", normalize=True)
    assert_same_values(mma_scores(base, q), want, "dump of bf16-rounded normalised queries")


# ------------------------------------------------------------------ 4. deferred search on a normalising index
@pytest.mark.parametrize("second", ["defer_same_batch", "defer_smaller_batch", "scan", "range"])
@pytest.mark.parametrize("storage", ["bfloat16", "float32"], ids=SHORT.get)
def test_deferred_search_redoes_its_own_queries(storage, second):
    """Identical rows tie every score, so the tensor-core search flags every query; its redo at
    finish_search must use its own queries although a second search (never larger, so no buffer is
    reallocated) has staged other queries on the index since."""
    import torch

    d, n, b, k = 64, 30000, 16, 7
    v, a, m, _ = unit_rows(1, d, 255, seed=3)
    qs, qi, mq, _ = unit_rows(2 * b, d, 255, seed=4)
    unit, qunit = a * 2.0 ** -m, qi * 2.0 ** -mq  # exact normalised forms (float64)
    qa, qb = qs[:b], qs[b:]
    base = make_index(np.repeat(v, n, axis=0), storage, "mma", normalize=True)

    def want(qn, kk=k):
        s = scores_of((qn @ unit[0]).astype(np.float32))  # exact in float64, and so in float32
        return np.repeat(s[:, None], kk, axis=1)

    res_a = base.search_device(torch.from_numpy(qa).cuda(), k, -2.0, defer_check=True)
    if second.startswith("defer"):
        nb = b if second == "defer_same_batch" else b // 2
        res_b = base.search_device(torch.from_numpy(qb[:nb]).cuda(), k, -2.0, defer_check=True)
    elif second == "scan":
        base.force_path = "scan"
        got_b = base.search_arrays(qb, k, -2.0)
        np.testing.assert_array_equal(got_b[1], want(qunit[b:]))
    else:
        base.force_path = "scan"
        offsets, items, scores = base.search_range(qb[:2], 1.5)  # nothing passes; the queries are staged all the same
        assert offsets[-1] == 0
    redone = base.finish_search()
    torch.cuda.synchronize()
    assert redone == b + (nb if second.startswith("defer") else 0)  # every query of every deferred search
    items, scores, counts = (t.cpu().numpy() for t in res_a)
    assert (counts == k).all() and (items == np.arange(n - 1, n - 1 - k, -1)).all()
    assert_same_values(scores, want(qunit[:b]), f"search A after a {second} search")
    if second.startswith("defer"):
        assert_same_values(res_b[1].cpu().numpy(), want(qunit[b:b + nb]), "search B")


@pytest.mark.parametrize("storage", ["bfloat16", "float32"], ids=SHORT.get)
def test_deferred_searches_stay_deferred_when_their_queries_outgrow_the_buffer(storage):
    """Four deferred searches of 96 to 200 KB of normalised queries each (more than the 64 KB first
    allocation, and each of the second and fourth more than what is left): the held-query space grows while
    the earlier searches are still outstanding, none of them is finished early, so finish_search redoes every
    query of all four, each with its own queries."""
    import torch

    d, n, k = 256, 30000, 5
    sizes = [128, 160, 96, 200]
    v, a, m, _ = unit_rows(1, d, 255, seed=13)
    qs, qi, mq, _ = unit_rows(sum(sizes), d, 255, seed=14)
    unit, qunit = a[0] * 2.0 ** -m, qi * 2.0 ** -mq
    base = make_index(np.repeat(v, n, axis=0), storage, "mma", normalize=True)
    bounds = np.cumsum([0] + sizes)
    res = [base.search_device(torch.from_numpy(qs[lo:hi]).cuda(), k, -2.0, defer_check=True)
           for lo, hi in zip(bounds[:-1], bounds[1:])]
    assert base.finish_search() == sum(sizes)
    torch.cuda.synchronize()
    for i, (lo, hi) in enumerate(zip(bounds[:-1], bounds[1:])):
        items, scores, counts = (t.cpu().numpy() for t in res[i])
        assert (counts == k).all() and (items == np.arange(n - 1, n - 1 - k, -1)).all()
        want = np.repeat(scores_of((qunit[lo:hi] @ unit).astype(np.float32))[:, None], k, axis=1)
        assert_same_values(scores, want, f"deferred search {i} of {len(sizes)}")


# ------------------------------------------------------------------ 5. tav_mma_scores on a normalising index
@pytest.mark.parametrize("storage", ["bfloat16", "float32"], ids=SHORT.get)
def test_mma_scores_normalise_like_the_search(storage):
    """The search equals top-k of the dots tav_mma_scores dumps for every unflagged query, and the dump is
    within the rigorous bound of the exact dots of the stored rows and the (exactly normalised) queries."""
    import torch

    n, d, b, k = 40000, 64, 130, 32
    rng = np.random.default_rng(17)
    v = (rng.standard_normal((n, d)) * np.exp2(rng.integers(-60, 60, (n, 1)))).astype(np.float32)
    q, qa, m, _ = unit_rows(b, d, 255, seed=18, e_range=(-60, 60))
    qn = qa.astype(np.float32) * np.float32(2.0 ** -m)
    split = storage == "float32"
    base = make_index(v, storage, "mma", normalize=True)
    stored = read_rows(*base._ensure_device())
    dump = mma_scores(base, q)
    assert_dump_within_bound(dump, qn, stored, split)
    res = base.search_device(torch.from_numpy(q).cuda(), k, 0.0, defer_check=True)
    torch.cuda.synchronize()
    items, scores, counts = (t.cpu().numpy() for t in res)
    assert base.last_timing()["path"] == ("mma_split" if split else "mma")
    want = expected_topk(dump, k, 0.0)
    same = (counts == want[2]) & (items == want[0]).all(1) & (scores.view(np.uint32) == want[1].view(np.uint32)).all(1)
    flagged = np.flatnonzero(~same)
    assert (counts[flagged] == 0).all(), f"q{flagged[:5]} differ from the dump's top-k but were not flagged"
    assert len(flagged) <= base.finish_search() <= b // 10
