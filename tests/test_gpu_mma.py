"""The wgmma tensor-core path (bf16 / fp16 storage, batched queries) against the oracle.

Inputs are rounded to the storage dtype first ("identical fp32 inputs": the oracle gets the
rounded values upcast to float32), so products are exact in float32 and only the summation
order differs between the tensor core and OpenBLAS: scores agree to ~1e-6, index sets up to
ties at that level (tests/parity.py).
  * raw GEMM check: every dot product the kernel computes (tav_mma_scores) vs float64;
  * search parity vs the oracle, with and without the sampled admission threshold;
  * row-scan kernel vs tensor-core kernel on the same data (two independent CUDA paths);
  * the exact-fallback: score distributions that defeat the sampled threshold.
"""

from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import typeagent_py_b200 as tab
from oracle import vectorbase_oracle as O
from tests.exact import dot_error_bound
from tests.parity import assert_hits_match
from typeagent_py_b200 import _capi

pytestmark = pytest.mark.gpu


def make_base(v, storage, path="mma"):
    base = tab.VectorBase(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()), storage_dtype=storage)
    base.add_embeddings(None, v)
    base.force_path = path
    base.enable_timing()
    return base


def mma_scores(base, q):
    import torch

    lib, ix = base._ensure_device()
    out = torch.empty((len(q), len(base)), dtype=torch.float32, device="cuda")
    q = np.ascontiguousarray(q, np.float32)
    _capi.check(lib.tav_mma_scores(ix, q.ctypes.data_as(C.c_void_p), len(q), 0,
                                   C.c_void_p(out.data_ptr()), None))
    return out.cpu().numpy()


@pytest.mark.parametrize("storage", ["bfloat16", "float16"])
@pytest.mark.parametrize("n,d,b", [(256, 64, 128), (1000, 768, 5), (3001, 136, 130), (700, 1536, 256),
                                    (513, 8, 300), (40000, 384, 64), (3001, 72, 1), (2000, 64, 133 * 128 + 5)])
def test_every_dot_product_of_the_tensor_core_path(storage, n, d, b):
    v, q = O.make_corpus(n, d, seed=n + d, n_queries=b)
    vr, qr = O.round_to_storage(v, storage), O.round_to_storage(q, storage)
    base = make_base(v, storage)
    got = mma_scores(base, q)
    want = qr.astype(np.float64) @ vr.astype(np.float64).T
    assert got.shape == want.shape
    # fp32 accumulation of exact products: at most gamma_d * sum |q_i v_i| in any order, typically
    # ~sqrt(d) * 2^-24 * |x|
    assert (np.abs(got - want) <= dot_error_bound(qr, vr)).all()
    np.testing.assert_allclose(got, want, atol=2e-6, rtol=0)


@pytest.mark.parametrize("storage,n,d,b,k,ms", [
    ("bfloat16", 20000, 768, 64, 32, 0.0),      # sampled threshold
    ("bfloat16", 50000, 384, 300, 5, 0.0),      # two query chunks (256 + 44), RelatedTerms shape
    ("float16", 30000, 1536, 17, 100, 0.0),
    ("bfloat16", 4000, 128, 200, 10, 0.0),      # small corpus: no sampling, floor threshold
    ("float16", 20011, 256, 33, 50, 0.52),      # min_score above the sampled threshold for some
    ("bfloat16", 16385, 64, 256, 2048, 0.0),    # k = pass limit
    ("bfloat16", 100000, 64, 8, 10, 0.0),
])
def test_search_matches_oracle(storage, n, d, b, k, ms):
    v, q = O.make_corpus(n, d, seed=n + b, n_queries=b)
    vr, qr = O.round_to_storage(v, storage), O.round_to_storage(q, storage)
    base = make_base(v, storage)
    batch = base.fuzzy_lookup_embeddings(qr, max_hits=k, min_score=ms)
    assert base.last_timing()["path"] == "mma"
    for i in list(range(min(b, 12))) + [b - 1]:
        assert_hits_match(batch[i], O.lookup(vr, qr[i], k, ms), min_score=ms, what=f"{storage} q{i}")


@pytest.mark.parametrize("storage,n,d,b,k,ms", [
    ("bfloat16", 50000, 384, 1000, 5, 0.0),     # BASELINE configs[4] shape
    ("bfloat16", 50000, 384, 40, 5, 0.56),      # threshold cuts most rows
    ("float16", 300, 64, 130, 8, 0.0),          # corpus smaller than one tile... and k = register limit
    ("bfloat16", 70000, 128, 256, 1, 0.0),
    ("float16", 20000, 200, 17, 3, 0.9),        # nothing passes for most queries
])
def test_small_k_many_queries(storage, n, d, b, k, ms):
    """k <= 8 (the RelatedTerms shape): the threshold is the 8th largest block maximum of the sample, so
    at least 8 >= k rows are always admitted — no query may ever need the exact fallback here."""
    v, q = O.make_corpus(n, d, seed=n + b + k, n_queries=b)
    vr, qr = O.round_to_storage(v, storage), O.round_to_storage(q, storage)
    base = make_base(v, storage)
    batch = base.fuzzy_lookup_embeddings(qr, max_hits=k, min_score=ms)
    t = base.last_timing()
    assert t["path"] == "mma" and t["launches"] <= 4      # prep, [sample], main, finalize: ONE pass for all chunks
    for i in list(range(min(b, 10))) + [b // 2, b - 1]:
        assert_hits_match(batch[i], O.lookup(vr, qr[i], k, ms), min_score=ms, what=f"{storage} q{i}")


def test_small_k_ties_and_duplicates():
    row = O.round_to_bfloat16(O.make_corpus(1, 64, seed=9)[0])
    same = np.repeat(row, 20000, axis=0)
    base = make_base(same, "bfloat16")
    for hits in base.fuzzy_lookup_embeddings(np.repeat(row, 20, axis=0), 7, 0.0):
        assert [h.item for h in hits] == list(range(19999, 19992, -1))


@pytest.mark.parametrize("storage,k", [("bfloat16", 20), ("bfloat16", 4), ("float32", 20)])
def test_thresholds_on_the_tensor_core_path(storage, k):
    """min_score edges through the admission-threshold machinery: nothing can pass (> 1), everything
    passes (negative), and a threshold equal to an achieved score keeps that row (>=)."""
    v, q = O.make_corpus(20000, 64, seed=77, n_queries=24)
    if storage != "float32":
        v, q = O.round_to_storage(v, storage), O.round_to_storage(q, storage)
    base = make_base(v, storage, None)
    assert all(h == [] for h in base.fuzzy_lookup_embeddings(q, k, 1.5))
    assert base.last_timing()["path"] in ("mma", "mma_split")
    everything = base.fuzzy_lookup_embeddings(q, k, -2.0)
    top = base.fuzzy_lookup_embeddings(q, k, 0.0)
    assert [[h.item for h in a] for a in everything] == [[h.item for h in b] for b in top]
    cut = float(top[5][k // 2].score)
    again = base.fuzzy_lookup_embeddings(q, k, cut)[5]
    assert [h.item for h in again] == [h.item for h in top[5][: k // 2 + 1]]
    for i in (0, 5, 23):
        assert_hits_match(base.fuzzy_lookup_embeddings(q, k, 0.55)[i], O.lookup(v, q[i], k, 0.55), min_score=0.55)


def test_unrounded_float32_queries_are_rounded_like_the_corpus():
    v, q = O.make_corpus(20000, 256, seed=5, n_queries=20)
    base = make_base(v, "bfloat16")
    vr, qr = O.round_to_bfloat16(v), O.round_to_bfloat16(q)
    for got, qq in zip(base.fuzzy_lookup_embeddings(q, 10, 0.0), qr):
        assert_hits_match(got, O.lookup(vr, qq, 10, 0.0))


def test_scan_and_mma_paths_agree():
    v, q = O.make_corpus(60000, 512, seed=77, n_queries=40)
    qr = O.round_to_bfloat16(q)
    a = make_base(v, "bfloat16", "mma").search_arrays(qr, 64, 0.0)
    b = make_base(v, "bfloat16", "scan").search_arrays(qr, 64, 0.0)
    np.testing.assert_array_equal(a[2], b[2])
    for i in range(len(qr)):
        assert_hits_match({"items": a[0][i].tolist(), "scores": a[1][i].tolist()},
                          {"items": b[0][i].tolist(), "scores": b[1][i].tolist()}, score_tol=2e-6)


def test_auto_path_selection():
    v, q = O.make_corpus(20000, 128, seed=3, n_queries=32)
    base = make_base(v, "bfloat16", None)
    base.fuzzy_lookup_embeddings(q, 5, 0.0)
    assert base.last_timing()["path"] == "mma"
    base.fuzzy_lookup_embedding(q[0], 5, 0.0)
    assert base.last_timing()["path"] == "scan"
    f32 = make_base(v, "float32", None)
    f32.fuzzy_lookup_embeddings(q, 5, 0.0)
    assert f32.last_timing()["path"] == "mma_split"   # float32 rows through their two fp16 planes
    f32.fuzzy_lookup_embeddings(q[:4], 5, 0.0)
    assert f32.last_timing()["path"] == "scan"
    odd = make_base(O.make_corpus(5000, 100, seed=1)[0], "bfloat16", "mma")  # 200-byte rows: no TMA
    with pytest.raises(ValueError):
        odd.fuzzy_lookup_embeddings(O.make_corpus(20, 100, seed=2)[0], 5, 0.0)


def test_fallback_when_the_sampled_threshold_cannot_decide():
    """(a) 30000 identical rows: every score ties -> all rows admitted -> candidate overflow;
    (b) the best rows hide in one unsampled tile and everything else scores far lower:
    the threshold from the sample is fine (admits them) — but a corpus whose sampled tiles are
    all high-scoring and the rest low starves the admission.  Both must still be exact."""
    row = O.round_to_bfloat16(O.make_corpus(1, 64, seed=9)[0])
    same = np.repeat(row, 30000, axis=0)
    base = make_base(same, "bfloat16")
    got = base.fuzzy_lookup_embeddings(np.repeat(row, 3, axis=0), 7, 0.0)
    for hits in got:
        assert [h.item for h in hits] == list(range(29999, 29992, -1))
    # starvation: tile 0 is sampled and holds near-duplicates of the query; nothing else comes close
    v, q = O.make_corpus(40000, 64, seed=10, n_queries=2)
    v = v.copy()
    v[:256] = q[0] + 0.01 * v[:256]
    v[:256] /= np.linalg.norm(v[:256], axis=1, keepdims=True)
    vr, qr = O.round_to_bfloat16(v), O.round_to_bfloat16(q)
    base = make_base(v, "bfloat16")
    got = base.fuzzy_lookup_embeddings(qr, 400, 0.0)
    for hits, qq in zip(got, qr):
        assert_hits_match(hits, O.lookup(vr, qq, 400, 0.0))


def test_deferred_check_async_search_and_finish():
    """search_device(defer_check=True) never synchronises; finish_search() redoes flagged queries."""
    import torch

    # (a) ordinary data: nothing to redo, results final right after the stream drains
    v, q = O.make_corpus(30000, 128, seed=12, n_queries=40)
    vr, qr = O.round_to_bfloat16(v), O.round_to_bfloat16(q)
    base = make_base(v, "bfloat16")
    qd = torch.from_numpy(qr).cuda()
    items, scores, counts = base.search_device(qd, 20, 0.0, defer_check=True)
    assert base.finish_search() == 0 and base.finish_search() == 0
    for b in range(0, 40, 7):
        got = {"items": items[b, : counts[b]].tolist(), "scores": scores[b, : counts[b]].tolist()}
        assert_hits_match(got, O.lookup(vr, qr[b], 20, 0.0))
    # (b) every score ties -> candidate overflow -> every query flagged -> exact after finish
    row = O.round_to_bfloat16(O.make_corpus(1, 64, seed=9)[0])
    same = make_base(np.repeat(row, 30000, axis=0), "bfloat16")
    qd = torch.from_numpy(np.repeat(row, 5, axis=0)).cuda()
    items, scores, counts = same.search_device(qd, 9, 0.0, defer_check=True)
    assert same.finish_search() == 5
    torch.cuda.synchronize()
    for b in range(5):
        assert items[b].tolist() == list(range(29999, 29990, -1)) and int(counts[b]) == 9
    # several searches may be outstanding: each is corrected into its OWN outputs by one finish
    outs = [same.search_device(qd, 9, 0.0, defer_check=True) for _ in range(3)]
    assert same.finish_search() == 15
    torch.cuda.synchronize()
    for items, scores, counts in outs:
        for b in range(5):
            assert items[b].tolist() == list(range(29999, 29990, -1)) and int(counts[b]) == 9
    # ... also with different queries per search (ordinary data: nothing flagged, all exact)
    pend = []
    for j in range(4):
        qj = torch.from_numpy(qr[j * 10:(j + 1) * 10]).cuda()
        pend.append((j, base.search_device(qj, 20, 0.0, defer_check=True)))
    assert base.finish_search() == 0
    for j, (items, scores, counts) in pend:
        got = {"items": items[3, : counts[3]].tolist(), "scores": scores[3, : counts[3]].tolist()}
        assert_hits_match(got, O.lookup(vr, qr[j * 10 + 3], 20, 0.0))


@pytest.mark.parametrize("storage,n,d,b,k", [
    ("float16", 30000, 256, 1024 + 37, 100),    # BASELINE configs[3]'s batch: five query chunks in ONE pass
    ("bfloat16", 66000, 128, 700, 32),
])
def test_many_query_chunks_one_pass(storage, n, d, b, k):
    v, q = O.make_corpus(n, d, seed=n + b, n_queries=b)
    vr, qr = O.round_to_storage(v, storage), O.round_to_storage(q, storage)
    base = make_base(v, storage)
    items, scores, counts = base.search_arrays(qr, k, 0.0)
    t = base.last_timing()
    assert t["path"] == "mma" and t["launches"] == 4, t
    assert sum(1 for name, _ in t["kernels"] if name == "main") == 1
    for i in [0, 1, 127, 128, 255, 256, 511, 512, b // 2, b - 2, b - 1]:
        got = {"items": items[i, : counts[i]].tolist(), "scores": scores[i, : counts[i]].tolist()}
        assert_hits_match(got, O.lookup(vr, qr[i], k, 0.0), what=f"{storage} q{i}")


# ------------------------------------------------------------------ float32 index on tensor cores
@pytest.mark.parametrize("n,d,b", [(256, 64, 128), (3001, 136, 130), (700, 1536, 256), (40000, 384, 64),
                                   (3001, 72, 1), (2000, 64, 133 * 128 + 5)])
def test_split_every_dot_product_float32(n, d, b):
    """float32 rows as two fp16 planes (x = hi + lo/2048): every dot vs float64 on the UNROUNDED data."""
    v, q = O.make_corpus(n, d, seed=n + d + 1, n_queries=b)
    base = make_base(v, "float32")
    got = mma_scores(base, q)
    want = q.astype(np.float64) @ v.astype(np.float64).T
    assert (np.abs(got - want) <= dot_error_bound(q, v, split=True)).all()
    np.testing.assert_allclose(got, want, atol=1e-6, rtol=0)
    assert np.abs(got - want).max() < 5e-7


@pytest.mark.parametrize("n,d,b,k,ms", [
    (20000, 768, 64, 32, 0.0),
    (50000, 384, 300, 5, 0.0),       # in-register top-k on the split form
    (30000, 1536, 17, 100, 0.0),
    (20011, 256, 33, 50, 0.52),
    (6000, 128, 200, 10, 0.0),       # no sampling
])
def test_split_search_matches_reference_on_float32_inputs(n, d, b, k, ms):
    """The north-star statement itself: identical float32 inputs, batched, on tensor cores."""
    v, q = O.make_corpus(n, d, seed=n + b + 7, n_queries=b)
    base = make_base(v, "float32", None)
    batch = base.fuzzy_lookup_embeddings(q, max_hits=k, min_score=ms)
    assert base.last_timing()["path"] == "mma_split"
    for i in list(range(min(b, 10))) + [b - 1]:
        assert_hits_match(batch[i], O.lookup(v, q[i], k, ms), min_score=ms, what=f"split q{i}")


def test_split_planes_follow_appends_and_clear():
    v, q = O.make_corpus(30000, 64, seed=3, n_queries=20)
    base = make_base(v[:10000], "float32", None)
    for got, qq in zip(base.fuzzy_lookup_embeddings(q, 10, 0.0), q):
        assert_hits_match(got, O.lookup(v[:10000], qq, 10, 0.0))
    base.add_embeddings(None, v[10000:30000])          # grows past the planes' capacity
    for got, qq in zip(base.fuzzy_lookup_embeddings(q, 10, 0.0), q):
        assert_hits_match(got, O.lookup(v, qq, 10, 0.0))
    base.add_embedding(None, q[3])                      # one more row
    assert base.fuzzy_lookup_embeddings(q, 1, 0.0)[3][0].item == 30000
    base.clear()
    base.add_embeddings(None, v[5000:12000])
    for got, qq in zip(base.fuzzy_lookup_embeddings(q, 10, 0.0), q):
        assert_hits_match(got, O.lookup(v[5000:12000], qq, 10, 0.0))
    assert base.last_timing()["path"] == "mma_split"


def test_split_values_beyond_fp16_range_fall_back_to_the_exact_scan():
    v, q = O.make_corpus(8000, 64, seed=4, n_queries=20)
    v = v.copy()
    v[1234] *= 3.0e5                                     # |x| > 65504: the fp16 planes cannot hold it
    base = make_base(v, "float32", None)
    with np.errstate(over="ignore"):
        for got, qq in zip(base.fuzzy_lookup_embeddings(q, 10, 0.0), q):
            assert_hits_match(got, O.lookup(v, qq, 10, 0.0))
    big_q = q * 1.0e6                                    # queries out of range as well
    ok = make_base(O.make_corpus(8000, 64, seed=4)[0], "float32", None)
    for got, qq in zip(ok.fuzzy_lookup_embeddings(big_q, 10, 0.0), big_q):
        assert_hits_match(got, O.lookup(O.make_corpus(8000, 64, seed=4)[0], qq, 10, 0.0))


# ------------------------------------------------------------------ many query chunks against the exact row scan
@pytest.mark.parametrize("storage,n,d,b,k,ms", [
    ("bfloat16", 30000, 768, 256, 100, 0.0),     # the config-3 shape, two query chunks
    ("float16", 50000, 384, 1000, 5, 0.0),       # eight query chunks (config 5)
    ("bfloat16", 20011, 136, 130, 10, 0.0),      # ragged K (136 = 2 slices + 8) and a ragged last tile
    ("float16", 777, 512, 200, 30, 0.0),         # small corpus: no sampling, most units idle
    ("bfloat16", 40000, 64, 300, 8, 0.55),       # one K slice; threshold from min_score
    ("bfloat16", 33000, 640, 129, 64, 0.0),      # one query past a full chunk
])
def test_queries_in_tensor_memory_form(storage, n, d, b, k, ms):
    """More than 128 queries on 16-bit storage spread over several query chunks of the tensor-core
    kernel; it must agree with the exact row-scan kernels and the oracle, also under a row mask.
    (The name dates from a kernel form that parked the query block in tensor memory; the shapes
    that covered it are kept under the same test ids.)"""
    v, q = O.make_corpus(n, d, seed=n + d + b, n_queries=b)
    vr, qr = O.round_to_storage(v, storage), O.round_to_storage(q, storage)
    ts = make_base(v, storage, "mma")
    ss = make_base(v, storage, "scan")
    a = ts.search_arrays(qr, k, ms)
    c = ss.search_arrays(qr, k, ms)
    assert ts.last_timing()["path"] == "mma" and ss.last_timing()["path"] == "scan"
    np.testing.assert_array_equal(a[2], c[2])
    for i in list(range(0, b, max(1, b // 16))) + [b - 1]:
        got = {"items": a[0][i, : a[2][i]].tolist(), "scores": a[1][i, : a[2][i]].tolist()}
        other = {"items": c[0][i, : c[2][i]].tolist(), "scores": c[1][i, : c[2][i]].tolist()}
        assert_hits_match(got, other, score_tol=2e-6, min_score=ms, what=f"mma vs scan q{i}")
        assert_hits_match(got, O.lookup(vr, qr[i], k, ms), min_score=ms, what=f"mma vs oracle q{i}")
    allowed = np.random.default_rng(1).random(n) < 0.5
    m = ts.search_arrays(qr[:200], k, ms, allowed=allowed)
    for i in (0, 57, min(b, 200) - 1):
        got = {"items": m[0][i, : m[2][i]].tolist(), "scores": m[1][i, : m[2][i]].tolist()}
        assert_hits_match(got, O.lookup(vr, qr[i], k, ms, predicate=lambda r: bool(allowed[r])), min_score=ms)
