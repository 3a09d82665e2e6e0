"""Parity of the CUDA path (through the C ABI, via the Python VectorBase) with the reference.

Three anchors, all on identical float32 inputs:
  1. the committed golden vectors produced by the unmodified reference (tests/golden/);
  2. the reference's own known-answer tests (tests/test_vectorbase.py:148-159, :209-252);
  3. the CPU oracle (oracle/vectorbase_oracle.py) on seeded inputs and edge cases.
Bar: scores within 1e-4 (north_star); index sets identical up to exact-arithmetic ties
(tests/parity.py: a row may differ only if its score is within 2e-6 of the boundary).
In practice float32 paths agree to ~1e-7; the tolerances are the contract, not the result.
"""

from __future__ import annotations

import asyncio
import ctypes as C

import numpy as np
import pytest

import typeagent_py_b200 as tab
from oracle import vectorbase_oracle as O
from tests.golden import cases as GC
from tests.parity import SCORE_TOL, TIE_TOL, assert_hits_match
from typeagent_py_b200 import _capi

pytestmark = pytest.mark.gpu

GOLDEN = GC.load_golden()


def gpu_base(vectors=None, **kw):
    base = tab.VectorBase(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()), **kw)
    if vectors is not None:
        base.add_embeddings(None, vectors)
    return base


# ------------------------------------------------------------------ 1. golden vectors
@pytest.mark.parametrize("case", GC.CASES, ids=[c["name"] for c in GC.CASES])
def test_golden_vectors_fp32_storage(case):
    vectors, queries = GC.build_inputs(case)
    base = gpu_base(vectors)
    recorded = GOLDEN["cases"][case["name"]]
    for (kind, kw), per_query in zip(case["lookups"], recorded):
        for qi, (q, want) in enumerate(zip(queries, per_query)):
            kw2 = dict(kw)
            if kind == "lookup":
                got = base.fuzzy_lookup_embedding(q, **kw2)
            elif kind == "subset":
                subset = GC.build_subset(kw2.pop("subset"))
                got = base.fuzzy_lookup_embedding_in_subset(q, subset, **kw2)
            else:
                pred = GC.PREDICATES[kw2.pop("predicate")]
                got = base.fuzzy_lookup_embedding(q, predicate=pred, **kw2)
            assert all(isinstance(h, tab.ScoredInt) for h in got)
            assert all(isinstance(h.item, int) and isinstance(h.score, float) for h in got)
            assert_hits_match(got, want, score_tol=SCORE_TOL, tie_tol=TIE_TOL,
                              min_score=kw.get("min_score"), what=f"{case['name']}/{kind}/{kw}/q{qi}")
            # float32 arithmetic on both sides: in fact far tighter than the contract
            gs = {h.item: h.score for h in got}
            for item, score in zip(want["items"], want["scores"]):
                if item in gs:
                    assert abs(gs[item] - score) <= 2e-6


@pytest.mark.parametrize("storage", ["bfloat16", "float16"])
def test_golden_vectors_16bit_storage(storage):
    """The bf16 / fp16 golden inputs are exactly representable in the storage dtype, so the
    device copy is loss-free and the reference outputs must be reproduced (row-scan path)."""
    case = next(c for c in GC.CASES if c["make"][1].get("storage") == storage)
    vectors, queries = GC.build_inputs(case)
    base = gpu_base(vectors, storage_dtype=storage)
    base.force_path = "scan"
    for (kind, kw), per_query in zip(case["lookups"], GOLDEN["cases"][case["name"]]):
        batch = base.fuzzy_lookup_embeddings(queries, **kw)
        for got, want in zip(batch, per_query):
            assert_hits_match(got, want, min_score=kw.get("min_score"), what=f"{storage}/{kw}")


# ------------------------------------------------------------------ 2. reference known answers
def test_reference_known_answer_score_scale():
    base = gpu_base()
    base.add_embedding(None, np.array([1.0, 0.0], dtype=np.float32))
    base.add_embedding(None, np.array([0.0, 1.0], dtype=np.float32))
    base.add_embedding(None, np.array([-1.0, 0.0], dtype=np.float32))
    results = base.fuzzy_lookup_embedding(np.array([1.0, 0.0], dtype=np.float32), max_hits=3, min_score=0.0)
    assert [r.item for r in results] == [0, 1, 2]
    assert [r.score for r in results] == [1.0, 0.5, 0.0]


def test_reference_fuzzy_lookup_by_key():
    base = gpu_base()
    for key in ("word1", "word2", "word3"):
        asyncio.run(base.add_key(key))
    results = asyncio.run(base.fuzzy_lookup("word1", max_hits=2, min_score=0.0))
    assert 1 <= len(results) <= 2
    assert results[0].item == 0 and results[0].score > 0.9
    batch = asyncio.run(base.fuzzy_lookup_keys(["word1", "word3"], max_hits=2, min_score=0.0))
    assert batch[0][0].item == 0 and batch[1][0].item == 2


def test_reference_subset_cases():
    base = gpu_base()
    rows = [np.array(v, np.float32) for v in ([0.1, 0.2, 0.3], [0.4, 0.5, 0.6], [0.7, 0.8, 0.9])]
    for r in rows:
        base.add_embedding(None, r)
    q = rows[0]
    assert 0 in [h.item for h in base.fuzzy_lookup_embedding_in_subset(q, [0, 1, 2])]
    one = base.fuzzy_lookup_embedding_in_subset(q, [1])
    assert len(one) == 1 and one[0].item == 1
    assert base.fuzzy_lookup_embedding_in_subset(q, []) == []
    assert gpu_base().fuzzy_lookup_embedding(q) == []


# ------------------------------------------------------------------ 3. oracle, seeded + edges
@pytest.mark.parametrize("n,d,seed", [(1, 4, 1), (31, 3, 2), (32, 8, 3), (33, 20, 4), (1000, 384, 5),
                                       (4097, 768, 6), (20000, 96, 7), (777, 1536, 8), (513, 5, 9)])
def test_random_shapes_match_oracle(n, d, seed):
    v, q = O.make_corpus(n, d, seed, n_queries=3)
    base = gpu_base(v)
    for qq in q:
        for k, ms in ((10, 0.0), (None, None), (1, 0.0), (n + 3, 0.45), (37, 0.5), (0, 0.5)):
            want = O.lookup(v, qq, k, ms)
            got = base.fuzzy_lookup_embedding(qq, max_hits=k, min_score=ms)
            assert_hits_match(got, want, min_score=ms, what=f"n={n} d={d} k={k} ms={ms}")


def test_batched_equals_single_and_oracle():
    v, q = O.make_corpus(6000, 128, 21, n_queries=21)  # 21 -> chunks of 8, 8, 4(+1)
    base = gpu_base(v)
    batch = base.fuzzy_lookup_embeddings(q, max_hits=15, min_score=0.4)
    assert len(batch) == 21
    for qq, got in zip(q, batch):
        assert_hits_match(got, O.lookup(v, qq, 15, 0.4), min_score=0.4)
        # the batch takes the tensor-core form of the float32 index (21 queries, 6000 rows), the
        # single lookup the row scan: two CUDA paths, same float32 inputs
        single = base.fuzzy_lookup_embedding(qq, max_hits=15, min_score=0.4)
        assert_hits_match(single, got, score_tol=2e-6, min_score=0.4)
    base.force_path = "scan"
    for qq, got in zip(q, base.fuzzy_lookup_embeddings(q, max_hits=15, min_score=0.4)):
        single = base.fuzzy_lookup_embedding(qq, max_hits=15, min_score=0.4)
        assert [(h.item, h.score) for h in single] == [(h.item, h.score) for h in got]  # scan: bit-identical
    base.force_path = None
    items, scores, counts = base.search_arrays(q, 15, 0.4)
    assert items.shape == (21, 15) and scores.dtype == np.float32 and counts.dtype == np.int32
    assert np.all(items[np.arange(15)[None, :] >= counts[:, None]] == -1)


def test_subset_duplicates_negatives_and_bounds():
    v, q = O.make_corpus(500, 33, 31)
    base = gpu_base(v)
    subset = [5, 5, 499, -1, 0, -500, 77, 5]
    want = O.lookup_in_subset(v, q[0], subset, 6, 0.0)
    got = base.fuzzy_lookup_embedding_in_subset(q[0], subset, 6, 0.0)
    assert_hits_match(got, want)
    assert sorted(h.item for h in got if h.item in (5, -1, 499)) == sorted(
        h.item for h in want if h.item in (5, -1, 499))
    with pytest.raises(IndexError):
        base.fuzzy_lookup_embedding_in_subset(q[0], [0, 500])
    with pytest.raises(IndexError):
        base.fuzzy_lookup_embedding_in_subset(q[0], [-501])
    big = np.random.default_rng(1).integers(0, 500, size=5000).tolist()
    assert_hits_match(base.fuzzy_lookup_embedding_in_subset(q[0], big, 40, 0.5),
                      O.lookup_in_subset(v, q[0], big, 40, 0.5), min_score=0.5)


def test_predicate_path_matches_oracle_including_order():
    v, q = O.make_corpus(3000, 64, 41)
    base = gpu_base(v)
    for pred in (lambda i: i % 3 == 0, lambda i: i > 2900, lambda i: False, lambda i: True):
        for k, ms in ((10, 0.0), (5, 0.55), (200, 0.5)):
            want = O.lookup(v, q[0], k, ms, predicate=pred)
            got = base.fuzzy_lookup_embedding(q[0], k, ms, predicate=pred)
            assert_hits_match(got, want, min_score=ms)


def test_thresholds_edges():
    v, q = O.make_corpus(2000, 48, 51)
    base = gpu_base(v)
    qq = q[0]
    assert base.fuzzy_lookup_embedding(qq, 10, 1.5) == []
    assert base.fuzzy_lookup_embedding(qq, 10, float("nan")) == []
    assert len(base.fuzzy_lookup_embedding(qq, 10, -3.0)) == 10
    # a threshold exactly equal to an achieved score keeps that row (>=, float32 compare)
    top = base.fuzzy_lookup_embedding(qq, 5, 0.0)
    again = base.fuzzy_lookup_embedding(qq, 50, top[4].score)
    assert [h.item for h in again] == [h.item for h in top]
    # python float vs float32 threshold (NEP 50): 0.85 rounds UP in float32
    row = np.zeros((1, 48), np.float32)
    row[0, 0] = 0.7
    one = gpu_base(np.concatenate([row, v[:10]]))
    e = np.zeros(48, np.float32)
    e[0] = 1.0
    assert O.lookup(np.concatenate([row, v[:10]]), e, 3, 0.85)[0].score == pytest.approx(0.85, abs=1e-7)
    assert [h.item for h in one.fuzzy_lookup_embedding(e, 3, 0.85)] == [
        h.item for h in O.lookup(np.concatenate([row, v[:10]]), e, 3, 0.85)]
    # clipping: un-normalised rows give dots outside [-1, 1]
    scaled = gpu_base(v * 3.0)
    got = scaled.fuzzy_lookup_embedding(qq * 2.0, 2000, 0.0)
    want = O.lookup(v * 3.0, qq * 2.0, 2000, 0.0)
    assert len(got) == len(want) == 2000
    assert sorted(h.score for h in got) == pytest.approx(sorted(h.score for h in want), abs=1e-6)
    assert max(h.score for h in got) <= 1.0 and min(h.score for h in got) >= 0.0


def test_nan_rows_are_never_returned():
    v, q = O.make_corpus(300, 16, 61)
    v = v.copy()
    v[7, 3] = np.nan
    base = gpu_base(v)
    got = base.fuzzy_lookup_embedding(q[0], 300, 0.0)
    with np.errstate(invalid="ignore"):
        want = O.lookup(v, q[0], 300, 0.0)
    assert 7 not in [h.item for h in got] and len(got) == 299 == len(want)


def test_everything_passing_multi_pass_paging():
    """max_hits=0 (reference quirk Q2) returns every passing row, sorted: k = N > 2048 per
    pass exercises the key-bounded 'next page' passes; result must be a permutation."""
    v, q = O.make_corpus(7000, 32, 71)
    base = gpu_base(v)
    got = base.fuzzy_lookup_embedding(q[0], max_hits=0, min_score=0.0)
    want = O.lookup(v, q[0], 0, 0.0)
    assert len(got) == len(want) == 7000
    assert sorted(h.item for h in got) == list(range(7000))
    assert all(a.score >= b.score for a, b in zip(got, got[1:]))
    assert_hits_match(got, want)
    part = base.fuzzy_lookup_embedding(q[0], max_hits=5000, min_score=0.5)
    assert_hits_match(part, O.lookup(v, q[0], 5000, 0.5), min_score=0.5)


def test_equal_scores_are_ordered_by_descending_row_and_deterministic():
    row = O.make_corpus(1, 24, 81)[0]
    v = np.repeat(row, 300, axis=0)  # 300 identical rows: every score ties
    base = gpu_base(v)
    got = base.fuzzy_lookup_embedding(row[0], max_hits=10, min_score=0.0)
    assert [h.item for h in got] == list(range(299, 289, -1))
    assert len({h.score for h in got}) == 1


def test_incremental_append_between_lookups():
    v, q = O.make_corpus(3000, 40, 91)
    base = gpu_base()
    done = 0
    for chunk in (1, 10, 500, 1489, 1000):
        base.add_embeddings(None, v[done:done + chunk])
        done += chunk
        assert_hits_match(base.fuzzy_lookup_embedding(q[0], 8, 0.0), O.lookup(v[:done], q[0], 8, 0.0))
    base.add_embedding(None, q[0])
    assert base.fuzzy_lookup_embedding(q[0], 1, 0.0)[0].item == 3000
    base.clear()
    assert base.fuzzy_lookup_embedding(q[0], 1, 0.0) == []
    base.add_embeddings(None, v[:5])
    assert_hits_match(base.fuzzy_lookup_embedding(q[0], 8, 0.0), O.lookup(v[:5], q[0], 8, 0.0))
    base.deserialize(v[100:200])
    assert_hits_match(base.fuzzy_lookup_embedding(q[0], 8, 0.0), O.lookup(v[100:200], q[0], 8, 0.0))


@pytest.mark.parametrize("storage", ["bfloat16", "float16"])
def test_16bit_storage_scan_matches_oracle_on_rounded_values(storage):
    """Unrounded float32 rows are rounded (RNE) by the convert-on-append kernel; the oracle is
    fed the same rounded values upcast to float32 — identical inputs, float32 accumulate."""
    v, q = O.make_corpus(5000, 264, 101, n_queries=5)
    base = gpu_base(v, storage_dtype=storage)
    base.force_path = "scan"
    vr = O.round_to_storage(v, storage)
    lib = _capi.load()
    back = np.empty((5000, 264), np.float32)
    base.fuzzy_lookup_embedding(q[0])  # forces the upload
    _capi.check(lib.tav_read_rows(base._ix, 0, 5000, back.ctypes.data_as(C.c_void_p), None))
    np.testing.assert_array_equal(back, vr)  # device rounding == oracle rounding, bit for bit
    for qq in q:
        assert_hits_match(base.fuzzy_lookup_embedding(qq, 32, 0.0), O.lookup(vr, qq, 32, 0.0))


def test_normalize_flag_gives_cosine_for_unnormalised_inputs():
    rng = np.random.default_rng(111)
    raw = (rng.standard_normal((2000, 72)) * rng.uniform(0.1, 9, (2000, 1))).astype(np.float32)
    qraw = (rng.standard_normal((3, 72)) * 5).astype(np.float32)
    base = gpu_base(raw, normalize=True)
    unit = raw / np.linalg.norm(raw, axis=1, keepdims=True)
    for qq in qraw:
        want = O.lookup(unit, qq / np.linalg.norm(qq), 12, 0.0)
        got = base.fuzzy_lookup_embedding(qq, 12, 0.0)
        assert_hits_match(got, want, score_tol=1e-5)
    np.testing.assert_array_equal(base.serialize(), raw)  # the host mirror keeps the caller's rows


def test_embedding_index_wrapper_lookups():
    v, q = O.make_corpus(1500, 56, 121, n_queries=4)
    idx = tab.EmbeddingIndex(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()), v)
    assert_hits_match(idx.get_indexes_of_nearest(q[0], 7, 0.3), O.lookup(v, q[0], 7, 0.3), min_score=0.3)
    sub = list(range(0, 1500, 7))
    assert_hits_match(idx.get_indexes_of_nearest_in_subset(q[1], sub, 7, 0.3),
                      O.lookup_in_subset(v, q[1], sub, 7, 0.3), min_score=0.3)
    for got, qq in zip(idx.get_indexes_of_nearest_batch(q, 9, 0.0), q):
        assert_hits_match(got, O.lookup(v, qq, 9, 0.0))


def test_query_shape_errors():
    base = gpu_base(O.make_corpus(10, 8, 1)[0])
    with pytest.raises(ValueError):
        base.fuzzy_lookup_embedding(np.zeros(7, np.float32))
    with pytest.raises(ValueError):
        base.fuzzy_lookup_embedding(np.zeros(8, np.float32), max_hits=-2)
    with pytest.raises(ValueError, match="Expected 2D"):
        base.fuzzy_lookup_embeddings(np.zeros(8, np.float32))


# ------------------------------------------------------------------ sharded merge on one GPU
@pytest.mark.parametrize("world,dyadic", [pytest.param(2, False, id="2"), pytest.param(3, False, id="3"),
                                          pytest.param(8, False, id="8"), pytest.param(3, True, id="3-dyadic_coarse")])
def test_shard_merge_kernel_equals_unsharded(world, dyadic):
    """Split the corpus over `world` indexes on this GPU, search each with its row offset,
    pack as the all-gather would, merge with tav_merge_topk: bit-identical to one index
    (and, on an exact-arithmetic corpus with heavy ties, to tests/exact.py's expectation)."""
    import torch

    from tests.exact import dyadic_corpus, expected_topk, preset
    from typeagent_py_b200.sharded import CudaShardEngine, packed_layout, shard_bounds

    if dyadic:
        v, q, dots = dyadic_corpus(5003, 64, 9, *preset("coarse", 64), seed=131)
    else:
        v, q = O.make_corpus(5003, 64, 131, n_queries=9)
        v = np.concatenate([v, v[:50]])  # exact duplicates across shards -> exact ties
    k, ms = 25, 0.45
    whole = gpu_base(v)
    want_items, want_scores, want_counts = whole.search_arrays(q, k, ms)
    settings = tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel())
    parts = []
    for lo, hi in shard_bounds(len(v), world):
        eng = CudaShardEngine(settings, 0)
        eng.load_rows(v[lo:hi])
        parts.append(eng.search_packed(q, k, ms, lo))
    gathered = torch.stack(parts)
    assert gathered.shape[1] == packed_layout(len(q), k)[2]
    items, scores, counts = eng.merge(gathered, world, len(q), k)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(counts.cpu().numpy(), want_counts)
    for b in range(len(q)):
        c = want_counts[b]
        np.testing.assert_array_equal(items[b, :c].cpu().numpy(), want_items[b, :c])
        np.testing.assert_array_equal(scores[b, :c].cpu().numpy(), want_scores[b, :c])
    if dyadic:
        e_items, e_scores, e_counts = expected_topk(dots, k, ms)
        np.testing.assert_array_equal(counts.cpu().numpy(), e_counts)
        for b, c in enumerate(e_counts):
            np.testing.assert_array_equal(items[b, :c].cpu().numpy(), e_items[b, :c])
            np.testing.assert_array_equal(scores[b, :c].cpu().numpy(), e_scores[b, :c])


def test_device_tensor_handles_and_timing():
    import torch

    v, q = O.make_corpus(9000, 128, 141, n_queries=6)
    t = torch.from_numpy(v).cuda()
    base = tab.VectorBase.from_device_tensor(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()), t)
    base.enable_timing()
    assert len(base) == 9000
    items, scores, counts = base.search_device(torch.from_numpy(q).cuda(), 12, 0.0)
    torch.cuda.synchronize()
    for b, qq in enumerate(q):
        got = {"items": items[b, : counts[b]].tolist(), "scores": scores[b, : counts[b]].tolist()}
        assert_hits_match(got, O.lookup(v, qq, 12, 0.0))
    timing = base.last_timing()
    assert timing["path"] == "scan" and timing["launches"] >= 2 and 0 < timing["scan_ms"] <= timing["total_ms"]
    with pytest.raises(RuntimeError):
        base.add_embedding(None, v[0])
