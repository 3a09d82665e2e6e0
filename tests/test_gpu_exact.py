"""Every search path bit for bit, for every query of the batch (tests/exact.py).

(a) Exact-arithmetic (dyadic) corpora: all paths compute the same float32 dots, so items, scores and
    counts must EQUAL ``expected_topk`` — no tolerance, no sampling of queries.
(b) Random data on the tensor cores: the search must equal ``expected_topk`` of the dots its own kernel
    dumps (``tav_mma_scores``: same template, tiles, K order and split combine), for every query it did
    not flag for the exact redo; the flagged ones, once redone, match float64 within the rigorous
    rounding bound, and so does the dump itself, element by element.

Every parameter id names the branch it covers (regime table).  make_plan (tav_mma.cu), with
target = max(16k, min(2048, max(128, N/4096))) for k > 8 and min(2048, max(32, N/4096)) for k <= 8:
  * sampling only when N > 16384 and 8 * target < N (the clause n_full_tiles < 8 is then implied);
  * sample block 128 rows when target/N * 128 <= 0.7, else 32 rows when target/N * 32 <= 0.7, else 8;
  * candidate segments hold every row a unit sees without sampling (no overflow possible);
  * per_chunk = max(1, SMs / nqc): 1 once nqc = ceil(B / 128) > 132, and the 134 units then queue;
  * batches of more than kMmaMaxQueries = 32768 queries run as slabs of launches.
finalize_kernel: total admitted <= fast_cap (8192 here) -> k <= 512 and total > 256: histogram select,
falling back to the bitonic sort when the boundary bucket holds > 1024 keys (ties); otherwise bitonic;
total > fast_cap -> the streaming k-best list.
Single-launch scan (one host query, k * min(ceil(N/32), 132) <= 8192): merge by rank selection when
k <= 32 and the CTAs' survivors (grid * k, grid <= 2048 / k) are <= 4096; by histogram select when
there are > 256 of them and k <= 512; by the bitonic sort otherwise; completion watched on the result
slots for k <= 64, on a completion word above.  (k between 513 and 1024 cannot pass the fit test: it
would need N >= k rows in <= 8192 / k row tiles of 32.)
"""

from __future__ import annotations

import numpy as np
import pytest

from oracle import vectorbase_oracle as O
from tests.exact import dot_error_bound, dyadic_corpus, expected_topk, preset, scores_of
from tests.parity import assert_hits_match
from tests.test_gpu_mma import make_base, mma_scores

pytestmark = pytest.mark.gpu


def row_mask(kind, n, seed=0):
    if kind is None:
        return None
    r = np.arange(n)
    if kind == "bit0":
        return r % 32 == 0
    if kind == "bit31":
        return r % 32 == 31
    return np.random.default_rng(seed).random(n) < {"half": 0.5, "sparse": 0.01}[kind]


def min_score_for(kind, dots, k):
    """-2 / 0 / 1 / 1.5 / nan, or an unclipped score query 0 achieves (rank ~k/2), or its float32 neighbours;
    "low": a score below 0.25 that query 0 achieves — there (x + 1) is exact, so the dot threshold the
    tensor-core path derives from it is that row's dot itself."""
    s = scores_of(dots[0])
    if kind == "low":
        low = np.sort(s[(s > 0) & (s < 0.25)])
        return float(low[len(low) // 2])
    if kind not in ("hit", "hit+ulp", "hit-ulp"):
        return float(kind)
    hit = np.sort(s[(s > 0) & (s < 1)])[-max(1, k // 2)]
    step = {"hit": None, "hit+ulp": np.float32(2), "hit-ulp": np.float32(-2)}[kind]
    return float(hit if step is None else np.nextafter(hit, step))


def search(base, path, q, k, ms, allowed):
    """The lookup through one API form -> ((items, scores, counts) as numpy arrays, queries redone)."""
    import torch

    if path == "scan1":  # one host query per call: the single-launch form
        out = [base.search_arrays(q[i:i + 1], k, ms, allowed=allowed) for i in range(len(q))]
        return tuple(np.concatenate([o[j] for o in out]) for j in range(3)), 0
    if path in ("device", "defer"):
        res = base.search_device(torch.from_numpy(q).cuda(), k, ms, defer_check=path == "defer", allowed=allowed)
        redone = base.finish_search()
        torch.cuda.synchronize()
        return tuple(t.cpu().numpy() for t in res), redone
    return base.search_arrays(q, k, ms, allowed=allowed), 0


def assert_equal_results(got, want, what):
    gi, gs, gc = got
    wi, ws, wc = want
    bad = np.flatnonzero((gc != wc) | (gi != wi).any(1) | (gs.view(np.uint32) != ws.view(np.uint32)).any(1))
    if len(bad):
        b = bad[0]
        col = np.flatnonzero((gi[b] != wi[b]) | (gs[b] != ws[b]))
        j = col[0] if len(col) else 0
        raise AssertionError(f"{what}: {len(bad)} of {len(gc)} queries differ, first q{b}: count {gc[b]} vs {wc[b]}, "
                             f"at rank {j}: ({gi[b, j]}, {gs[b, j]!r}) vs ({wi[b, j]}, {ws[b, j]!r})")


def assert_boundary_cuts_a_tie(dots, want, k):
    """Some query's k-th score is shared by rows beyond rank k: the order among ties decides."""
    items, scores, counts = want
    for b in range(len(counts)):
        if counts[b] == k:
            s = scores_of(dots[b])
            if (s == scores[b, k - 1]).sum() > (scores[b] == scores[b, k - 1]).sum():
                return
    raise AssertionError("no query's rank-k boundary falls inside a tied group")


# (storage, path, n, d, b, k, min_score, preset, mask)  path: scan1 = single launch, scan2 = scan + select
# kernels, device = general scan on device queries (force scan) or tensor cores (force mma), mma, defer
P = pytest.param
DYADIC = [
    # ---- single-launch scan
    P("bfloat16", "scan1", 16384, 64, 3, 8, "0", "fine", None, id="scan1-rank_select-k8-N16384"),
    P("float16", "scan1", 16385, 56, 2, 32, "hit", "fine", None, id="scan1-rank_select-k32-min_at_score"),
    P("float32", "scan1", 16384, 72, 2, 33, "0", "fine", None, id="scan1-hist_select-k33"),
    P("bfloat16", "scan1", 16384, 64, 2, 33, "0", "coarse", None, id="scan1-hist_select_ties_to_bitonic-k33-coarse"),
    P("float16", "scan1", 4000, 64, 2, 64, "hit+ulp", "fine", None, id="scan1-hist_select-k64-watch_slots-min_ulp_above"),
    P("bfloat16", "scan1", 4000, 136, 2, 65, "hit-ulp", "fine", None, id="scan1-hist_select-k65-completion_word-min_ulp_below"),
    P("bfloat16", "scan1", 255, 8, 2, 64, "-2", "fine", None, id="scan1-bitonic-N255"),
    P("float32", "scan1", 512, 64, 2, 512, "0", "fine", None, id="scan1-hist_select-k512-N512"),
    P("bfloat16", "scan1", 1, 8, 2, 1, "-2", "fine", None, id="scan1-N1"),
    P("bfloat16", "scan1", 16384, 64, 2, 9, "0", "fine", "bit31", id="scan1-rank_select-k9-mask_bit31"),
    P("float16", "scan1", 3000, 64, 2, 40, "1", "coarse", None, id="scan1-min_score_1-clipped_ties"),
    # ---- row scan, several queries
    P("bfloat16", "scan2", 513, 64, 3, 513, "0", "fine", None, id="scan2-k513-N513"),
    P("float16", "scan2", 16384, 64, 17, 1024, "0", "fine", None, id="scan2-k1024"),
    P("bfloat16", "scan2", 16385, 8, 3, 2048, "-2", "fine", None, id="scan2-k2048-one_pass"),
    P("bfloat16", "scan2", 16385, 64, 3, 2049, "0", "fine", "half", id="scan2-k2049-two_passes-mask_half"),
    P("float32", "scan2", 16385, 56, 3, 4097, "-2", "coarse", None, id="scan2-k4097-three_passes-coarse"),
    P("bfloat16", "scan2", 8000, 64, 5, 257, "0", "coarse", None, id="scan2-k257-tie_at_boundary-coarse"),
    P("float16", "device", 16384, 64, 63, 9, "0", "fine", "half", id="scan_device-fused-k9-B63-mask_half"),
    P("bfloat16", "device", 5000, 72, 65, 65, "hit", "fine", None, id="scan_device-scan_select-k65-B65"),
    P("bfloat16", "device", 6000, 64, 17, 256, "0", "coarse", None, id="scan_device-k256-tie_at_boundary-coarse"),
    # ---- tensor cores, no sampling (N <= 16384)
    P("bfloat16", "mma", 16384, 64, 1, 8, "0", "fine", None, id="mma-B1-no_sampling-finalize_stream"),
    P("float16", "mma", 1, 8, 16, 1, "-2", "fine", None, id="mma-N1"),
    P("bfloat16", "mma", 255, 56, 17, 8, "0", "fine", None, id="mma-N255-finalize_bitonic_le256"),
    P("float16", "mma", 256, 64, 64, 32, "-2", "fine", None, id="mma-N256-B64-finalize_bitonic_le256"),
    P("bfloat16", "mma", 257, 72, 65, 64, "0", "fine", None, id="mma-N257-B65-finalize_select"),
    P("bfloat16", "mma", 2047, 136, 127, 65, "0", "fine", None, id="mma-N2047_7_full_tiles_ragged-B127"),
    P("float16", "mma", 2049, 64, 128, 256, "0", "fine", "bit0", id="mma-N2049_8_full_tiles_ragged-B128-mask_bit0"),
    P("bfloat16", "mma", 5000, 64, 129, 512, "0", "fine", None, id="mma-B129-k512-finalize_select"),
    P("float16", "mma", 5000, 64, 33, 513, "0", "fine", None, id="mma-k513-finalize_bitonic"),
    P("bfloat16", "mma", 8192, 64, 40, 256, "0", "coarse", None, id="mma-finalize_select_ties_to_bitonic-coarse"),
    P("bfloat16", "mma", 16384, 64, 20, 1025, "-2", "fine", None, id="mma-k1025-finalize_stream"),
    P("float16", "mma", 16384, 8, 20, 2048, "0", "fine", None, id="mma-k2048-finalize_stream"),
    P("bfloat16", "mma", 3000, 1536, 257, 32, "0", "fine", None, id="mma-D1536-B257-three_chunks"),
    P("float16", "mma", 6000, 64, 30, 20, "1", "coarse", None, id="mma-min_score_1-clipped_ties"),
    P("bfloat16", "mma", 6000, 64, 30, 20, "1.5", "fine", None, id="mma-min_score_above_1"),
    P("bfloat16", "mma", 6000, 64, 30, 20, "nan", "fine", None, id="mma-min_score_nan"),
    P("float32", "mma", 5000, 72, 40, 64, "0", "fine", "half", id="mma_split-no_sampling-mask_half"),
    P("float32", "mma", 4097, 136, 129, 33, "hit", "coarse", None, id="mma_split-B129-coarse"),
    P("bfloat16", "defer", 6000, 64, 64, 100, "0", "coarse", None, id="defer-tie_at_boundary-no_overflow-coarse"),
    P("float16", "mma", 2048, 64, 20, 2048, "low", "fine", None, id="mma-min_score_low-threshold_equals_a_dot"),
    P("bfloat16", "scan2", 3000, 64, 3, 3000, "low", "fine", None, id="scan2-min_score_low"),
    # ---- tensor cores, sampled thresholds
    P("float16", "mma", 16385, 64, 16, 32, "0", "fine", None, id="mma-N16385-sample8"),
    P("bfloat16", "mma", 20000, 72, 17, 16, "hit", "fine", None, id="mma-sample32-min_at_score"),
    P("bfloat16", "mma", 20000, 72, 17, 16, "hit+ulp", "fine", None, id="mma-sample32-min_ulp_above"),
    P("bfloat16", "mma", 20000, 72, 17, 16, "hit-ulp", "fine", None, id="mma-sample32-min_ulp_below"),
    P("float16", "mma", 40000, 136, 65, 9, "0", "fine", None, id="mma-sample128-k9-B65"),
    P("bfloat16", "mma", 40000, 64, 128, 1, "0", "fine", "bit31", id="mma-sample128-k1-B128-mask_bit31"),
    P("bfloat16", "mma", 40000, 64, 129, 8, "0", "fine", "half", id="mma-sample128-k8-B129-mask_half"),
    P("float32", "mma", 20000, 64, 65, 32, "0", "fine", None, id="mma_split-sample8-B65"),
    P("bfloat16", "defer", 30000, 56, 130, 32, "0", "fine", "half", id="defer-sample32-mask_half"),
    # ---- batch shapes
    P("bfloat16", "mma", 2000, 64, 133 * 128 + 5, 8, "0", "fine", None, id="mma-B17029-nqc134_gt_SMs-per_chunk1"),
    P("float16", "mma", 300, 8, 32769, 4, "0", "fine", None, id="mma-B32769-second_slab"),
]


@pytest.mark.parametrize("storage,path,n,d,b,k,ms_kind,pre,mask", DYADIC)
def test_dyadic_corpus_every_path_every_query(request, storage, path, n, d, b, k, ms_kind, pre, mask):
    amp, exp = preset(pre, d)
    v, q, dots = dyadic_corpus(n, d, b, amp, exp, seed=n + d + b + k)
    allowed = row_mask(mask, n, seed=n)
    ms = min_score_for(ms_kind, dots, k)
    k = min(k, n)  # search_arrays' clamp
    base = make_base(v, storage, {"scan1": "scan", "scan2": "scan2", "device": "scan"}.get(path, "mma"))
    want = expected_topk(dots, k, ms, allowed)
    if pre == "coarse" and ms_kind in ("0", "-2") and k < n:
        assert_boundary_cuts_a_tie(dots, want, k)
    got, redone = search(base, path, q, k, ms, allowed)
    assert_equal_results(got, want, f"{path} {storage}")
    if ms_kind == "nan":
        return  # `score >= nan` admits nothing: answered before any kernel runs
    t = base.last_timing()
    if path in ("mma", "defer"):
        sampled = "-sample" in request.node.callspec.id
        slabs = -(-b // 32768)
        assert t["path"] == ("mma_split" if storage == "float32" else "mma"), t
        assert sum(1 for name, _ in t["kernels"] if name == "sample") == int(sampled), t
        # per slab: query prep, [sample], main, finalize; + the fp16 planes of a fresh float32 index
        assert t["launches"] == slabs * (3 + sampled) + (storage == "float32"), t
        if not sampled:
            # the threshold is min_score and every row a unit sees fits its segments, so even a tie cut
            # through thousands of equal scores never overflows: nothing was redone
            assert redone == 0
    else:
        assert t["path"] == "scan", t
        if path == "scan1":
            assert t["launches"] == 1, t
        if path == "scan2":
            n_pass = -(-k // 2048)
            assert t["launches"] % (2 * n_pass) == 0, t  # scan + select per pass and query block


# ------------------------------------------------------------------ (b) random data: the kernel's own dots
def assert_dump_within_bound(dump, q, v, split):
    exact = q.astype(np.float64) @ v.astype(np.float64).T
    nan = np.isnan(exact)
    np.testing.assert_array_equal(np.isnan(dump), nan)
    err = np.where(nan, 0.0, np.abs(dump - exact))
    bound = np.where(nan, 0.0, dot_error_bound(np.nan_to_num(q), np.nan_to_num(v), split=split))
    worst = np.unravel_index(np.argmax(err - bound), err.shape)
    assert (err <= bound).all(), f"dot {worst}: error {err[worst]:.3g} > bound {bound[worst]:.3g}"
    return exact, bound


RANDOM = [
    P("bfloat16", 40000, 128, 200, 32, 0.0, None, id="bf16-sample32-B200"),
    P("float16", 100000, 64, 64, 10, 0.0, None, id="fp16-sample128-k10"),
    P("float32", 20000, 136, 130, 50, 0.0, None, id="split-sample8-B130-D136"),
    P("bfloat16", 6000, 64, 129, 20, 0.0, None, id="bf16-no_sampling-B129"),
    P("bfloat16", 40000, 64, 64, 32, 0.52, None, id="bf16-sample32-min_score_cuts"),
    P("bfloat16", 40000, 128, 130, 32, 0.0, "half", id="bf16-sample32-mask_half"),
    P("float16", 40000, 72, 64, 16, 0.0, "sparse", id="fp16-sample32-mask_0.01"),
    P("bfloat16", 40000, 64, 64, 8, 0.0, "bit0", id="bf16-sample128-mask_bit0"),
    P("float32", 30000, 64, 64, 9, 0.0, "bit31", id="split-sample128-mask_bit31"),
    P("bfloat16", 40000, 64, 129, 32, 0.0, "nan_rows", id="bf16-sample32-nan_rows_in_sampled_tile"),
    P("float32", 40000, 64, 65, 20, 0.0, "nan_rows", id="split-sample32-nan_rows_in_sampled_tile"),
]


@pytest.mark.parametrize("storage,n,d,b,k,ms,mask", RANDOM)
def test_tensor_core_search_equals_top_k_of_its_own_dots(request, storage, n, d, b, k, ms, mask):
    import torch

    v, q = O.make_corpus(n, d, seed=n + d + b + k, n_queries=b)
    allowed = None
    if mask == "nan_rows":
        v = v.copy()
        v[[3, 100, 255]] = np.nan  # tile 0: always a sample tile
    else:
        allowed = row_mask(mask, n, seed=b)
    split = storage == "float32"
    if not split:  # identical inputs for the tensor cores and the exact row-scan redo
        v, q = O.round_to_storage(v, storage), O.round_to_storage(q, storage)
    base = make_base(v, storage, "mma")
    with np.errstate(invalid="ignore"):
        dump = mma_scores(base, q)
        exact, bound = assert_dump_within_bound(dump, q, v, split)
    res = base.search_device(torch.from_numpy(q).cuda(), k, ms, defer_check=True, allowed=allowed)
    torch.cuda.synchronize()
    items, scores, counts = before = tuple(t.cpu().numpy() for t in res)
    t = base.last_timing()
    assert t["path"] == ("mma_split" if split else "mma")
    assert sum(1 for name, _ in t["kernels"] if name == "sample") == int("no_sampling" not in request.node.callspec.id), t
    redone = base.finish_search()
    torch.cuda.synchronize()
    after = tuple(t.cpu().numpy() for t in res)
    want = expected_topk(dump, k, ms, allowed)
    same = (counts == want[2]) & (items == want[0]).all(1) & (scores.view(np.uint32) == want[1].view(np.uint32)).all(1)
    flagged = np.flatnonzero(~same)
    # a query the kernel did not flag is final: top-k of its own dots, bit for bit; a flagged one shows no hits
    assert (counts[flagged] == 0).all() and (items[flagged] == -1).all(), f"q{flagged[:5]} wrong, not flagged"
    assert len(flagged) <= redone
    if allowed is None:  # well-mixed unit-norm rows: the sampled threshold always settles the query
        assert redone == 0, redone
    else:
        assert redone <= b // 10, redone
    with np.errstate(invalid="ignore"):
        ref = expected_topk(exact.astype(np.float32), k, ms, allowed)
    for i in flagged:
        tol = 0.5 * float(np.nanmax(bound[i])) + 2.0 ** -24
        got = {"items": after[0][i, : after[2][i]].tolist(), "scores": after[1][i, : after[2][i]].tolist()}
        wnt = {"items": ref[0][i, : ref[2][i]].tolist(), "scores": ref[1][i, : ref[2][i]].tolist()}
        assert_hits_match(got, wnt, score_tol=tol, tie_tol=tol, min_score=ms, what=f"redone q{i}")
    for j in range(3):  # unflagged queries are untouched by the redo
        np.testing.assert_array_equal(after[j][same], before[j][same])
