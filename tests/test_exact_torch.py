"""The torch reference (tests/exact_torch.py) against the numpy expectations, bit for bit (CPU only):
``exact.expected_topk``, ``test_gpu_range.expected_range`` and ``test_gpu_subsets.exact_subset_topk``."""

from __future__ import annotations

import numpy as np
import pytest

torch = pytest.importorskip("torch")

from tests import exact_torch as T  # noqa: E402
from tests.exact import dyadic_corpus, expected_topk, preset, scores_of  # noqa: E402
from tests.test_gpu_range import expected_range  # noqa: E402
from tests.test_gpu_subsets import exact_subset_topk  # noqa: E402


def blocks_of(dots, rows):
    """A [B, N] dots matrix as a source of row blocks of `rows` (a block boundary inside tied groups)."""
    t = torch.from_numpy(np.ascontiguousarray(dots, np.float32))
    return [(r0, t[:, r0:r0 + rows]) for r0 in range(0, t.shape[1], rows)]


def assert_bits(got, want, what):
    got = got.cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got)
    want = np.asarray(want)
    if want.dtype == np.float32:
        got, want = got.view(np.uint32), want.view(np.uint32)
    assert got.shape == want.shape, f"{what}: shapes {got.shape} vs {want.shape}"
    bad = np.argwhere(got != want)
    assert len(bad) == 0, f"{what}: {len(bad)} differ, first at {bad[0]}: {got[tuple(bad[0])]} vs {want[tuple(bad[0])]}"


def tied_dots(b, n, seed):
    """Heavy ties, clipped scores on both sides, NaN rows, and one query of distinct scores."""
    rng = np.random.default_rng(seed)
    dots = rng.choice(np.float32([-1.5, -1, -0.25, 0, 0.5, 0.75, 1, 2.5]), size=(b, n))
    dots[1, ::3] = np.nan
    dots[2] = rng.standard_normal(n).astype(np.float32) * np.float32(0.4)
    return dots


def min_scores(dots):
    s = scores_of(dots[2])
    s = np.sort(s[~np.isnan(s)])
    hit = np.float32(s[-min(7, len(s))])
    return [-2.0, 0.0, 0.5, 1.0, 1.5, float("nan"), float(hit), float(np.nextafter(hit, np.float32(2))),
            float(np.nextafter(hit, np.float32(-1)))]


@pytest.mark.parametrize("n,k,rows", [(1, 1, 1), (40, 40, 7), (40, 64, 16), (300, 17, 13), (300, 17, 300),
                                      (1000, 257, 64)])
def test_topk_equals_expected_topk(n, k, rows):
    dots = tied_dots(5, n, seed=n + k)
    allowed = np.random.default_rng(k).random(n) < 0.6
    for ms in min_scores(dots):
        for mask, off in ((None, 0), (allowed, 1000), (None, (1 << 32) + 5)):
            got = T.topk_ref(blocks_of(dots, rows), k, ms, None if mask is None else torch.from_numpy(mask),
                             item_offset=off)
            want = expected_topk(dots, k, ms, mask, item_offset=off)
            for j, what in enumerate(("items", "scores", "counts")):
                assert_bits(got[j], want[j], f"n={n} k={k} ms={ms!r} offset={off} {what}")


def test_per_query_masks_and_ties_low_equal_the_range_head():
    """Per-query masks: each row equals the shared-mask search of its own mask; ties-low top-k is the head of
    the ties-low threshold list."""
    b, n, k = 6, 500, 40
    dots = tied_dots(b, n, seed=7)
    rng = np.random.default_rng(8)
    masks = rng.random((b, n)) < np.array([1.0, 0.5, 0.1, 0.01, 0.0, 0.9])[:, None]
    for ms in min_scores(dots):
        for ties_low in (False, True):
            got = T.topk_ref(blocks_of(dots, 37), k, ms, torch.from_numpy(masks), ties_low=ties_low, item_offset=3)
            for q in range(b):
                wo, wi, ws = expected_range(dots[q:q + 1], ms, masks[q], ties_low, item_offset=3)
                c = min(k, len(wi))
                assert int(got[2][q]) == c
                assert_bits(got[0][q, :c], wi[:c], f"q{q} items ms={ms!r} ties_low={ties_low}")
                assert_bits(got[1][q, :c], ws[:c], f"q{q} scores")
                assert (got[0][q, c:] == -1).all() and (got[1][q, c:] == 0).all()
            if not ties_low:
                want = expected_topk(dots[1:2], k, ms, masks[1], item_offset=3)
                for j in range(3):
                    assert_bits(got[j][1:2], want[j], "per-query mask vs expected_topk")


@pytest.mark.parametrize("rows", [1, 9, 250, 1000])
def test_range_equals_expected_range(rows):
    dots = tied_dots(4, 250, seed=rows)
    allowed = np.random.default_rng(rows).random(250) < 0.5
    for ms in min_scores(dots):
        for ties_low in (False, True):
            for mask, off in ((None, 0), (allowed, (1 << 32) + 5)):
                got = T.range_ref(blocks_of(dots, rows), ms, None if mask is None else torch.from_numpy(mask),
                                  ties_low, item_offset=off)
                want = expected_range(dots, ms, mask, ties_low, item_offset=off)
                for j, what in enumerate(("offsets", "items", "scores")):
                    assert_bits(got[j], want[j], f"rows={rows} ms={ms!r} ties_low={ties_low} {what}")


def test_subsets_equal_the_one_query_order():
    n, b = 300, 5
    dots = tied_dots(b, n, seed=11)
    rng = np.random.default_rng(12)
    subsets = [np.empty(0, np.int64), rng.integers(-n, n, size=700), np.array([5, 5, -1, n - 1, 0, -n, 5]),
               np.full(50, 17), rng.integers(-n, n, size=129)]
    offsets = np.zeros(b + 1, np.int64)
    offsets[1:] = np.cumsum([len(s) for s in subsets])
    ordinals = np.concatenate(subsets).astype(np.int64)
    td = torch.from_numpy(dots)
    o_t, ord_t = torch.from_numpy(offsets), torch.from_numpy(ordinals)
    q_of = np.searchsorted(offsets, np.arange(len(ordinals)), side="right") - 1
    flat = dots[q_of, ordinals % n]
    for ms in min_scores(dots):
        for ties_low in (False, True):
            for k in (1, 10, 700):
                for step in (1, 64, 10_000):
                    src = [(j0, torch.from_numpy(flat[j0:j0 + step])) for j0 in range(0, len(flat), step)]
                    got_k, got_r = T.subsets_ref(src, o_t, ord_t, k, ms, ties_low)
                    want_k, want_r = exact_subset_topk(dots, subsets, k, ms, ties_low)
                    tag = f"ms={ms!r} ties_low={ties_low} k={k} step={step}"
                    for j in range(3):
                        assert_bits(got_k[j], want_k[j], tag + " top-k")
                        assert_bits(got_r[j], want_r[j], tag + " range")
    # the flat entry dots of a dyadic corpus, as subset_dots computes them
    amp, exp = preset("scale", 64)
    v, q, d = dyadic_corpus(n, 64, b, amp, exp, seed=13)
    got = torch.cat([x for _, x in T.subset_dots(torch.from_numpy(v).to(torch.bfloat16), torch.from_numpy(q), exp,
                                                   o_t, ord_t, block_entries=100)])
    assert_bits(got, d[q_of, ordinals % n], "subset_dots")


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("d,pre", [(64, "scale"), (768, "scale"), (136, "fine"), (56, "coarse")])
def test_dyadic_dots_are_the_exact_dots(dtype, d, pre):
    amp, exp = preset(pre, d)
    v, q, dots = dyadic_corpus(1000, d, 7, amp, exp, seed=d)
    blocks = list(T.dyadic_dots(torch.from_numpy(v).to(dtype), torch.from_numpy(q), exp, block_rows=333))
    assert [r0 for r0, _ in blocks] == [0, 333, 666, 999]
    assert_bits(torch.cat([x for _, x in blocks], dim=1), dots, "dots")
    want = expected_topk(dots, 50, 0.0)
    got = T.topk_ref(blocks, 50, 0.0)
    for j in range(3):
        assert_bits(got[j], want[j], "top-k of the dyadic dots")


def test_dyadic_dots_refuses_inexact_inputs():
    v = torch.full((4, 8), 0.3)
    with pytest.raises(AssertionError, match="dyadic"):
        list(T.dyadic_dots(v, torch.ones((1, 8)), 10))
    big = torch.full((2, 300), 255.0)  # dots of 300 * 255^2 >= 2^24: no longer exact in float32
    with pytest.raises(AssertionError, match="float32"):
        list(T.dyadic_dots(big, big, 0))
