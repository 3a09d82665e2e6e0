"""The exact-expectation helpers of tests/exact.py against brute force (CPU only)."""

from __future__ import annotations

import numpy as np
import pytest

from tests.exact import dot_error_bound, dyadic_corpus, expected_topk, preset, scores_of


def brute_topk(dots, k, min_score, allowed=None):
    """One query at a time, a Python sort of (score, row) pairs."""
    floor = np.float32(min_score)
    out = []
    for x in np.asarray(dots, np.float32):
        s = scores_of(x)
        keep = [(float(s[r]), r) for r in range(len(x))
                if not np.isnan(s[r]) and s[r] >= floor and (allowed is None or allowed[r])]
        keep.sort(reverse=True)
        out.append(keep[:k])
    return out


def assert_same_as_brute(dots, k, min_score, allowed=None, item_offset=0):
    items, scores, counts = expected_topk(dots, k, min_score, allowed, item_offset)
    assert items.shape == scores.shape == (len(dots), k) and counts.shape == (len(dots),)
    for b, want in enumerate(brute_topk(dots, k, min_score, allowed)):
        c = len(want)
        assert counts[b] == c
        assert items[b, :c].tolist() == [r + item_offset for _, r in want]
        assert scores[b, :c].tolist() == [s for s, _ in want]
        assert (items[b, c:] == -1).all() and (scores[b, c:] == 0).all()


@pytest.mark.parametrize("n,k", [(1, 1), (7, 3), (40, 40), (40, 64), (300, 17)])
def test_expected_topk_matches_brute_force(n, k):
    rng = np.random.default_rng(n + k)
    dots = rng.choice(np.float32([-1.5, -1, -0.25, 0, 0.5, 0.75, 1, 2.5]), size=(5, n))  # ties + clipping
    dots[1, ::3] = np.nan
    dots[2] = rng.standard_normal(n).astype(np.float32)
    allowed = rng.random(n) < 0.6
    for ms in (-2.0, 0.0, 0.5, 1.0, 1.5, float("nan")):
        assert_same_as_brute(dots, k, ms)
        assert_same_as_brute(dots, k, ms, allowed, item_offset=1000)


def test_min_score_at_and_one_ulp_around_an_achieved_score():
    dots = np.random.default_rng(3).standard_normal((3, 200)).astype(np.float32) * np.float32(0.4)
    s = scores_of(dots[0])
    hit = np.sort(s)[-20]
    for ms in (hit, np.nextafter(hit, np.float32(2)), np.nextafter(hit, np.float32(-2))):
        assert_same_as_brute(dots, 50, float(ms))
    at = expected_topk(dots, 50, float(hit))[2][0]
    above = expected_topk(dots, 50, float(np.nextafter(hit, np.float32(2))))[2][0]
    assert at == (s >= hit).sum() and above == at - (s == hit).sum()


def test_ties_order_by_descending_row():
    dots = np.zeros((1, 10), np.float32)
    dots[0, [2, 5, 7]] = 0.5
    items, scores, counts = expected_topk(dots, 4, 0.0)
    assert items[0].tolist() == [7, 5, 2, 9] and counts[0] == 4


def test_blocks_of_queries_agree_with_one_block():
    import tests.exact as E

    dots = np.random.default_rng(4).standard_normal((37, 500)).astype(np.float32)
    whole = expected_topk(dots, 9, 0.3)
    saved = E._BLOCK_ELEMS
    try:
        E._BLOCK_ELEMS = 3 * 500  # three queries per block
        parts = expected_topk(dots, 9, 0.3)
    finally:
        E._BLOCK_ELEMS = saved
    for a, b in zip(whole, parts):
        np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("name", ["fine", "coarse"])
@pytest.mark.parametrize("d", [8, 56, 64, 72, 136, 1536])
def test_dyadic_dots_are_exact_in_float32(name, d):
    amp, exp = preset(name, d)
    assert d * amp * amp < 1 << 24
    v, q, dots = dyadic_corpus(300, d, 7, amp, exp, seed=d, dup=[(299, 3)])
    np.testing.assert_array_equal(v[299], v[3])
    # numpy's own float32 GEMV (blocked, any order) and a float64 product give the exact dots
    np.testing.assert_array_equal(v @ q[0], dots[0])
    np.testing.assert_array_equal((q.astype(np.float64) @ v.T.astype(np.float64)).astype(np.float32), dots)
    # the values survive bfloat16 / float16 rounding, and the fp16 split has lo = 0
    from oracle import vectorbase_oracle as O

    for storage in ("bfloat16", "float16"):
        np.testing.assert_array_equal(O.round_to_storage(v, storage), v)
        np.testing.assert_array_equal(O.round_to_storage(q, storage), q)
    s = scores_of(dots)
    if name == "coarse":  # heavy ties, both clipped tails present
        assert (s == 1).any() and (s == 0).any() and len(np.unique(s)) <= min(s.size // 4, 2 ** (2 * exp + 1) + 1)
    else:
        assert 0.01 < np.abs(dots).mean() < 1 and len(np.unique(s)) > s.size // 2


def test_dyadic_corpus_refuses_inexact_widths():
    with pytest.raises(AssertionError):
        dyadic_corpus(4, 1024, 1, 255, 10, seed=0)


def test_dot_error_bound_covers_float32_accumulation():
    rng = np.random.default_rng(5)
    for d in (8, 136, 1536):
        v = rng.standard_normal((50, d)).astype(np.float32)
        q = rng.standard_normal((3, d)).astype(np.float32)
        exact = q.astype(np.float64) @ v.astype(np.float64).T
        naive = np.zeros((3, 50), np.float32)
        for i in range(d):  # sequential float32 sums: the worst ordinary order
            naive += q[:, i:i + 1] * v[:, i][None, :]
        assert (np.abs(naive - exact) <= dot_error_bound(q, v)).all()
        assert (dot_error_bound(q, v) <= dot_error_bound(q, v, split=True)).all()
