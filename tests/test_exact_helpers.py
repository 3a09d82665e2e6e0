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


# ---------------------------------------------------------------- storage conversion references
def test_bfloat16_and_float16_references_match_torch():
    import torch

    from tests.exact import conversion_edges, round_to

    rng = np.random.default_rng(6)
    edges = np.concatenate(list(conversion_edges().values()))
    x = np.concatenate([edges, -edges, (rng.standard_normal(20000) * np.exp2(rng.integers(-150, 126, 20000)))
                        .astype(np.float32)])
    for dtype, tdtype in (("bfloat16", torch.bfloat16), ("float16", torch.float16)):
        want = torch.from_numpy(x).to(tdtype).to(torch.float32).numpy()
        got = round_to(x, dtype)
        nan = np.isnan(want)
        np.testing.assert_array_equal(np.isnan(got), nan)
        np.testing.assert_array_equal(got[~nan].view(np.uint32), want[~nan].view(np.uint32))  # -0.0 too


def test_conversion_edges_hit_their_cases():
    from tests.exact import conversion_edges, round_to, to_bits16

    e = conversion_edges()
    bf_ties = e["bf16_halfway"][:9]
    up = round_to(bf_ties, "bfloat16")
    # ties go to the even neighbour: last bfloat16 bit of the result is 0
    assert ((up.view(np.uint32) >> 16) & 1 == 0).all() and (up != bf_ties).all()
    h_ties = e["fp16_halfway"][:8]
    r = round_to(h_ties, "float16")
    assert (to_bits16(r, "float16") & 1 == 0).all() and (r != h_ties).all()
    assert round_to(np.float32([65520.0]), "float16")[0] == np.inf
    assert round_to(np.float32([np.nextafter(np.float32(65520), np.float32(0))]), "float16")[0] == 65504
    assert np.isinf(round_to(e["max_finite"][3:4], "bfloat16")).all()  # half a bfloat16 ulp past the max
    assert (round_to(e["rounds_to_zero"][:2], "float16") == 0).all()
    assert round_to(e["rounds_to_zero"][2:3], "float16")[0] == 2.0 ** -24
    assert round_to(np.float32([-2.0 ** -26]), "float16").view(np.uint32)[0] == 0x80000000  # -0.0
    assert round_to(np.float32([2.0 ** -133]), "bfloat16")[0] == 2.0 ** -133


# ---------------------------------------------------------------- normalisation: exact rows and the bound
def test_four_squares():
    from tests.exact import four_squares

    for r in list(range(0, 300)) + [2 * 255 * 255, 130049, 99991]:
        parts = four_squares(r, 255)
        assert sum(p * p for p in parts) == r and max(parts) <= 255
    with pytest.raises(ValueError):
        four_squares(4 * 9 + 1, 3)


@pytest.mark.parametrize("d", [4, 5, 64, 136, 1536])
def test_unit_rows_normalise_exactly(d):
    from oracle import vectorbase_oracle as O
    from tests.exact import unit_rows

    amp = min(255, int(np.sqrt((1 << 24) / d - 1)))
    rows, a, m, e = unit_rows(400, d, amp, seed=d)
    assert ((a * a).sum(1) == 4 ** m).all() and np.abs(a).max() <= amp and m <= 11
    assert e.min() <= -90 and e.max() >= 55  # the scales span [2^-100, 2^64]
    np.testing.assert_array_equal(rows.astype(np.float64), a * np.exp2(e.astype(np.float64))[:, None])
    unit = a.astype(np.float32) * np.float32(2.0 ** -m)
    for storage in ("bfloat16", "float16"):
        np.testing.assert_array_equal(O.round_to_storage(unit, storage), unit)
    # the float32 sum of squares of the raw rows leaves the float32 range at both ends
    with np.errstate(over="ignore", under="ignore"):
        ss = (rows * rows).sum(1, dtype=np.float32)
    assert (ss[e <= -80] < 2.0 ** -126).all() and np.isinf(ss[e >= 64 - 2]).all()


def _normalise_f32(v, scaled=True, order="seq"):
    """The append kernel's arithmetic in numpy float32: power-of-two scaling (exact), sum of squares
    in the given order, sqrt, division."""
    v = np.asarray(v, np.float32)
    with np.errstate(over="ignore", under="ignore", invalid="ignore", divide="ignore"):
        amax = np.abs(v).max(1, keepdims=True)
        shift = np.frexp(amax)[1] if scaled else np.zeros_like(amax, np.int32)
        w = np.ldexp(v, -shift).astype(np.float32)
        sq = w * w
        if order == "seq":
            ss = np.zeros(len(v), np.float32)
            for i in range(v.shape[1]):
                ss = ss + sq[:, i]
        elif order == "reverse":
            ss = np.zeros(len(v), np.float32)
            for i in reversed(range(v.shape[1])):
                ss = ss + sq[:, i]
        else:
            ss = sq.sum(1, dtype=np.float32)  # numpy's pairwise order
        nrm = np.sqrt(ss)[:, None]
        return np.where(nrm > 0, w / nrm, v).astype(np.float32)


@pytest.mark.parametrize("storage", ["float32", "bfloat16", "float16"])
def test_normalize_error_bound_covers_the_kernel_arithmetic(storage):
    from tests.exact import normalize_error_bound, round_to

    rng = np.random.default_rng(8)
    for d in (1, 7, 64, 1536):
        n = 200
        v = rng.standard_normal((n, d)) * np.exp2(rng.integers(-140, 101, (n, 1)))
        v *= np.where(rng.random((n, d)) < 0.2, 2.0 ** -60, 1.0)
        v = v.astype(np.float32)
        v = v[np.abs(v).max(1) > 0]
        vv = v.astype(np.float64)
        exact = vv / np.sqrt((vv * vv).sum(1, keepdims=True))
        bound = normalize_error_bound(v, storage)
        for order in ("seq", "reverse", "pairwise"):
            got = round_to(_normalise_f32(v, True, order), storage).astype(np.float64)
            assert (np.abs(got - exact) <= bound).all(), (d, order)
        # not vacuous: a few float32 ulps (plus the storage rounding)
        u_s = {"float32": 0.0, "bfloat16": 2.0 ** -8, "float16": 2.0 ** -11}[storage]
        assert (bound <= (d + 8) * 2.0 ** -24 * np.abs(exact) + u_s * np.abs(exact) * 1.01 + 2.0 ** -25 + 2.0 ** -140).all()
        # unscaled arithmetic breaks the bound on rows whose squares leave the float32 range
        tiny_or_huge = np.abs(v).max(1) < 1e-20
        if tiny_or_huge.any():
            got = round_to(_normalise_f32(v[tiny_or_huge], False), storage).astype(np.float64)
            assert (np.abs(got - exact[tiny_or_huge]) > bound[tiny_or_huge]).any()


def test_normalize_error_bound_zero_rows():
    from tests.exact import normalize_error_bound

    b = normalize_error_bound(np.zeros((2, 5), np.float32), "bfloat16")
    assert (b < 2.0 ** -100).all()
