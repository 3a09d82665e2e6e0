"""Grouped lookups (``search_groups`` / ``search_range_groups`` / ``tav_*_groups``) bit for bit, every query, no
tolerances.  On dyadic corpora (tests/exact.py) every row's float32 dot is exact, so the expected result is the
numpy statement of the semantics in tests/test_groups_host.py; every result is also checked against the first
occurrence of each group in ``search_range``'s list of the same query.  At 10M rows the expectation is a device
reference built on tests/exact_torch.py."""

from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import typeagent_py_b200 as tab
from oracle import vectorbase_oracle as O
from tests.exact import dyadic_corpus, preset, scores_of
from tests.test_groups_host import first_occurrences, grouped_hits, grouped_topk
from typeagent_py_b200 import _capi

pytestmark = pytest.mark.gpu

SCORERS = [("float32", "scan"), ("bfloat16", "scan"), ("float16", "scan"),
           ("bfloat16", "mma"), ("float16", "mma"), ("float32", "mma")]


def make(v, storage, path):
    base = tab.VectorBase(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()), storage_dtype=storage)
    base.add_embeddings(None, v)
    base.force_path = path
    return base


def layout(kind, n, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "single":
        return np.arange(n)
    if kind in ("runs4", "runs37"):
        return np.arange(n) // int(kind[4:])
    if kind == "random":
        return rng.integers(0, max(1, n // 5), n)
    if kind == "half":  # one group holds half the rows, the rest are singletons
        g = np.arange(n) + 1
        g[rng.permutation(n)[: n // 2]] = 0
        return g
    raise ValueError(kind)


def check_all(base, q, dots, groups, k, ms, allowed=None, ties=False):
    """search_groups and search_range_groups against the oracle and against search_range's first occurrences."""
    scores = scores_of(dots)
    want = grouped_topk(scores, groups, min(k, len(groups)), ms, allowed, ties)
    got = base.search_groups(q, k, groups, ms, allowed=allowed, ties_low_first=ties)
    for a, b in zip(got, want):
        assert np.array_equal(a, b)
    off, g, s, r = base.search_range_groups(q, groups, ms, allowed=allowed, ties_low_first=ties)
    roff, ritems, rscores = base.search_range(q, ms, allowed=allowed, ties_low_first=ties)
    for i in range(len(q)):
        a = None if allowed is None else (allowed[i] if np.ndim(allowed) == 2 else allowed)
        eg, es, er = grouped_hits(scores[i], groups, ms, a, ties)
        sl = slice(off[i], off[i + 1])
        assert np.array_equal(g[sl], eg) and np.array_equal(s[sl].view(np.uint32), es.view(np.uint32))
        assert np.array_equal(r[sl], er)
        fg, fs, fr = first_occurrences(ritems[roff[i]:roff[i + 1]], rscores[roff[i]:roff[i + 1]], groups)
        assert np.array_equal(fg, eg) and np.array_equal(fr, er) and np.array_equal(fs, es)
    return got


@pytest.mark.parametrize("storage,path", SCORERS)
@pytest.mark.parametrize("kind", ["single", "runs4", "runs37", "random", "half"])
def test_layouts_on_every_scorer(storage, path, kind):
    n, d, b = 5000, 64, 24
    amp, exp = preset("fine", d)
    v, q, dots = dyadic_corpus(n, d, b, amp, exp, seed=11)
    base = make(v, storage, path)
    groups = layout(kind, n)
    for k in (1, 8, 100, 2048, int(groups.max()) + 5):
        check_all(base, q, dots, groups, k, 0.0)
    if kind == "single":  # singletons: the grouped search is the plain one, items = rows
        items, scores, counts = base.search_arrays(q, 100, 0.5)
        g, s, r, c = base.search_groups(q, 100, groups, 0.5)
        assert np.array_equal(g, items) and np.array_equal(r, items) and np.array_equal(s, scores)
        assert np.array_equal(c, counts)


@pytest.mark.parametrize("storage,path", SCORERS)
def test_min_score_at_a_leader_and_one_ulp_either_side(storage, path):
    n, d, b = 3000, 128, 20
    amp, exp = preset("fine", d)
    v, q, dots = dyadic_corpus(n, d, b, amp, exp, seed=12)
    base = make(v, storage, path)
    groups = layout("runs37", n)
    lead = grouped_hits(scores_of(dots[0]), groups)[1][10]
    for ms in (lead, np.nextafter(lead, np.float32(2)), np.nextafter(lead, np.float32(-2)), 1.5):
        check_all(base, q, dots, groups, 8, float(ms))  # 1.5: no group has a passing row


@pytest.mark.parametrize("storage,path", [("float32", "scan"), ("bfloat16", "mma")])
def test_heavy_ties_inside_and_across_groups(storage, path):
    n, d, b = 6000, 32, 20
    amp, exp = preset("coarse", d)
    v, q, dots = dyadic_corpus(n, d, b, amp, exp, seed=13)
    base = make(v, storage, path)
    for kind in ("runs4", "random"):
        groups = layout(kind, n)
        for k in (1, 8, 100):
            check_all(base, q, dots, groups, k, 0.0)
            if path == "scan":
                check_all(base, q, dots, groups, k, 0.0, ties=True)


@pytest.mark.parametrize("storage,path", [("float32", "scan"), ("bfloat16", "mma"), ("float32", "mma")])
def test_row_masks_and_per_query_masks(storage, path):
    n, d, b = 4000, 64, 18
    amp, exp = preset("fine", d)
    v, q, dots = dyadic_corpus(n, d, b, amp, exp, seed=14)
    base = make(v, storage, path)
    groups = layout("runs4", n)
    rng = np.random.default_rng(1)
    check_all(base, q, dots, groups, 50, 0.0, allowed=rng.random(n) < 0.3)
    check_all(base, q, dots, groups, 50, 0.0, allowed=rng.random((b, n)) < 0.2)


@pytest.mark.parametrize("path", ["mma", "scan"])
def test_random_unit_rows_equal_first_occurrences(path):
    """Unit Gaussian rows: each scorer's grouped result is the first occurrences of its own search_range (the tensor
    cores and the row scan round the dots differently, so their results are compared on dyadic corpora above)."""
    v, q = O.make_corpus(20000, 128, seed=21, n_queries=64)
    groups = layout("runs37", 20000)
    base = make(v, "bfloat16", path)
    g, s, r, c = base.search_groups(q, 100, groups)
    roff, ritems, rscores = base.search_range(q, 0.0)
    for i in range(len(q)):
        fg, fs, fr = first_occurrences(ritems[roff[i]:roff[i + 1]], rscores[roff[i]:roff[i + 1]], groups)
        assert c[i] == min(100, len(fg))
        assert np.array_equal(g[i], fg[:100]) and np.array_equal(r[i], fr[:100]) and np.array_equal(s[i], fs[:100])


@pytest.mark.parametrize("storage,path", [("bfloat16", "mma"), ("float32", "mma"), ("bfloat16", "scan")])
def test_redo_when_the_best_rows_fill_few_groups(storage, path):
    """100k near-duplicate rows in 50 groups beat every other row: the top rows hold 50 groups, fewer than k, so
    every query is redone by the grouped threshold search.  Integer vectors scaled by 2^-6 keep every dot exact on
    every scorer."""
    rng = np.random.default_rng(5)
    d, n_dup, n_rest, b = 64, 100_000, 20_000, 32
    c = rng.integers(-8, 9, d)
    q = (c + rng.integers(-2, 3, (b, d))).astype(np.float32) * np.float32(2.0 ** -6)
    dup = c + rng.integers(-2, 3, (n_dup, d))
    rest = -c + rng.integers(-2, 3, (n_rest, d))
    v = np.concatenate([dup, rest]).astype(np.float32) * np.float32(2.0 ** -6)
    dots = (q.astype(np.float64) @ v.T.astype(np.float64)).astype(np.float32)  # exact: integers times 2^-12
    groups = np.concatenate([rng.integers(0, 50, n_dup), 50 + np.arange(n_rest)])
    base = make(v, storage, path)
    got = base.search_groups(q, 100, groups)
    assert base.last_redone == b
    for a, w in zip(got, grouped_topk(scores_of(dots), groups, 100)):
        assert np.array_equal(a, w)
    assert (got[3] == 100).all() and (got[0][:, :50] < 50).all()


def test_range_groups_segment_overflow_repass():
    """A capacity hint far below the hits: the collection's re-pass, then the leaders."""
    n, d, b = 30000, 64, 20
    amp, exp = preset("fine", d)
    v, q, dots = dyadic_corpus(n, d, b, amp, exp, seed=15)
    groups = layout("runs4", n)
    for path in ("mma", "scan"):
        base = make(v, "bfloat16", path)
        base._range_hint = 64
        check_all(base, q, dots, groups, 100, 0.0)


def _lib_ix(base):
    return base._ensure_device()


def test_lifecycle_append_remove_overwrite_clear():
    n, d, b = 2000, 32, 17
    amp, exp = preset("fine", d)
    v, q, dots = dyadic_corpus(n + 100, d, b, amp, exp, seed=16)
    base = make(v[:n], "float32", None)
    groups = layout("runs4", n)
    check_all(base, q, dots[:, :n], groups, 20, 0.0)
    lib, ix = _lib_ix(base)
    out = [np.zeros((b, 20), np.int64), np.zeros((b, 20), np.float32), np.zeros((b, 20), np.int64),
           np.zeros(b, np.int32)]
    qp = np.ascontiguousarray(q)

    def raw():
        return lib.tav_search_groups(ix, qp.ctypes.data_as(C.c_void_p), b, 20, C.c_float(0.0), 0,
                                     *[o.ctypes.data_as(C.c_void_p) for o in out], None, None)

    assert raw() == 0
    base.add_embeddings(None, v[n:])  # an append invalidates the map
    lib, ix = _lib_ix(base)
    assert raw() == _capi.TAV_ERR_STATE
    groups2 = layout("runs4", n + 100)
    check_all(base, q, dots, groups2, 20, 0.0)
    base.set_embeddings_at(5, v[n + 1:n + 3])  # an overwrite keeps it
    dots2 = dots.copy()
    dots2[:, 5:7] = dots[:, n + 1:n + 3]
    assert raw() == 0
    check_all(base, q, dots2, groups2, 20, 0.0)
    base.remove_embeddings([0, 7])  # a removal drops it
    assert raw() == _capi.TAV_ERR_STATE
    keep = np.setdiff1d(np.arange(n + 100), [0, 7])
    check_all(base, q, dots2[:, keep], groups2[keep], 20, 0.0)
    assert lib.tav_clear(ix) == 0 and lib.tav_size(ix) == 0
    bad = np.full(lib.tav_size(ix) + 1, -1, np.int32)
    assert lib.tav_set_row_groups(ix, bad.ctypes.data_as(C.c_void_p), len(bad), 0, None) == _capi.TAV_ERR_INVALID


def test_negative_device_group_is_refused_and_the_map_kept():
    import torch

    n, d, b = 1000, 32, 4
    amp, exp = preset("fine", d)
    v, q, dots = dyadic_corpus(n, d, b, amp, exp, seed=17)
    base = make(v, "float32", None)
    groups = torch.arange(n, dtype=torch.int32, device="cuda") // 3
    check_all(base, q, dots, groups.cpu().numpy(), 10, 0.0)
    got = base.search_groups(q, 10, groups)
    assert np.array_equal(got[0], grouped_topk(scores_of(dots), np.arange(n) // 3, 10)[0])
    lib, ix = _lib_ix(base)
    bad = groups.clone()
    bad[n // 2] = -5
    assert lib.tav_set_row_groups(ix, C.c_void_p(bad.data_ptr()), n, 1, None) == _capi.TAV_ERR_INVALID
    out = [np.zeros((b, 10), np.int64), np.zeros((b, 10), np.float32), np.zeros((b, 10), np.int64),
           np.zeros(b, np.int32)]
    qp = np.ascontiguousarray(q)
    assert lib.tav_search_groups(ix, qp.ctypes.data_as(C.c_void_p), b, 10, C.c_float(0.0), 0,
                                 *[o.ctypes.data_as(C.c_void_p) for o in out], None, None) == 0
    assert np.array_equal(out[0], got[0])  # the previous map is still in place


def test_set_row_groups_behind_a_held_stream():
    """A map written on a side stream held by a sleep, set on that stream: the search after it sees the new map."""
    import torch

    n, d, b = 4000, 32, 8
    amp, exp = preset("fine", d)
    v, q, dots = dyadic_corpus(n, d, b, amp, exp, seed=18)
    base = make(v, "float32", None)
    old = np.arange(n) // 2
    check_all(base, q, dots, old, 30, 0.0)
    lib, ix = _lib_ix(base)
    side = torch.cuda.Stream()
    new_host = torch.from_numpy((np.arange(n) // 7).astype(np.int32)).pin_memory()
    dev = torch.empty(n, dtype=torch.int32, device="cuda")
    with torch.cuda.stream(side):
        torch.cuda._sleep(100_000_000)
        dev.copy_(new_host, non_blocking=True)
    assert lib.tav_set_row_groups(ix, C.c_void_p(dev.data_ptr()), n, 1, C.c_void_p(side.cuda_stream)) == 0
    out = [np.zeros((b, 30), np.int64), np.zeros((b, 30), np.float32), np.zeros((b, 30), np.int64),
           np.zeros(b, np.int32)]
    qp = np.ascontiguousarray(q)
    assert lib.tav_search_groups(ix, qp.ctypes.data_as(C.c_void_p), b, 30, C.c_float(0.0), 0,
                                 *[o.ctypes.data_as(C.c_void_p) for o in out], None, None) == 0
    want = grouped_topk(scores_of(dots), np.arange(n) // 7, 30)
    for a, w in zip(out, want):
        assert np.array_equal(a, w)


# ---------------------------------------------------------------------------------------------- 10M x 768 bf16
def grouped_topk_ref(t, qd, exp, groups_t, n_groups, k, chunk=64):
    """Device reference of the grouped top-k: every row's exact key, the largest key per group (scatter amax),
    the k largest group keys."""
    import torch

    from tests import exact_torch as T

    out = []
    for q0 in range(0, len(qd), chunk):
        qs = qd[q0:q0 + chunk]
        best = torch.full((len(qs), n_groups), -1, dtype=torch.int64, device=qd.device)
        for r0, dots in T.dyadic_dots(t, qs, exp):
            keys = T._admitted(dots, r0, 0.0, None, False)
            idx = groups_t[r0:r0 + dots.shape[1]].to(torch.int64)[None, :].expand_as(keys)
            best.scatter_reduce_(1, idx, keys, reduce="amax", include_self=True)
        top = torch.topk(best, k, dim=1).values
        row, s = T._decode(top, False)
        valid = top >= 0
        out.append((torch.where(valid, groups_t[row.clamp(min=0)].to(torch.int64), -1),
                    torch.where(valid, s, torch.zeros_like(s)), torch.where(valid, row, -1),
                    valid.sum(1).to(torch.int32)))
    return [torch.cat([o[j] for o in out]).cpu().numpy() for j in range(4)]


@pytest.mark.parametrize("kind", ["runs8", "random"])
def test_10m_grouped_topk_every_query(kind):
    import torch

    n, d, b, k = 10_000_000, 768, 256, 100
    if torch.cuda.mem_get_info()[0] < n * d * 2 + 16 * (1 << 30):
        pytest.skip("not enough free device memory for the 10M corpus")
    amp, exp = preset("scale", d)
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev).manual_seed(31)
    t = torch.empty((n, d), dtype=torch.bfloat16, device=dev)
    step = (1 << 28) // d
    for r0 in range(0, n, step):
        r1 = min(n, r0 + step)
        t[r0:r1] = torch.randint(-amp, amp + 1, (r1 - r0, d), generator=gen, device=dev, dtype=torch.int16).to(t.dtype)
    t.mul_(2.0 ** -exp)
    qd = torch.randint(-amp, amp + 1, (b, d), generator=gen, device=dev, dtype=torch.int16).float() * 2.0 ** -exp
    n_groups = n // 8
    if kind == "runs8":
        groups_t = torch.arange(n, device=dev, dtype=torch.int32) // 8
    else:
        groups_t = torch.randint(0, n_groups, (n,), generator=gen, device=dev, dtype=torch.int32)
    base = tab.VectorBase.from_device_tensor(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()), t)
    got = base.search_groups(qd.cpu().numpy(), k, groups_t)
    want = grouped_topk_ref(t, qd, exp, groups_t, n_groups, k)
    for a, w in zip(got, want):
        assert np.array_equal(a, w)
    del base, t
    torch.cuda.empty_cache()
