"""Sharded filtered and subset lookups on the GPU, bit for bit on dyadic corpora (tests/exact.py) with heavy ties
(identical rows in different row blocks):

(a) W in {1, 2, 3, 8} row blocks of one corpus on one GPU, each a ``CudaShardEngine`` driven through its own
    per-rank steps (``search_subset_packed``, ``search_rows_packed``, ``range_local`` with a subset), the packed
    buffers stacked as the all-gather produces them, merged (``merge_ordered`` / ``merge_range``) and decoded
    (``map_items``): equal to one ``VectorBase`` over the whole corpus for every query;
(b) ``ShardedVectorBase`` with one rank equal to ``VectorBase`` for every new method;
(c) the argument errors of TAV_ITEMS_AS_POSITIONS, ``tav_merge_topk_ordered`` and ``tav_map_items``;
(d) deliberately broken builds (``TAV_SHARDED_FILTER_MUTANT``), each caught by (a)'s checks.
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

from oracle import vectorbase_oracle as O
from tests.exact import dyadic_corpus, preset
from typeagent_py_b200 import _capi

pytestmark = pytest.mark.gpu

N, D = 6000, 64


def blocks(n, w):
    per = -(-n // w)
    return [(min(g * per, n), min((g + 1) * per, n)) for g in range(w)]


def settings():
    import typeagent_py_b200 as tab

    return tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel())


def corpus(b, seed, pre="coarse"):
    """Rows of the first 600 copied to [1500, 2100) and [3000, 3600): equal scores in different blocks for
    every W here."""
    amp, exp = preset(pre, D)
    dup = [(1500 + j, j) for j in range(0, 600, 2)] + [(3000 + j, j) for j in range(1, 600, 2)]
    v, q, _ = dyadic_corpus(N, D, b, amp, exp, seed=seed, dup=dup)
    return v, q


def subset_of(seed, m=2600):
    """Unsorted, with duplicates that straddle blocks (the copied rows and their originals) and negatives."""
    rng = np.random.default_rng(seed)
    perm = rng.permutation(N)
    sub = np.concatenate([perm[:m], perm[:200], np.arange(0, 600, 7), 1500 + np.arange(0, 600, 7),
                          -(perm[:100] + 1), [0, N - 1, -1, -N]])
    rng.shuffle(sub)
    return sub.astype(np.int64)


def engines_for(v, w, storage):
    from typeagent_py_b200.sharded import CudaShardEngine

    out = []
    for lo, hi in blocks(len(v), w):
        eng = CudaShardEngine(settings(), 0, storage)
        eng.load_rows(v[lo:hi] if hi > lo else None)
        out.append(eng)
    return out


def whole(v, storage):
    import typeagent_py_b200 as tab

    one = tab.VectorBase(settings(), storage_dtype=storage)
    one.add_embeddings(None, v)
    return one


def subset_topk(engines, n, q, k, ms, sub, ties_low):
    import torch

    from typeagent_py_b200.sharded import subset_share

    parts = []
    for eng, (lo, hi) in zip(engines, blocks(n, len(engines))):
        pos, local = subset_share(sub, n, lo, hi)
        parts.append(eng.search_subset_packed(q, k, ms, local, pos, ties_low))
    items, scores, counts = engines[0].merge_ordered(torch.stack(parts), len(engines), len(q), k, 3 if ties_low else 2)
    engines[0].map_items(items, sub)
    return items.cpu().numpy(), scores.cpu().numpy(), counts.cpu().numpy()


def masked_topk(engines, n, q, k, ms, allowed, ties_low):
    import torch

    from typeagent_py_b200.sharded import block_mask

    parts = []
    for g, (eng, (lo, hi)) in enumerate(zip(engines, blocks(n, len(engines)))):
        parts.append(eng.search_rows_packed(q, k, ms, lo, ties_low, block_mask(allowed, n, lo, hi),
                                            ("test", id(allowed), g), allowed))
    items, scores, counts = engines[0].merge_ordered(torch.stack(parts), len(engines), len(q), k, 1 if ties_low else 0)
    return items.cpu().numpy(), scores.cpu().numpy(), counts.cpu().numpy()


def subset_range(engines, n, q, ms, sub, ties_low):
    import torch

    from typeagent_py_b200.sharded import offsets_with_status, pack_range_payload, range_pad, subset_share

    locals_ = []
    for eng, (lo, hi) in zip(engines, blocks(n, len(engines))):
        pos, local = subset_share(sub, n, lo, hi)
        locals_.append(eng.range_local(q, ms, lo, ties_low, subset=local, positions=pos))
    dev = engines[0].comm_device()
    offsets_all = torch.from_numpy(np.stack([offsets_with_status(loc.offsets, False) for loc in locals_])).to(dev)
    totals = [int(loc.offsets[-1]) for loc in locals_]
    t_pad = max(range_pad(totals), 2)
    payload = torch.stack([pack_range_payload(loc, t_pad, dev) for loc in locals_])
    o, i, s = engines[0].merge_range(offsets_all, payload, len(engines), len(q), t_pad, sum(totals), ties_low)
    engines[0].map_items(i, sub)
    return o.cpu().numpy(), i.cpu().numpy(), s.cpu().numpy()


def assert_same(got, want, what):
    for g, w, name in zip(got, want, ("items/offsets", "scores/items", "counts/scores")):
        g, w = np.asarray(g), np.asarray(w)
        if g.dtype == np.float32:
            g, w = g.view(np.uint32), w.view(np.uint32)
        np.testing.assert_array_equal(g, w, err_msg=f"{what}: {name}")


P = pytest.param
# (W, storage, B, k, ties_low)
SUBSET_CASES = [
    P(1, "float32", 1, 50, False, id="W1-f32-single-k50"),
    P(2, "bfloat16", 1, 100, True, id="W2-bf16-single-k100-ties_low"),
    P(3, "float16", 1, 50, False, id="W3-fp16-single-k50"),
    P(8, "float32", 1, 100, False, id="W8-f32-single-k100"),
    P(3, "float32", 5, 50, True, id="W3-f32-B5-k50-ties_low"),
    P(8, "bfloat16", 5, 2100, False, id="W8-bf16-B5-k2100"),
    P(2, "float16", 3, 2000, True, id="W2-fp16-B3-k2000-ties_low"),
    P(1, "bfloat16", 9, 100, False, id="W1-bf16-B9-k100"),
]


@pytest.mark.parametrize("w,storage,b,k,ties_low", SUBSET_CASES)
def test_subset_topk_equals_whole_corpus(w, storage, b, k, ties_low):
    v, q = corpus(b, seed=w * 10 + b)
    sub = subset_of(seed=k + w)
    one = whole(v, storage)
    engines = engines_for(v, w, storage)
    for ms in (0.0, 0.55):
        want = one.search_arrays(q, k, ms, subset=sub, ties_low_first=ties_low)
        assert_same(subset_topk(engines, N, q, k, ms, sub, ties_low), want, f"W={w} {storage} ms={ms}")
    # min_score exactly at a hit (the 10th of query 0)
    at = float(one.search_arrays(q[:1], 10, 0.0, subset=sub)[1][0, 9])
    assert_same(subset_topk(engines, N, q, k, at, sub, ties_low),
                one.search_arrays(q, k, at, subset=sub, ties_low_first=ties_low), f"W={w} at a hit")
    if b == 1 and k <= 1024:  # the single-launch form served every rank with a share
        assert all(e.base.last_timing()["launches"] == 1 for e in engines if e.n_local())


@pytest.mark.parametrize("w,storage,b,k", [(1, "float32", 4, 50), (2, "bfloat16", 20, 100), (3, "float16", 1, 64),
                                           (8, "float32", 6, 2100), (3, "bfloat16", 17, 10)])
@pytest.mark.parametrize("ties_low", [False, True], ids=["ties_high", "ties_low"])
def test_masked_topk_equals_whole_corpus(w, storage, b, k, ties_low):
    v, q = corpus(b, seed=7 * w + b)
    rng = np.random.default_rng(w + k)
    allowed = rng.random(N) < 0.45
    allowed[:600] = True
    allowed[1500:2100] = True
    one = whole(v, storage)
    engines = engines_for(v, w, storage)
    for ms in (0.0, 0.6):
        want = one.search_arrays(q, k, ms, allowed=allowed, ties_low_first=ties_low)
        assert_same(masked_topk(engines, N, q, k, ms, allowed, ties_low), want, f"W={w} {storage} ms={ms}")


@pytest.mark.parametrize("w,storage,b", [(1, "float32", 3), (3, "bfloat16", 4), (8, "float16", 2)])
@pytest.mark.parametrize("ties_low", [False, True], ids=["ties_high", "ties_low"])
def test_subset_range_equals_whole_corpus(w, storage, b, ties_low):
    v, q = corpus(b, seed=3 * w + b)
    sub = subset_of(seed=w, m=4000)
    one = whole(v, storage)
    engines = engines_for(v, w, storage)
    for ms in (0.0, 0.5):
        want = one.search_range(q, ms, subset=sub, ties_low_first=ties_low)
        assert_same(subset_range(engines, N, q, ms, sub, ties_low), want, f"W={w} {storage} range ms={ms}")


# ---------------------------------------------------------------- (b) one rank
@pytest.fixture(scope="module")
def one_rank_group():
    import socket

    import torch.distributed as dist

    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    dist.init_process_group("gloo", rank=0, world_size=1, init_method=f"tcp://127.0.0.1:{port}")
    yield
    dist.destroy_process_group()


@pytest.mark.parametrize("storage", ["float32", "bfloat16"])
def test_sharded_one_rank_equals_vectorbase(one_rank_group, storage):
    from typeagent_py_b200.sharded import ShardedVectorBase

    v, q = corpus(20, seed=41)
    one = whole(v, storage)
    sh = ShardedVectorBase(settings(), device=0, storage_dtype=storage)
    sh.deserialize(v)
    sub = subset_of(seed=9)
    rng = np.random.default_rng(2)
    allowed = rng.random(N) < 0.3
    words = one.pack_row_mask(allowed)
    pred = lambda i: bool(allowed[i])  # noqa: E731
    for ms in (0.0, 0.6):
        for tl in (False, True):
            for k in (10, 100):
                assert_same(sh.search_arrays(q, k, ms, subset=sub, ties_low_first=tl),
                            one.search_arrays(q, k, ms, subset=sub, ties_low_first=tl), f"subset {ms} {tl} {k}")
                for mask in (allowed, words):
                    assert_same(sh.search_arrays(q, k, ms, allowed=mask, ties_low_first=tl),
                                one.search_arrays(q, k, ms, allowed=mask, ties_low_first=tl), f"mask {ms} {tl} {k}")
            assert_same(sh.search_range(q, ms, ties_low_first=tl, subset=sub),
                        one.search_range(q, ms, subset=sub, ties_low_first=tl), f"range subset {ms} {tl}")
            assert_same(sh.search_range(q, ms, ties_low_first=tl, allowed=allowed),
                        one.search_range(q, ms, allowed=allowed, ties_low_first=tl), f"range mask {ms} {tl}")
        for mh in (None, 5, 0):
            assert sh.fuzzy_lookup_embedding(q[1], mh, ms, predicate=pred) == \
                one.fuzzy_lookup_embedding(q[1], mh, ms, predicate=pred)
            assert sh.fuzzy_lookup_embedding_in_subset(q[2], sub.tolist(), mh, ms) == \
                one.fuzzy_lookup_embedding_in_subset(q[2], sub.tolist(), mh, ms)
    # an unchanged mask object reaches the device once while the rows stay as they are
    lib = _capi.load()
    real_upload, uploads = lib.tav_set_row_mask, []
    lib.tav_set_row_mask = lambda *a: uploads.append(a[2]) or real_upload(*a)
    try:
        fresh = allowed.copy()
        for k in (3, 7):
            assert_same(sh.search_arrays(q, k, 0.0, allowed=fresh), one.search_arrays(q, k, 0.0, allowed=fresh),
                        f"mask reused k={k}")
    finally:
        lib.tav_set_row_mask = real_upload
    assert uploads == [N, N], uploads  # once by the sharded index, once by the whole-corpus one
    # every row of a subset above 8192 entries: the threshold route, as on one GPU
    big = np.concatenate([np.arange(N), np.arange(N)[::-1]])
    assert_same(sh.search_arrays(q[:3], len(big), 0.5, subset=big), one.search_arrays(q[:3], len(big), 0.5, subset=big),
                "routed subset")
    # k >= rows > 8192 with ties low-first alone, or a mask: the threshold route too
    v2 = np.concatenate([v, v[:3000]])
    one2 = whole(v2, storage)
    sh2 = ShardedVectorBase(settings(), device=0, storage_dtype=storage)
    sh2.deserialize(v2)
    allowed2 = np.arange(len(v2)) % 4 != 0
    for k in (len(v2), len(v2) + 3):
        assert_same(sh2.search_arrays(q[:3], k, 0.5, ties_low_first=True),
                    one2.search_arrays(q[:3], k, 0.5, ties_low_first=True), f"routed ties_low k={k}")
        assert_same(sh2.search_arrays(q[:3], k, 0.5, allowed=allowed2, ties_low_first=True),
                    one2.search_arrays(q[:3], k, 0.5, allowed=allowed2, ties_low_first=True), f"routed mask k={k}")
    for bad in ([0, N], [-N - 1]):
        with pytest.raises(IndexError):
            sh.fuzzy_lookup_embedding_in_subset(q[0], bad, 3, 0.0)
        with pytest.raises(IndexError):
            one.fuzzy_lookup_embedding_in_subset(q[0], bad, 3, 0.0)


# ---------------------------------------------------------------- (c) argument errors
def test_argument_errors():
    import torch

    lib = _capi.load()
    one = whole(corpus(1, seed=1)[0][:100], "float32")
    lib_, ix = one._ensure_device()
    qq = np.zeros((1, D), np.float32)
    items, scores, counts = np.empty((1, 4), np.int64), np.empty((1, 4), np.float32), np.empty(1, np.int32)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    rc = lib.tav_search(ix, ptr(qq), 1, 4, C.c_float(0.0), _capi.TAV_ITEMS_AS_POSITIONS, None, 0, 0, ptr(items),
                        ptr(scores), ptr(counts), None)
    assert rc == _capi.TAV_ERR_INVALID and "TAV_ITEMS_AS_POSITIONS" in _capi.last_error()
    offsets = np.zeros(2, np.int64)
    rc = lib.tav_range_search(ix, ptr(qq), 1, C.c_float(0.0), _capi.TAV_ITEMS_AS_POSITIONS, None, 0, 0, 0,
                              ptr(offsets), None)
    assert rc == _capi.TAV_ERR_INVALID and "TAV_ITEMS_AS_POSITIONS" in _capi.last_error()
    # with a subset the flag is accepted: items are positions
    sub = np.array([7, 7, -1, 3], np.int64)
    qq[0] = one._vectors[7]
    rc = lib.tav_search(ix, ptr(qq), 1, 4, C.c_float(0.0), _capi.TAV_ITEMS_AS_POSITIONS | _capi.TAV_TIES_LOW_FIRST,
                        ptr(sub), 4, 0, ptr(items), ptr(scores), ptr(counts), None)
    assert rc == 0 and sorted(items[0, : counts[0]].tolist()) == [0, 1, 2, 3]

    buf = torch.zeros(64, dtype=torch.int64, device="cuda")
    p = C.c_void_p(buf.data_ptr())

    def merge(n_lists=2, nq=1, k=4, it=p, sc=p, cn=p, order=2, oi=p, os_=p, oc=p, st=0):
        return lib.tav_merge_topk_ordered(0, n_lists, nq, k, it, sc, cn, st, st, st, order, oi, os_, oc, None)

    for bad in (dict(order=-1), dict(order=4), dict(n_lists=0), dict(k=0), dict(nq=-1), dict(it=None),
                dict(oc=None), dict(st=-1), dict(k=8193)):
        assert merge(**bad) == _capi.TAV_ERR_INVALID, bad
        assert "tav_merge_topk_ordered" in _capi.last_error()
    assert merge(nq=0) == 0

    for bad in (dict(n=-1), dict(tl=-1), dict(items=None), dict(table=None)):
        a = dict(n=4, table=p, tl=4, items=p) | bad
        assert lib.tav_map_items(0, a["n"], a["table"], a["tl"], a["items"], None) == _capi.TAV_ERR_INVALID, bad
    assert lib.tav_map_items(0, 0, None, 0, None, None) == 0
    vals = torch.tensor([-1, 0, 3, 4, 2, -7, 1], dtype=torch.int64, device="cuda")
    table = torch.tensor([10, -11, 12, 13], dtype=torch.int64, device="cuda")
    assert lib.tav_map_items(0, vals.numel(), C.c_void_p(table.data_ptr()), 4, C.c_void_p(vals.data_ptr()), None) == 0
    torch.cuda.synchronize()
    assert vals.tolist() == [-1, 10, 13, 4, 12, -7, -11]


# ---------------------------------------------------------------- (d) broken builds
MUTANTS = {1: "merge order argument ignored", 2: "position key replaced by the list-slot key",
           3: "subset position decoded despite the flag"}


@pytest.fixture(scope="module")
def mutant_libs():
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc) and not shutil.which(nvcc):
        pytest.skip("nvcc is needed to build the broken variants")
    from typeagent_py_b200 import build as B

    tmp = tempfile.mkdtemp(prefix="tav_filter_mutants_")
    procs = {}
    for m in MUTANTS:
        out = os.path.join(tmp, f"libtavec_mutant{m}.so")
        cmd = [nvcc, *[f for f in B.NVCC_FLAGS if f != "-Xptxas=-v"], f"-DTAV_SHARDED_FILTER_MUTANT={m}", "-o", out,
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
    """Indexes created inside run on ``lib``."""
    saved = _capi._lib
    _capi._lib = lib
    try:
        yield
    finally:
        _capi._lib = saved


def mutant_checks():
    """(a)'s checks on a few cases; returns the failures."""
    caught = []
    v, q = corpus(3, seed=5)
    sub = subset_of(seed=5)
    allowed = np.random.default_rng(5).random(N) < 0.5
    allowed[:600] = allowed[1500:2100] = True
    one = whole(v, "float32")
    engines = engines_for(v, 3, "float32")
    checks = [
        (lambda: subset_topk(engines, N, q[:1], 50, 0.0, sub, False), lambda: one.search_arrays(q[:1], 50, 0.0, subset=sub)),
        (lambda: subset_topk(engines, N, q, 100, 0.0, sub, True),
         lambda: one.search_arrays(q, 100, 0.0, subset=sub, ties_low_first=True)),
        (lambda: masked_topk(engines, N, q, 100, 0.0, allowed, True),
         lambda: one.search_arrays(q, 100, 0.0, allowed=allowed, ties_low_first=True)),
        (lambda: subset_range(engines, N, q, 0.5, sub, False), lambda: one.search_range(q, 0.5, subset=sub)),
    ]
    for got, want in checks:
        try:
            assert_same(got(), want(), "mutant")
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
