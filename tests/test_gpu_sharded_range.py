"""Sharded threshold search on the GPU, bit for bit on dyadic corpora (tests/exact.py):

(a) ``tav_merge_range`` through the C ABI: W indexes on the row blocks of one corpus, each block's
    ``tav_range_search`` with ``item_offset`` = its first row, packed into one padded [W, T_max] buffer as the
    all-gather produces it, merged — equal to ``expected_range`` of the whole corpus, every query;
(b) ``ShardedVectorBase`` with one rank: ``search_range``, ``max_hits=0`` lookups and ``search_arrays`` with
    k >= rows > 8192 equal to one ``VectorBase``;
(c) deliberately broken builds of the merge kernel (``TAV_MERGE_RANGE_MUTANT``), each caught by (a)'s checks.
"""

from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import vectorbase_oracle as O
from tests.exact import dyadic_corpus, preset
from tests.test_gpu_range import assert_same_range, expected_range
from typeagent_py_b200 import _capi

pytestmark = pytest.mark.gpu

PATH_NAMES = {"scan": "scan", "mma": "mma", "split": "mma"}


def blocks(n, w):
    per = -(-n // w)
    return [(min(g * per, n), min((g + 1) * per, n)) for g in range(w)]


def local_ranges(v, q, w, storage, path, ms, ties_low):
    """Every block's range search (host arrays) and the path each took."""
    import typeagent_py_b200 as tab

    parts, paths = [], set()
    b = len(q)
    for lo, hi in blocks(len(v), w):
        if hi == lo:
            parts.append((np.zeros(b + 1, np.int64), np.empty(0, np.int64), np.empty(0, np.float32)))
            continue
        base = tab.VectorBase(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()), storage_dtype=storage)
        base.add_embeddings(None, v[lo:hi])
        base.force_path = PATH_NAMES[path]
        base.enable_timing()
        lib, ix = base._ensure_device()
        flags = base._flags() | (_capi.TAV_TIES_LOW_FIRST if ties_low else 0)
        qq = np.ascontiguousarray(q, np.float32)
        offsets = np.zeros(b + 1, np.int64)
        _capi.check(lib.tav_range_search(ix, qq.ctypes.data_as(C.c_void_p), b, C.c_float(ms), flags, None, 0, lo, 0,
                                         offsets.ctypes.data_as(C.c_void_p), None))
        n = int(offsets[-1])
        items, scores = np.empty(n, np.int64), np.empty(n, np.float32)
        if n:
            _capi.check(lib.tav_range_fetch(ix, 0, n, items.ctypes.data_as(C.c_void_p),
                                            scores.ctypes.data_as(C.c_void_p), 0, None))
        paths.add(base.last_timing()["path"])
        parts.append((offsets, items, scores))
    return parts, paths


def merge(parts, ties_low, lib=None):
    """Pack the lists into one padded buffer per field, as the all-gather does, and merge on the device."""
    import torch

    lib = lib or _capi.load()
    w, b = len(parts), len(parts[0][0]) - 1
    t_max = max(1, max(int(o[-1]) for o, _, _ in parts))
    offs = np.zeros((w, b + 1), np.int64)
    items = np.full((w, t_max), -7, np.int64)
    scores = np.full((w, t_max), np.float32(0.125), np.float32)
    for g, (o, i, s) in enumerate(parts):
        offs[g], items[g, : len(i)], scores[g, : len(s)] = o, i, s
    dev = torch.device("cuda", 0)
    d_offs, d_items, d_scores = (torch.from_numpy(x).to(dev) for x in (offs, items, scores))
    cap = w * t_max + 1  # room for any total a broken build could claim
    out_o = torch.full((b + 1,), -1, dtype=torch.int64, device=dev)
    out_i = torch.full((cap,), -1, dtype=torch.int64, device=dev)
    out_s = torch.full((cap,), -1.0, dtype=torch.float32, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    _capi.check(lib.tav_merge_range(0, w, b, C.c_void_p(d_offs.data_ptr()), b + 1, C.c_void_p(d_items.data_ptr()),
                                    t_max, C.c_void_p(d_scores.data_ptr()), t_max, int(ties_low),
                                    C.c_void_p(out_o.data_ptr()), C.c_void_p(out_i.data_ptr()),
                                    C.c_void_p(out_s.data_ptr()), C.c_void_p(stream)))
    o = out_o.cpu().numpy()
    total = int(min(max(o[-1], 0), cap))
    return o, out_i.cpu().numpy()[:total], out_s.cpu().numpy()[:total]


def run_case(n, d, b, w, storage, path, pre, ms, ties_low, dup=(), seed=0, lib=None):
    amp, exp = preset(pre, d)
    v, q, dots = dyadic_corpus(n, d, b, amp, exp, seed=seed, dup=dup)
    parts, paths = local_ranges(v, q, w, storage, path, ms, ties_low)
    want_path = {"scan": "scan", "mma": "mma", "split": "mma_split"}[path]
    assert paths <= {want_path}, paths
    return merge(parts, ties_low, lib), expected_range(dots, ms, ties_low=ties_low), parts


P = pytest.param
# (n, d, b, W, storage, path, preset, min_score, ties_low)
CASES = [
    P(6000, 64, 3, 1, "float32", "scan", "fine", 0.0, False, id="W1-f32-scan"),
    P(6000, 64, 3, 2, "float32", "scan", "fine", 0.0, False, id="W2-f32-scan"),
    P(6000, 64, 5, 3, "float16", "scan", "coarse", 0.5, True, id="W3-fp16-scan-ties_low-coarse"),
    P(6000, 64, 4, 8, "bfloat16", "scan", "fine", -2.0, False, id="W8-bf16-scan-everything"),
    P(6000, 64, 16, 2, "bfloat16", "mma", "fine", 0.0, False, id="W2-bf16-mma"),
    P(6000, 72, 17, 3, "float16", "mma", "coarse", 0.5, False, id="W3-fp16-mma-coarse"),
    P(8192, 64, 16, 8, "bfloat16", "mma", "coarse", 0.0, True, id="W8-bf16-mma-ties_low"),
    P(6000, 64, 16, 3, "float32", "split", "fine", 0.0, False, id="W3-f32-split"),
    P(6000, 64, 20, 8, "float32", "split", "coarse", 0.5, True, id="W8-f32-split-ties_low"),
    P(4000, 32, 130, 3, "bfloat16", "scan", "fine", 0.6, False, id="W3-bf16-B130"),
    P(4096, 64, 130, 8, "float16", "mma", "fine", 0.55, False, id="W8-fp16-mma-B130"),
]


@pytest.mark.parametrize("n,d,b,w,storage,path,pre,ms,ties_low", CASES)
def test_merge_range_equals_whole_corpus(n, d, b, w, storage, path, pre, ms, ties_low):
    got, want, _ = run_case(n, d, b, w, storage, path, pre, ms, ties_low, seed=n + d + b + w)
    assert_same_range(got, want, f"W={w} {storage} {path}")


def dup_across_blocks(n, w):
    """(dst, src) pairs: rows of block 0 copied into every other block, so equal scores cross list boundaries."""
    out = []
    for g, (lo, hi) in enumerate(blocks(n, w)):
        if g:
            out += [(lo + j, j) for j in range(0, min(60, hi - lo), 2)]
    return out


@pytest.mark.parametrize("ties_low", [False, True], ids=["ties_high", "ties_low"])
@pytest.mark.parametrize("storage,path,w", [("float32", "scan", 3), ("bfloat16", "mma", 8), ("float32", "split", 2)])
def test_equal_scores_across_lists(storage, path, w, ties_low):
    n = 6000
    got, want, parts = run_case(n, 64, 16, w, storage, path, "coarse", 0.0, ties_low, dup=dup_across_blocks(n, w),
                                seed=3)
    assert_same_range(got, want, f"dups W={w} {storage} {path} ties_low={ties_low}")
    # the case does what it says: some score is returned from more than one list
    o, _, s = parts[0]
    assert any(np.isin(s[o[0]:o[1]].view(np.uint32), p[2][p[0][0]:p[0][1]].view(np.uint32)).any() for p in parts[1:])


def test_empty_lists_and_queries_without_hits():
    amp, exp = preset("fine", 64)
    v, q, dots = dyadic_corpus(3000, 64, 6, amp, exp, seed=9)
    # query 0: only block 1 can pass; query 1 (zero: every score 0.5): nothing anywhere
    d0 = dots[0]
    v[:1000][d0[:1000] > 0] *= -1
    v[2000:][d0[2000:] > 0] *= -1
    q[1] = 0
    dots = (q.astype(np.float64) @ v.astype(np.float64).T).astype(np.float32)
    ms = 0.5000001
    parts, _ = local_ranges(v, q, 3, "float32", "scan", ms, False)
    parts.insert(1, (np.zeros(len(q) + 1, np.int64), np.empty(0, np.int64), np.empty(0, np.float32)))  # an empty list
    assert parts[0][0][1] == 0 and parts[2][0][1] > 0
    assert_same_range(merge(parts, False), expected_range(dots, ms), "sparse lists")
    nothing = [(np.zeros(len(q) + 1, np.int64), np.empty(0, np.int64), np.empty(0, np.float32))] * 4
    o, i, s = merge(nothing, False)
    assert o.tolist() == [0] * (len(q) + 1) and len(i) == 0


def test_one_query_of_a_million_hits_over_eight_lists():
    amp, exp = preset("fine", 8)
    n = (1 << 20) + 4099
    v, q, dots = dyadic_corpus(n, 8, 1, amp, exp, seed=21)
    want = expected_range(dots, -2.0)
    parts, paths = local_ranges(v, q, 8, "bfloat16", "scan", -2.0, False)
    assert paths == {"scan"} and int(want[0][-1]) == n >= 1 << 20
    assert_same_range(merge(parts, False), want, "1M hits")
    parts, _ = local_ranges(v, q, 8, "bfloat16", "scan", -2.0, True)
    assert_same_range(merge(parts, True), expected_range(dots, -2.0, ties_low=True), "1M hits ties_low")


def test_merge_range_argument_errors():
    import torch

    lib = _capi.load()
    buf = torch.zeros(64, dtype=torch.int64, device="cuda")
    p = C.c_void_p(buf.data_ptr())

    def call(n_lists=2, nq=1, off=p, os_=2, it=p, is_=4, sc=p, ss=8, oo=p, oi=p, osc=p):
        return lib.tav_merge_range(0, n_lists, nq, off, os_, it, is_, sc, ss, 0, oo, oi, osc, None)

    for bad in (dict(n_lists=0), dict(n_lists=-1), dict(n_lists=33), dict(nq=-1), dict(os_=-1), dict(is_=-2),
                dict(ss=-3), dict(off=None), dict(it=None), dict(sc=None), dict(oo=None), dict(oi=None),
                dict(osc=None)):
        assert call(**bad) == _capi.TAV_ERR_INVALID, bad
        assert "tav_merge_range" in _capi.last_error()
    assert call(nq=0, off=None, it=None, sc=None, oo=None, oi=None, osc=None) == 0  # nothing to do
    torch.cuda.synchronize()


# ---------------------------------------------------------------- (b) one rank
def test_sharded_one_rank_equals_vectorbase():
    import socket

    import torch.distributed as dist

    import typeagent_py_b200 as tab
    from typeagent_py_b200.sharded import ShardedVectorBase

    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    dist.init_process_group("gloo", rank=0, world_size=1, init_method=f"tcp://127.0.0.1:{port}")
    try:
        amp, exp = preset("coarse", 64)
        n = 10000
        v, q, _ = dyadic_corpus(n, 64, 20, amp, exp, seed=31)
        settings = tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel())
        for storage in ("float32", "bfloat16"):
            one = tab.VectorBase(settings, storage_dtype=storage)
            one.add_embeddings(None, v)
            sh = ShardedVectorBase(settings, device=0, storage_dtype=storage)
            sh.deserialize(v)
            for ms in (0.0, 0.6):
                for tl in (False, True):
                    assert_same_range(sh.search_range(q, ms, ties_low_first=tl), one.search_range(q, ms, ties_low_first=tl),
                                      f"{storage} {ms} {tl}")
                want = one.fuzzy_lookup_embeddings(q, max_hits=0, min_score=ms)
                assert sh.fuzzy_lookup_embeddings(q, max_hits=0, min_score=ms) == want
                assert sh.fuzzy_lookup_embedding(q[3], max_hits=0, min_score=ms) == \
                    one.fuzzy_lookup_embedding(q[3], max_hits=0, min_score=ms)
                for k in (n, n + 5):
                    gi, gs, gc = sh.search_arrays(q, k, ms)
                    wi, ws, wc = one.search_arrays(q, k, ms)
                    np.testing.assert_array_equal(gc, wc)
                    np.testing.assert_array_equal(gi, wi)
                    np.testing.assert_array_equal(gs.view(np.uint32), ws.view(np.uint32))
    finally:
        dist.destroy_process_group()


# ---------------------------------------------------------------- (c) broken builds
MUTANTS = {1: "ties broken by list index", 2: "ties-low ignored", 3: "co-rank off by one",
           4: "out_offsets over the padded counts", 5: "last partial tile dropped"}


@pytest.fixture(scope="module")
def mutant_libs():
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc) and not shutil.which(nvcc):
        pytest.skip("nvcc is needed to build the broken variants")
    csrc = os.path.join(os.path.dirname(_capi.__file__), "csrc")
    tmp = tempfile.mkdtemp(prefix="tav_mutants_")
    shim = os.path.join(tmp, "shim.cu")
    with open(shim, "w") as f:  # the one library symbol the merge unit needs
        f.write("namespace tav { void set_error(const char*, ...) {} }\n")
    procs = {}
    for m in MUTANTS:
        out = os.path.join(tmp, f"libmerge_mutant{m}.so")
        cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
               "-shared", "-cudart", "static", f"-DTAV_MERGE_RANGE_MUTANT={m}", "-o", out,
               os.path.join(csrc, "tav_merge_range.cu"), shim]
        procs[m] = (subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True), out)
    libs = {}
    for m, (proc, out) in procs.items():
        log = proc.communicate()[0]
        assert proc.returncode == 0, log
        lib = C.CDLL(out)
        restype, argtypes = _capi.SIGNATURES["tav_merge_range"]
        lib.tav_merge_range.restype, lib.tav_merge_range.argtypes = restype, argtypes
        libs[m] = lib
    yield libs
    shutil.rmtree(tmp, ignore_errors=True)


def mutant_cases():
    n = 6000
    yield dict(n=n, d=64, b=16, w=3, storage="float32", path="scan", pre="coarse", ms=0.0, ties_low=False,
               dup=dup_across_blocks(n, 3), seed=3)
    yield dict(n=n, d=64, b=16, w=3, storage="float32", path="scan", pre="coarse", ms=0.0, ties_low=True,
               dup=dup_across_blocks(n, 3), seed=3)
    yield dict(n=8192, d=64, b=16, w=8, storage="bfloat16", path="mma", pre="fine", ms=0.3, ties_low=False, seed=4)


@pytest.mark.parametrize("m", sorted(MUTANTS), ids=[MUTANTS[m].replace(" ", "_") for m in sorted(MUTANTS)])
def test_broken_merge_is_caught(mutant_libs, m):
    caught = []
    for case in mutant_cases():
        got, want, _ = run_case(**case, lib=mutant_libs[m])
        try:
            assert_same_range(got, want, MUTANTS[m])
        except AssertionError as e:
            caught.append(str(e)[:200])
    assert caught, f"the exact checks did not catch: {MUTANTS[m]}"


# ---------------------------------------------------------------- the product's exchange layout on one GPU
@pytest.mark.parametrize("storage,path,w,ties_low", [("float32", "scan", 3, False), ("bfloat16", "mma", 8, True),
                                                     ("float32", "split", 2, False)])
def test_engine_glue_over_the_packed_exchange_layout(storage, path, w, ties_low):
    """What ShardedVectorBase.search_range does between the collectives, with the all-gathers replaced by
    stacking: W CudaShardEngines on the row blocks, each rank's offsets + status word and its hits fetched into
    the packed payload (pack_range_payload), CudaShardEngine.merge_range over the stacked buffers."""
    import torch

    from typeagent_py_b200.sharded import CudaShardEngine, offsets_with_status, pack_range_payload, range_pad

    n, b = 6000, 16
    amp, exp = preset("coarse", 64)
    v, q, dots = dyadic_corpus(n, 64, b, amp, exp, seed=41, dup=dup_across_blocks(n, w))
    settings = tab_settings()
    engines, locals_ = [], []
    for lo, hi in blocks(n, w):
        eng = CudaShardEngine(settings, 0, storage)
        eng.load_rows(v[lo:hi])
        eng.base.force_path = PATH_NAMES[path]
        engines.append(eng)
        locals_.append(eng.range_local(q, 0.25, lo, ties_low))
    want_path = {"scan": "scan", "mma": "mma", "split": "mma_split"}[path]
    assert {e.base.last_timing()["path"] for e in engines} == {want_path}
    dev = engines[0].comm_device()
    offsets_all = torch.from_numpy(np.stack([offsets_with_status(loc.offsets, False) for loc in locals_])).to(dev)
    totals = [int(loc.offsets[-1]) for loc in locals_]
    t_pad = range_pad(totals)
    assert len(set(totals)) > 1 or t_pad > totals[0]  # some rank's hits are padded
    payload = torch.stack([pack_range_payload(loc, t_pad, dev) for loc in locals_])
    got = engines[0].merge_range(offsets_all, payload, w, b, t_pad, sum(totals), ties_low)
    got = tuple(t.cpu().numpy() for t in got)
    assert_same_range(got, expected_range(dots, 0.25, ties_low=ties_low), f"engines W={w} {storage} {path}")


def tab_settings():
    import typeagent_py_b200 as tab

    return tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel())
