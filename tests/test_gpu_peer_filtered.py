"""Filtered and subset lookups through the peer-memory exchange, bit for bit, and its failure protocol.

W processes (tests/peer_filter_ranks.py) share the device and form one group over CUDA IPC, as in
tests/test_gpu_peer_exchange.py.  Every lookup here goes through ``tav_sharded_search`` with a row mask, per-query
masks or ties low-first, or through ``tav_sharded_search_subset`` (one subset, or per-query subsets), and every
rank's items, score bits and counts must equal one ``VectorBase`` over the whole corpus on dyadic corpora.

Cases at W = 2 and 3 with uneven blocks and one at W = 8: bf16 / fp16 / float32; row masks and predicates with both
tie orders; per-query masks; subsets with duplicates across block edges and negative ordinals; per-query subsets,
one set of them inside the first block only (the other ranks have no share); rows copied across block boundaries;
deferred filtered searches mixed with plain ones up to the group's depth (8), a ninth refused; the repair of
masked searches that only the last rank flags (a block of identical rows); and one rank whose per-query mask
allocation fails, through the upload agreement and through the slot's status word, and one rank whose local
search fails in cudaMalloc, synchronous and deferred: every rank must raise, and the searches after it complete.  Two deliberately broken builds (``TAV_PEER_FILTER_MUTANT``) are each caught.
"""

from __future__ import annotations

import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

import tests.test_gpu_peer_exchange as peer_exchange
from tests.peer_filter_ranks import filters, predicate_of
from tests.peer_ranks import corpus, queries
from tests.test_gpu_peer_exchange import assert_same, boundary_dups

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "peer_filter_ranks.py")
D = 64


def q(seed, b, **kw):
    return dict(seed=seed, b=b, **kw)


def s(key, qs, k, f, ms=0.0, **kw):
    return dict(op="search", key=key, q=qs, k=k, ms=float(ms), filters=f, **kw)


def filter_ops(n: int, world: int, prefix: str = "") -> list[dict]:
    per = -(-n // world)
    edges = [g * per for g in range(1, world)]
    ops = []
    for ties in (False, True):
        t = "low" if ties else "high"
        ops += [s(f"{prefix}row-{t}-B16", q(11, 16, favour=10), 10, dict(seed=1, allowed=True, ties=ties)),
                s(f"{prefix}row-{t}-B1", q(12, 1), 25, dict(seed=2, allowed=True, ties=ties)),
                s(f"{prefix}sub-{t}-B16", q(13, 16, favour=10), 10, dict(seed=3, subset=True, edges=edges, ties=ties)),
                s(f"{prefix}sub-{t}-B1", q(14, 1), 40, dict(seed=4, subset=True, edges=edges, ties=ties)),
                s(f"{prefix}subs-{t}", q(15, 12), 16, dict(seed=5, subsets=True, ties=ties)),
                s(f"{prefix}subs0-{t}", q(16, 9), 8, dict(seed=6, subsets=True, within=[0, per // 2], ties=ties)),
                s(f"{prefix}ties-{t}", q(17, 16, favour=10), 10, dict(seed=7, ties=ties))]
    ops += [s(f"{prefix}qm-B16", q(18, 16, favour=10), 10, dict(seed=8, masks=True)),
            s(f"{prefix}qm-B33", q(19, 33), 50, dict(seed=9, masks=True)),
            s(f"{prefix}qm-B1", q(20, 1), 10, dict(seed=10, masks=True)),
            dict(op="pred", key=f"{prefix}pred", q=q(21, 1, favour=10), k=10, ms=0.0, pred=dict(mod=3))]
    return ops


def storage_case(world: int, storage: str) -> dict:
    n = {2: 10001, 3: 15007, 8: 8 * 1300 + 5}[world]
    cspec = dict(n=n, d=D, seed=1100 + world, preset="coarse" if storage == "bfloat16" else "fine",
                 dup=boundary_dups(n, world))
    return dict(name=storage, storage=storage, corpus=cspec, ops=filter_ops(n, world))


def pipeline_case(world: int) -> dict:
    """Eight deferred searches (filtered and plain, the depth), a ninth refused, finish; then deferred subset
    lookups resolved by a synchronous one."""
    n = 4500 * world + 7
    cspec = dict(n=n, d=D, seed=1300 + world, preset="fine", dup=boundary_dups(n, world))
    kinds = [dict(seed=31, allowed=True), None, dict(seed=32, subset=True, ties=True), dict(seed=33, masks=True),
             dict(seed=34, subsets=True), None, dict(seed=31, allowed=True, ties=True), dict(seed=36, subset=True)]
    # the masks are uploaded (and agreed on) by synchronous lookups first: a deferred lookup then finds them in place
    ops = [s("w-row", q(1398, 16), 5, dict(seed=31, allowed=True)), s("w-qm", q(1399, 19), 5, dict(seed=33, masks=True))]
    ops += [s(f"d{i}", q(1400 + i, 16 + i), 5 + i, f or dict(seed=0), defer=True) for i, f in enumerate(kinds)]
    ops += [dict(op="raise", key="ninth", q=q(1499, 16), k=10, ms=0.0, filters=dict(seed=37, subset=True)),
            dict(op="finish", key="eight"),
            s("e0", q(1410, 16), 9, dict(seed=38, subset=True), defer=True),
            s("e1", q(1411, 8), 7, dict(seed=39, subsets=True, ties=True), defer=True),
            s("sync", q(1412, 16), 12, dict(seed=40, masks=True))]
    return dict(name="pipeline", storage="bfloat16", corpus=cspec, ops=ops)


def repair_case(world: int) -> dict:
    """The last block ends in 21,500 copies of row 100: the tensor-core searches that favour it overflow their
    candidates on that rank only, which redoes them at finish; the masked searches are re-merged."""
    per = 22000
    cspec = dict(n=per * world, d=D, seed=1500 + world, preset="fine",
                 copies=[100, per * (world - 1) + 500, per * world])
    ops = [s("w-row", q(1598, 16), 5, dict(seed=41, allowed=True)), s("w-qm", q(1599, 20), 5, dict(seed=43, masks=True)),
           s("rowA", q(1600, 16, favour=100), 10, dict(seed=41, allowed=True), defer=True),
           s("subA", q(1601, 16, favour=100), 10, dict(seed=42, subset=True, ties=True), defer=True),
           s("qmA", q(1602, 20, favour=100), 8, dict(seed=43, masks=True), defer=True),
           s("lowA", q(1603, 16, favour=100), 10, dict(seed=44, ties=True), defer=True),
           dict(op="finish", key="repair", expect="positive"),
           s("rowS", q(1604, 16, favour=100), 12, dict(seed=41, allowed=True))]
    return dict(name="repair", storage="bfloat16", corpus=cspec, ops=ops)


def failure_case(world: int) -> dict:
    """One rank's per-query mask upload fails: through the agreement, and past it (status word), synchronous and
    deferred.  Then a cudaMalloc inside one rank's local tensor-core search fails (a real, non-sticky allocation
    failure), synchronous and deferred.  Afterwards more searches than the group's depth (8) succeed on every
    rank: every failed search was merged and acknowledged, so no slot waits for an acknowledgement."""
    n = 5000 * world + 1  # every block above 4096 rows: B = 16 bf16 searches take the tensor cores
    cspec = dict(n=n, d=D, seed=1700 + world, preset="fine")
    last = world - 1
    fail = lambda key, seed, f, **kw: dict(op="fail", key=key, q=q(seed, 16), k=10, ms=0.0,  # noqa: E731
                                           filters=f, cap_rank=last, **kw)
    masks = lambda seed: dict(seed=seed, masks=True)  # noqa: E731
    ops = [fail("agree", 50, masks(50), agree=True), fail("status", 51, masks(51)),
           fail("status-defer", 52, masks(52), defer=True), s("after", q(53, 16), 10, masks(53)),
           fail("alloc", 54, dict(seed=54, allowed=True), alloc=True),
           fail("alloc-defer", 55, dict(seed=54, allowed=True), alloc=True, defer=True)]
    ops += [s(f"after{i}", q(60 + i, 16), 10, dict(seed=54, allowed=True)) for i in range(10)]
    return dict(name="failure", storage="bfloat16", corpus=cspec, ops=ops)


FAIL_EXPECT = {"agree": (1, 2, 0, 0), "status": (1, 2, 0, 0), "status-defer": (1, 0, 2, 2), "alloc": (1, 2, 0, 0),
               "alloc-defer": (1, 0, 2, 2)}  # (search codes: failing rank, others; finish codes: failing rank,
# others) with 0 nothing, 1 MemoryError, 2 RuntimeError


def cases_for(world: int) -> list[dict]:
    if world == 8:
        return [storage_case(8, "bfloat16")]
    return ([storage_case(world, st) for st in ("bfloat16", "float16", "float32")]
            + [pipeline_case(world), repair_case(world), failure_case(world)])


# ---------------------------------------------------------------- expectations
def expectations(case: dict) -> dict:
    """key -> (items, scores, counts) of every lookup of the case from one VectorBase over the whole corpus."""
    import typeagent_py_b200 as tab
    from oracle import vectorbase_oracle as O

    cspec = case["corpus"]
    v = corpus(cspec)
    whole = tab.VectorBase(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()), storage_dtype=case["storage"])
    whole.add_embeddings(None, v)
    out = {}
    for op in case["ops"]:
        if op["op"] == "search":
            qq = queries(op["q"], cspec, v)
            out[op["key"]] = whole.search_arrays(qq, op["k"], op["ms"], **filters(op["filters"], len(v), len(qq)))
        elif op["op"] == "pred":
            qq = queries(op["q"], cspec, v)
            hits = whole.fuzzy_lookup_embedding(qq[0], op["k"], op["ms"], predicate=predicate_of(op["pred"]))
            out[op["key"]] = (np.array([[h.item for h in hits]], np.int64),
                              np.array([[h.score for h in hits]], np.float32), np.array([len(hits)], np.int32))
    return out


def mismatches(case: dict, want: dict, world: int, out: str) -> list[str]:
    errors, finishes = [], {}
    for r in range(world):
        got = np.load(os.path.join(out, f"{case['name']}.r{r}.npz"))
        for key, w in want.items():
            try:
                assert_same([got[f"{key}.{f}"] for f in ("items", "scores", "counts")], w, f"rank {r} {key}")
            except (AssertionError, KeyError) as e:
                errors.append(str(e))
        for op in case["ops"]:
            if op["op"] == "finish":
                finishes.setdefault(op["key"], []).append(int(got[op["key"] + ".finish"][0]))
            if op["op"] == "raise" and int(got[op["key"] + ".raised"][0]) != 1:
                errors.append(f"rank {r} {op['key']}: the search was not refused for the outstanding searches")
            if op["op"] == "fail":
                capped = r == op["cap_rank"]
                e = FAIL_EXPECT[op["key"]]
                want_codes = (e[0], e[2]) if capped else (e[1], e[3])
                codes = tuple(int(c) for c in got[op["key"] + ".codes"])
                if codes != want_codes:
                    errors.append(f"rank {r} {op['key']}: raised {codes} (search, finish), expected {want_codes}")
    for op in case["ops"]:
        if op["op"] == "finish":
            counts = finishes[op["key"]]
            ok = counts[0] > 0 if op.get("expect") == "positive" else True
            if len(set(counts)) != 1 or not ok:
                errors.append(f"finish {op['key']}: counts {counts} per rank, expected {op.get('expect', 'any')}")
    return errors


_RUNS: dict = {}


def run_world(world: int, lib: str | None = None):
    """The ranks of one world over all its cases, launched once per session."""
    if (world, lib) not in _RUNS:
        cases = cases_for(world) if lib is None else [storage_case(2, "bfloat16"), failure_case(2)]
        want = {c["name"]: expectations(c) for c in cases}
        tmp = tempfile.mkdtemp(prefix=f"tav_peer_filter_w{world}_")
        try:
            worker, peer_exchange.WORKER = peer_exchange.WORKER, WORKER  # its launcher, with this file's worker
            try:
                out = peer_exchange.launch(world, cases, tmp, lib=lib)
            finally:
                peer_exchange.WORKER = worker
            errors = {c["name"]: mismatches(c, want[c["name"]], world, out) for c in cases}
            _RUNS[(world, lib)] = ("ok", errors)
        except pytest.skip.Exception as e:
            _RUNS[(world, lib)] = ("skip", str(e))
        except (Exception, pytest.fail.Exception) as e:
            _RUNS[(world, lib)] = ("fail", f"{type(e).__name__}: {e}"[:4000])
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
    kind, value = _RUNS[(world, lib)]
    if kind == "skip":
        pytest.skip(value)
    if kind == "fail":
        pytest.fail(f"the W={world} ranks failed:\n{value}")
    return value


CASE_NAMES = ["bfloat16", "float16", "float32", "pipeline", "repair", "failure"]


@pytest.mark.parametrize("name", CASE_NAMES)
@pytest.mark.parametrize("world", [2, 3])
def test_peer_filtered_equals_one_vectorbase(world, name):
    errors = run_world(world)[name]
    assert not errors, "\n".join(errors[:20])


def test_peer_filtered_eight_ranks():
    errors = run_world(8)["bfloat16"]
    assert not errors, "\n".join(errors[:20])


# ---------------------------------------------------------------- broken builds
MUTANTS = {1: "subset positions published unmapped", 2: "status word ignored"}


@pytest.fixture(scope="module")
def mutant_libs():
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc) and not shutil.which(nvcc):
        pytest.skip("nvcc is needed to build the broken variants")
    from typeagent_py_b200 import build as B

    tmp = tempfile.mkdtemp(prefix="tav_peer_filter_mutants_")
    procs = {}
    for m in MUTANTS:
        out = os.path.join(tmp, f"libtavec_peer_filter_mutant{m}.so")
        cmd = [nvcc, *[f for f in B.NVCC_FLAGS if f != "-Xptxas=-v"], f"-DTAV_PEER_FILTER_MUTANT={m}", "-o", out,
               *[os.path.join(B.CSRC, src) for src in B.SOURCES]]
        procs[m] = (subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True), out)
    libs = {}
    for m, (proc, out) in procs.items():
        log = proc.communicate()[0]
        assert proc.returncode == 0, log
        libs[m] = out
    yield libs
    shutil.rmtree(tmp, ignore_errors=True)


@pytest.mark.parametrize("m", sorted(MUTANTS), ids=[MUTANTS[m].replace(" ", "_") for m in sorted(MUTANTS)])
def test_broken_build_is_caught(mutant_libs, m):
    if any(kind == "fail" for kind, _ in _RUNS.values()):
        pytest.skip("the real build failed: its broken variants are not launched")
    errors = run_world(2, lib=mutant_libs[m])
    assert any(errors.values()), f"the checks did not catch: {MUTANTS[m]}"
