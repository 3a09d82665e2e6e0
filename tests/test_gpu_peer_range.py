"""Threshold searches through the peer-memory exchange (the group's range inbox), bit for bit, and their failure
protocol.

W processes (tests/peer_range_ranks.py) share the device and form one group over CUDA IPC, as in
tests/test_gpu_peer_exchange.py.  Every threshold search here goes through ``tav_sharded_range_search`` and its
merge, and every rank's offsets, items and score bits must equal one ``VectorBase.search_range`` over the whole
corpus on dyadic corpora.

Cases at W = 2 and 3 with uneven blocks and equal rows across block edges, and one at W = 8: bf16 / fp16 / float32 on
the tensor cores (B >= 16) and the row scan; min_score at a hit and one ulp either side, NaN, above every score and 0
(every row); row masks and per-query masks in both tie orders; subsets with duplicates and negative ordinals across
block edges; per-query subsets, one set inside the first block only; the routed calls (``fuzzy_lookup_embedding``
with max_hits=0, ``search_arrays`` with k >= rows > 8192, per-query subsets with k > 2048); a rank with no rows;
sizes that force a grow, repeat in one round and give the excess back to the retention size; deferred top-k lookups
outstanding across threshold searches; and failures: one rank's local search fails, one rank's inbox cannot grow,
one rank cannot allocate the merged result (with and without a grow and a give-back in the same call).
Three deliberately broken builds (``TAV_PEER_RANGE_MUTANT``) are each caught.
"""

from __future__ import annotations

import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

import tests.test_gpu_peer_exchange as peer_exchange
from tests.peer_filter_ranks import filters
from tests.peer_ranks import corpus, queries
from tests.test_gpu_peer_exchange import boundary_dups, dots_of, ulp_cases

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "peer_range_ranks.py")
D = 64


def q(seed, b, **kw):
    return dict(seed=seed, b=b, **kw)


def r(key, qs, ms, f=None, **kw):
    return dict(op="range", key=key, q=qs, ms=float(ms), filters=f or dict(seed=0), **kw)


def top_ms(cspec, v, qs, hits):
    """A min_score that about ``hits`` (query, row) pairs of the queries reach, from the exact scores."""
    sc = np.clip((dots_of(queries(qs, cspec, v), v) + np.float32(1)) / np.float32(2), 0, 1).astype(np.float32)
    return float(np.sort(sc.ravel())[-hits])


def range_ops(cspec, v, n: int, world: int, prefix: str = "") -> list[dict]:
    per = -(-n // world)
    edges = [g * per for g in range(1, world)]
    ops = [dict(o, op="range", key=prefix + o["key"]) for o in
           ulp_cases(cspec, v, "ms16", 5, 16, 0) + ulp_cases(cspec, v, "ms1", 6, 1, 0)]
    ops += [r(prefix + "nan", q(7, 16), float("nan")), r(prefix + "none", q(8, 16), 1.5),
            r(prefix + "all-B3", q(9, 3), 0.0), r(prefix + "all-B16", q(10, 16), 0.0)]
    for ties in (False, True):
        t = "low" if ties else "high"
        ops += [r(f"{prefix}row-{t}-B16", q(11, 16, favour=10), 0.5, dict(seed=1, allowed=True, ties=ties)),
                r(f"{prefix}row-{t}-B1", q(12, 1), 0.5, dict(seed=2, allowed=True, ties=ties)),
                r(f"{prefix}qm-{t}-B16", q(13, 16), 0.5, dict(seed=3, masks=True, ties=ties)),
                r(f"{prefix}sub-{t}", q(14, 16, favour=10), 0.3, dict(seed=4, subset=True, edges=edges, ties=ties)),
                r(f"{prefix}subs-{t}", q(15, 12), 0.3, dict(seed=5, subsets=True, ties=ties)),
                r(f"{prefix}subs0-{t}", q(16, 9), 0.0, dict(seed=6, subsets=True, within=[0, per // 2], ties=ties)),
                r(f"{prefix}ties-{t}", q(17, 16, favour=10), 0.5, dict(seed=7, ties=ties))]
    ops += [dict(op="fuzzy0", key=prefix + "fuzzy0", q=q(18, 1, favour=10), ms=0.5),
            dict(op="arrays", key=prefix + "arrays-all", q=q(19, 4), k=n, ms=0.55, filters=dict(seed=0)),
            dict(op="arrays", key=prefix + "arrays-subs", q=q(20, 200), k=3000, ms=0.0,
                 filters=dict(seed=8, subsets=True))]  # the longest subsets pass 2048 entries
    return ops


def storage_case(world: int, storage: str) -> dict:
    n = {2: 10001, 3: 15007, 8: 8 * 1300 + 5}[world]
    cspec = dict(n=n, d=D, seed=2100 + world, preset="coarse" if storage == "bfloat16" else "fine",
                 dup=boundary_dups(n, world))
    return dict(name=storage, storage=storage, corpus=cspec, ops=range_ops(cspec, corpus(cspec), n, world))


def sizes_case(world: int) -> dict:
    """A retention of 32768 hits per rank: a search that grows the inbox (4096 -> 32768), the same search again in
    one round, one that grows past the retention and gives the excess back, then a small one.  Deferred top-k
    lookups are outstanding before and after the threshold searches and finished at the end."""
    n = 4500 * world + 7
    cspec = dict(n=n, d=D, seed=2300 + world, preset="fine", dup=boundary_dups(n, world))
    retain_hits = 32768
    ops = [dict(op="search", key="d0", q=q(2400, 16), k=10, ms=0.0, defer=True),
           dict(op="search", key="d1", q=q(2401, 3), k=7, ms=0.0, defer=True),
           r("grow", q(2402, 4), 0.0, rounds=2, cap=retain_hits),
           r("again", q(2403, 4), 0.0, rounds=1, cap=retain_hits),
           dict(op="search", key="d2", q=q(2404, 16), k=12, ms=0.0, defer=True),
           r("big", q(2405, 16), 0.0, rounds=2, cap=retain_hits),
           # grows past the retention, and the last rank cannot allocate the merged result: it alone raises, and
           # every rank still gives the excess back
           dict(op="ofail", key="ofail", q=q(2408, 16), ms=0.0, filters=dict(seed=0), cap_rank=world - 1),
           r("small", q(2406, 2), 0.6, rounds=1, cap=retain_hits, retained=True),
           dict(op="search", key="d3", q=q(2407, 5), k=9, ms=0.0, defer=True),
           dict(op="finish", key="fin", expect="any")]
    return dict(name="sizes", storage="bfloat16", corpus=cspec, ops=ops, retain=12 * world * retain_hits)


def empty_case(world: int) -> dict:
    """Rank 0's whole block removed: it has no rows and publishes empty lists."""
    n = 4500 * world + 9
    per = -(-n // world)
    cspec = dict(n=n, d=D, seed=2500 + world, preset="fine")
    v = corpus(cspec)
    ops = [dict(op="remove", key="rm", ordinals=list(range(per)))]
    rows = len(v) - per  # the filters are drawn over the rows left
    ops += [r("e-all", q(2501, 3), 0.0), r("e-row", q(2502, 16), 0.5, dict(seed=9, allowed=True), rows=rows),
            r("e-sub", q(2503, 16), 0.3, dict(seed=10, subset=True), rows=rows),
            dict(op="fuzzy0", key="e-fuzzy0", q=q(2504, 1), ms=0.5)]
    return dict(name="empty", storage="float16", corpus=cspec, ops=ops, removed=per)


def failure_case(world: int) -> dict:
    """One rank's per-query mask upload fails past the upload agreement: its local search publishes status 1 and
    every rank raises.  Then one rank's inbox may not grow, and a search needs a grow: every rank raises
    MemoryError and holds no inbox.  Then one rank cannot allocate the merged result after the rounds: it alone
    raises, its round acknowledged.  The searches after each failure are exact."""
    n = 5000 * world + 1
    cspec = dict(n=n, d=D, seed=2700 + world, preset="fine")
    v = corpus(cspec)
    last = world - 1
    few = top_ms(cspec, v, q(50, 16), 2000)  # fits in the first inbox: no rank grows after a failure
    ops = [dict(op="rfail", key="rfail", q=q(50, 16), ms=few, filters=dict(seed=50, masks=True), cap_rank=last),
           r("after", q(51, 16), 0.0, dict(seed=51, masks=True)),
           dict(op="gfail", key="gfail", q=q(52, 64), ms=0.0, filters=dict(seed=0), cap_rank=last),
           r("after2", q(53, 16), 0.0), r("after3", q(54, 16), few),
           dict(op="ofail", key="ofail", q=q(55, 16), ms=few, filters=dict(seed=0), cap_rank=last),
           r("after4", q(56, 16), few), r("after5", q(57, 16), 0.0)]
    return dict(name="failure", storage="bfloat16", corpus=cspec, ops=ops)


FAIL_EXPECT = {"rfail": (1, 2), "gfail": (1, 1), "ofail": (1, 0)}  # (failing rank, others): 1 MemoryError, 2 RuntimeError


def cases_for(world: int) -> list[dict]:
    if world == 8:
        return [storage_case(8, "bfloat16")]
    return ([storage_case(world, st) for st in ("bfloat16", "float16", "float32")]
            + [sizes_case(world), empty_case(world), failure_case(world)])


# ---------------------------------------------------------------- expectations
def expectations(case: dict) -> dict:
    """key -> what one VectorBase over the whole corpus (after the case's removal) returns for the operation."""
    import typeagent_py_b200 as tab
    from oracle import vectorbase_oracle as O

    cspec = case["corpus"]
    v = corpus(cspec)
    whole = tab.VectorBase(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()), storage_dtype=case["storage"])
    whole.add_embeddings(None, v)
    if case.get("removed"):
        whole.remove_embeddings(np.arange(case["removed"]))
    out = {}
    for op in case["ops"]:
        if op["op"] not in ("range", "fuzzy0", "arrays", "search", "ofail"):
            continue
        qq = queries(op["q"], cspec, v)
        f = filters(op.get("filters", {"seed": 0}), op.get("rows", len(v)), len(qq))
        if op["op"] in ("range", "ofail"):
            out[op["key"]] = whole.search_range(qq, op["ms"], **f)
        elif op["op"] == "fuzzy0":
            hits = whole.fuzzy_lookup_embedding(qq[0], 0, op["ms"])
            out[op["key"]] = (np.array([0, len(hits)], np.int64), np.array([h.item for h in hits], np.int64),
                              np.array([h.score for h in hits], np.float32))
        else:
            out[op["key"]] = whole.search_arrays(qq, op["k"], op["ms"], **f)
    return out


def fields(op: dict) -> tuple[str, ...]:
    return ("items", "scores", "counts") if op["op"] in ("arrays", "search") else ("offsets", "items", "scores")


def mismatches(case: dict, want: dict, world: int, out: str) -> list[str]:
    errors = []
    for rk in range(world):
        got = np.load(os.path.join(out, f"{case['name']}.r{rk}.npz"))
        for op in case["ops"]:
            key = op["key"]
            try:
                if key in want and not (op["op"] == "ofail" and rk == op["cap_rank"]):
                    names = fields(op)
                    g = [got[f"{key}.{f}"] for f in names]
                    for a, w, name in zip(g, want[key], names):
                        a, w = np.asarray(a), np.asarray(w)
                        if a.dtype == np.float32:
                            a, w = a.view(np.uint32), w.view(np.uint32)
                        assert a.shape == w.shape and (a == w).all(), \
                            f"rank {rk} {key}: {name} differ ({a.shape} vs {w.shape})"
                if "rounds" in op:
                    rounds = int(got[key + ".rounds"][0])
                    assert rounds == op["rounds"], f"rank {rk} {key}: {rounds} rounds, expected {op['rounds']}"
                if "cap" in op:
                    cap, group, process = (int(x) for x in got[key + ".inbox"])
                    assert cap == op["cap"], f"rank {rk} {key}: inbox capacity {cap}, expected {op['cap']}"
                    assert group == process, f"rank {rk} {key}: {process} inbox bytes in the process, {group} in use"
                    if op.get("retained"):
                        assert group <= case["retain"] + (1 << 16), \
                            f"rank {rk} {key}: the inbox keeps {group} bytes, above the retention {case['retain']}"
                if op["op"] in FAIL_EXPECT:
                    e = FAIL_EXPECT[op["op"]]
                    want_code = e[0] if rk == op["cap_rank"] else e[1]
                    code = int(got[key + ".codes"][0])
                    assert code == want_code, f"rank {rk} {key}: raised {code}, expected {want_code}"
                    if op["op"] == "gfail":
                        assert tuple(int(x) for x in got[key + ".inbox"]) == (0, 0, 0), \
                            f"rank {rk} {key}: an inbox survived the failed grow"
            except (AssertionError, KeyError) as ex:
                errors.append(str(ex))
    return errors


_RUNS: dict = {}


def run_world(world: int, lib: str | None = None):
    """The ranks of one world over all its cases, launched once per session."""
    if (world, lib) not in _RUNS:
        cases = cases_for(world) if lib is None else [sizes_case(2), failure_case(2), storage_case(2, "bfloat16")]
        want = {c["name"]: expectations(c) for c in cases}
        tmp = tempfile.mkdtemp(prefix=f"tav_peer_range_w{world}_")
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


CASE_NAMES = ["bfloat16", "float16", "float32", "sizes", "empty", "failure"]


@pytest.mark.parametrize("name", CASE_NAMES)
@pytest.mark.parametrize("world", [2, 3])
def test_peer_range_equals_one_vectorbase(world, name):
    errors = run_world(world)[name]
    assert not errors, "\n".join(errors[:20])


def test_peer_range_eight_ranks():
    errors = run_world(8)["bfloat16"]
    assert not errors, "\n".join(errors[:20])


# ---------------------------------------------------------------- broken builds
MUTANTS = {1: "last hit vector not published", 2: "republish without hits", 3: "status words not summed"}


@pytest.fixture(scope="module")
def mutant_libs():
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc) and not shutil.which(nvcc):
        pytest.skip("nvcc is needed to build the broken variants")
    from typeagent_py_b200 import build as B

    tmp = tempfile.mkdtemp(prefix="tav_peer_range_mutants_")
    procs = {}
    for m in MUTANTS:
        out = os.path.join(tmp, f"libtavec_peer_range_mutant{m}.so")
        cmd = [nvcc, *[f for f in B.NVCC_FLAGS if f != "-Xptxas=-v"], f"-DTAV_PEER_RANGE_MUTANT={m}", "-o", out,
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
