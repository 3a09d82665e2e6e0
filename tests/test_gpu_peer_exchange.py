"""The peer-memory exchange of ``ShardedVectorBase(exchange="peer")`` on one GPU, bit for bit.

W processes (tests/peer_ranks.py) share the device (``rank % device_count`` when more are visible) and form one
group over CUDA IPC, so every group search runs the whole product path: the local search into the rank's slot,
``publish_kernel`` storing it into every peer's region, ``merge_kernel<0>`` waiting for every rank, merging,
acknowledging and adding up the slot tails, and ``tav_sharded_finish`` repairing what some rank corrected.  The
ranks run on dyadic corpora (tests/exact.py), so every rank's items, score bits and counts must equal the exact
top-k of the exact dots (``exact.expected_topk``: equal scores higher row first), which this test computes, and
checks against one ``VectorBase`` over the whole corpus, before it launches the ranks.

Cases, at W = 2 and 3 with uneven blocks and one at W = 8: bf16 / fp16 / float32 (split form and row scan), B = 1,
16, 129, 1029, k = 1, 10, 100, 2048 and one above 2048, min_score at a hit and one ulp either side, rows copied
across block boundaries; 22 searches in a row (slots reused, counts varying); eight deferred searches and one
finish, a ninth refused, deferred searches before a synchronous one, a non-default stream; the group rebuilt
for a larger batch or k with deferred searches outstanding; ranks without rows; the repair of searches that one
rank flags (21,500 copies of one row in its block), alone and as the middle of three deferred searches; and a
float32 corpus with a value beyond the fp16 range in one block, whose split-form searches only the owning rank
redoes.  Three deliberately broken builds (``TAV_GROUP_MUTANT``) are each caught.
"""

from __future__ import annotations

import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np
import pytest

from tests.exact import expected_topk
from tests.peer_ranks import corpus, queries

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "peer_ranks.py")
D = 64


# ---------------------------------------------------------------- cases
def boundary_dups(n: int, world: int) -> list[list[int]]:
    """Rows [0, 80) copied to the 80 rows around every block boundary, rows [100, 400) spread over the other
    blocks: equal scores on different ranks, on both sides of each boundary."""
    per = -(-n // world)
    dup = [[g * per - 40 + j, j] for g in range(1, world) for j in range(80)]
    rng = np.random.default_rng(n + world)
    dst = rng.choice(np.arange(per, n - 50), size=300, replace=False)
    taken = {d for d, _ in dup}
    dup += [[int(d), 100 + i] for i, d in enumerate(dst) if int(d) not in taken]
    return dup


def q(seed, b, **kw):
    return dict(seed=seed, b=b, **kw)


def s(key, qs, k, ms=0.0, **kw):
    return dict(op="search", key=key, q=qs, k=k, ms=float(ms), **kw)


def fin(key, expect="any"):
    return dict(op="finish", key=key, expect=expect)


def ulp_cases(cspec, v, key, seed, b, k):
    """min_score exactly at the 10th hit of query 0, and one float32 ulp below and above it."""
    qs = q(seed, b, favour=10)
    qq = queries(qs, cspec, v)
    at = expected_topk(dots_of(qq[:1], v), 10, 0.0)[1][0, 9]
    return [s(f"{key}-{name}", qs, k, ms) for name, ms in
            (("at", at), ("below", np.nextafter(at, np.float32(0))), ("above", np.nextafter(at, np.float32(2))))]


def storage_case(world: int, storage: str) -> dict:
    n = {2: 10001, 3: 15007}[world]
    cspec = dict(n=n, d=D, seed=100 + world, preset="coarse" if storage == "bfloat16" else "fine",
                 dup=boundary_dups(n, world))
    v = corpus(cspec)
    shapes = [(1, 1), (1, 100), (16, 10), (16, 2048), (129, 100), (129, 1), (1029, 10), (1029, 100), (16, 3000)]
    if storage == "bfloat16":
        shapes.append((1029, 2048))
    ops = [s(f"B{b}-k{k}", q(7 * b + k, b, favour=10 if b > 1 else None), k) for b, k in shapes]
    ops += ulp_cases(cspec, v, "ms", 5, 16, 100) + ulp_cases(cspec, v, "ms1", 6, 1, 100)
    return dict(name=f"{storage}", storage=storage, corpus=cspec, ops=ops)


def slot_reuse_case(world: int) -> dict:
    """22 synchronous searches in a row (depth 8: the acks are waited for from the 9th on), the batch, k and
    min_score changing every time, so that no slot holds the counts the next search there produces."""
    n = 4500 * world + 3
    # scores spread below the clip at 1.0, so that a min_score at a hit cuts the counts
    cspec = dict(n=n, d=D, seed=200 + world, preset="scale", dup=boundary_dups(n, world))
    v = corpus(cspec)
    ops = []
    for i in range(22):
        b = (16, 20, 37, 5, 64, 1, 16, 33)[i % 8]
        k = 3 + (5 * i) % 14
        qs = q(300 + i, b)
        rank = 1 + (3 * i) % (k + 4)  # min_score at query 0's rank-th hit: counts below and at k
        ms = expected_topk(dots_of(queries(qs, cspec, v)[:1], v), rank + 1, 0.0)[1][0, rank]
        ops.append(s(f"s{i}", qs, k, ms))
    return dict(name="slot_reuse", storage="bfloat16", corpus=cspec, ops=ops)


def pipeline_case(world: int) -> dict:
    n = 4500 * world + 7
    cspec = dict(n=n, d=D, seed=300 + world, preset="fine", dup=boundary_dups(n, world))
    ops = [s(f"d{i}", q(400 + i, 16 + 3 * i), 5 + i, defer=True) for i in range(8)]
    ops += [dict(op="raise", key="ninth", q=q(499, 16), k=10, ms=0.0), fin("eight")]
    ops += [s("after", q(410, 17), 11)]
    ops += [s("dd0", q(420, 16), 9, defer=True), s("dd1", q(421, 40), 16, defer=True), s("sync", q(422, 24), 12)]
    ops += [s("st-d0", q(430, 16), 10, defer=True, stream=True), s("st-d1", q(431, 19), 7, defer=True, stream=True),
            fin("st-finish"), s("st-sync", q(432, 16), 16, stream=True)]
    return dict(name="pipeline", storage="bfloat16", corpus=cspec, ops=ops)


def growth_case(world: int) -> dict:
    """A batch beyond cap_q (256) and a k beyond cap_k (16) rebuild the group, with deferred searches outstanding:
    they are finished first."""
    n = 4500 * world + 11
    cspec = dict(n=n, d=D, seed=400 + world, preset="fine", dup=boundary_dups(n, world))
    ops = [s("g0", q(500, 16), 10, defer=True), s("g1", q(501, 16), 10, defer=True), s("big-b", q(502, 300), 10),
           fin("after-b"), s("big-k", q(503, 16), 17), s("g2", q(504, 16), 10, defer=True),
           s("g3", q(505, 20), 40, defer=True), fin("after-k"), s("g4", q(506, 600), 16, defer=True),
           s("g5", q(507, 16), 100)]
    return dict(name="growth", storage="bfloat16", corpus=cspec, ops=ops)


def empty_cases(world: int) -> list[dict]:
    """A rank with no rows: N < W at deserialize (then an append fills the last block), and a block emptied by
    remove_embeddings."""
    small = dict(n=64, d=D, seed=500 + world, preset="fine")
    few = dict(name="fewer_rows_than_ranks", storage="float32", corpus=small, load=world - 1,
               ops=[s("b1", q(600, 1), 10), s("b16", q(601, 16), 10), s("d", q(602, 16), 4, defer=True), fin("f"),
                    dict(op="append", key="append", q=q(603, 4), take=3), s("found", q(603, 4), 10),
                    s("found16", q(603, 16), 2)])
    n = 5000 * world
    big = dict(n=n, d=D, seed=600 + world, preset="fine", dup=boundary_dups(n, world))
    removed = dict(name="emptied_block", storage="bfloat16", corpus=big,
                   ops=[s("before", q(610, 16), 10),
                        dict(op="remove", key="remove", ordinals=list(range(5000, 10000))),
                        s("b16", q(611, 16), 10), s("b1", q(612, 1), 10), s("d0", q(613, 16), 10, defer=True),
                        s("d1", q(614, 32), 20, defer=True), fin("f"),
                        dict(op="append", key="append", q=q(615, 2), take=2), s("found", q(615, 16), 5)])
    return [few, removed]


def repair_case(world: int) -> dict:
    """The last rank's block ends in 21,500 copies of row 100: its tensor-core search flags the queries that favour
    that row (candidate overflow) and finish redoes them exactly; the other ranks do not flag.  Every rank learns
    it from the slot tails alone."""
    per = 22000
    cspec = dict(n=per * world, d=D, seed=700 + world, preset="fine", copies=[100, per * (world - 1) + 500, per * world])
    fav = lambda seed, b: q(seed, b, favour=100)  # noqa: E731
    away = lambda seed, b: q(seed, b, against=100)  # noqa: E731
    ops = [s("sync", fav(800, 16), 10),
           s("soloA", away(801, 16), 10, defer=True), fin("soloA", "zero"),
           s("soloB", fav(802, 20), 8, defer=True), fin("soloB", "positive"),
           s("soloC", away(803, 16), 12, defer=True), fin("soloC", "zero"),
           s("A", away(801, 16), 10, defer=True), s("B", fav(802, 20), 8, defer=True),
           s("C", away(803, 16), 12, defer=True), fin("ABC", "positive"),
           s("sync2", fav(804, 32), 100)]
    return dict(name="repair", storage="bfloat16", corpus=cspec, ops=ops)


def split_case(world: int) -> dict:
    """float32 rows, one of them 2^17 in column 5 (beyond the fp16 range) in the last rank's block: its split-form dots
    are NaN, so the owning rank redoes every query of every split search at finish, and every rank must learn
    that from the tails.  Its exact score is 1.0 for these queries, whatever the summation order."""
    per = 6000
    big = per * world - 10
    cspec = dict(n=per * world, d=D, seed=800 + world, preset="fine", big=[[big, 5]])
    ops = [s("sync16", q(900, 16, big_col=5), 10, contains=big), s("sync32", q(901, 32, big_col=5), 100, contains=big),
           s("d16", q(902, 16, big_col=5), 10, defer=True, contains=big),
           s("d20", q(903, 20, big_col=5), 50, defer=True, contains=big),
           fin("d", "at_least_36"), s("scan1", q(904, 1, big_col=5), 10, contains=big)]
    return dict(name="split_overflow", storage="float32", corpus=cspec, ops=ops)


def cases_for(world: int) -> list[dict]:
    if world == 8:
        n = 8 * 4200 + 5
        cspec = dict(n=n, d=D, seed=8, preset="coarse", dup=boundary_dups(n, 8))
        return [dict(name="w8", storage="bfloat16", corpus=cspec,
                     ops=[s("B16", q(1, 16, favour=10), 100), s("B129", q(2, 129), 10), s("B1029", q(3, 1029), 16),
                          s("B1", q(4, 1, favour=20), 10), s("d0", q(5, 16), 10, defer=True),
                          s("d1", q(6, 64), 33, defer=True), fin("f", "any")])]
    return ([storage_case(world, st) for st in ("bfloat16", "float16", "float32")] + [slot_reuse_case(world),
            pipeline_case(world), growth_case(world)] + empty_cases(world) + [repair_case(world), split_case(world)])


# ---------------------------------------------------------------- expectations
def dots_of(qq: np.ndarray, v: np.ndarray) -> np.ndarray:
    """Exact dots as float32: dyadic inputs make every product and partial sum exact in float64 too."""
    return (qq.astype(np.float64) @ v.astype(np.float64).T).astype(np.float32)


def expectations(case: dict, check_whole: bool = True) -> dict:
    """key -> (items, scores, counts) of every search of the case over the corpus as it stands at that point,
    with one VectorBase over that corpus as a second witness."""
    import typeagent_py_b200 as tab
    from oracle import vectorbase_oracle as O

    cspec = case["corpus"]
    v0 = corpus(cspec)
    cur = v0[: case.get("load", len(v0))]
    whole = None
    out = {}
    for op in case["ops"]:
        if op["op"] == "remove":
            cur = np.delete(cur, op["ordinals"], axis=0)
            whole = None
        elif op["op"] == "append":
            cur = np.concatenate([cur, queries(op["q"], cspec, v0)[: op["take"]]])
            whole = None
        elif op["op"] == "search":
            qq = queries(op["q"], cspec, v0)
            k = max(1, min(op["k"], max(len(cur), 1)))
            want = expected_topk(dots_of(qq, cur), k, np.float32(op["ms"]))
            if "contains" in op:  # the case is only a test if the row it is about is in every expected list
                assert (want[0] == op["contains"]).any(axis=1).all(), f"{case['name']}/{op['key']}"
            if check_whole:
                if whole is None:
                    whole = tab.VectorBase(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()),
                                           storage_dtype=case["storage"])
                    whole.add_embeddings(None, cur)
                assert_same(whole.search_arrays(qq, k, op["ms"]), want, f"{case['name']}/{op['key']}: one VectorBase")
            out[op["key"]] = want
    return out


def assert_same(got, want, what):
    for g, w, name in zip(got, want, ("items", "scores", "counts")):
        g, w = np.asarray(g), np.asarray(w)
        if g.dtype == np.float32:
            g, w = g.view(np.uint32), w.view(np.uint32)
        assert g.shape == w.shape, f"{what}: {name} shape {g.shape} != {w.shape}"
        bad = np.flatnonzero((g != w).reshape(len(g), -1).any(axis=1)) if g.ndim else []
        assert len(bad) == 0, f"{what}: {name} differ in {len(bad)} of {len(g)} queries, first {bad[:5].tolist()}"


def mismatches(case: dict, want: dict, world: int, out: str) -> list[str]:
    """Every way the ranks' outputs of ``case`` differ from the expectation (empty: all equal)."""
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
    for op in case["ops"]:
        if op["op"] != "finish":
            continue
        counts = finishes[op["key"]]
        ok = {"zero": counts[0] == 0, "positive": counts[0] > 0, "at_least_36": counts[0] >= 36,
              "any": True}[op["expect"]]
        if len(set(counts)) != 1 or not ok:
            errors.append(f"finish {op['key']}: counts {counts} per rank, expected {op['expect']} on every rank")
    return errors


# ---------------------------------------------------------------- launching the ranks
def launch(world: int, cases: list[dict], tmp: str, lib: str | None = None, timeout: float = 900) -> str:
    """Run the ranks over ``cases``; returns the output directory.  Every rank is waited for, killed at the
    deadline and reaped: no process outlives this call."""
    out = os.path.join(tmp, "out")
    os.makedirs(out, exist_ok=True)
    spec_path = os.path.join(tmp, "spec.json")
    with open(spec_path, "w") as f:
        json.dump(dict(world=world, store=os.path.join(tmp, "store"), out=out, lib=lib, cases=cases), f)
    env = dict(os.environ, GLOO_SOCKET_IFNAME="lo")
    py = [sys.executable] + (["-s"] if sys.flags.no_user_site else [])
    logs = [open(os.path.join(tmp, f"rank{r}.log"), "w") for r in range(world)]
    procs = []
    try:
        for r in range(world):
            procs.append(subprocess.Popen(py + [WORKER, spec_path, str(r)], stdout=logs[r], stderr=subprocess.STDOUT,
                                          cwd=ROOT, env=env))
        deadline = time.monotonic() + timeout
        for p in procs:
            p.wait(timeout=max(1.0, deadline - time.monotonic()))
    except subprocess.TimeoutExpired:
        pass
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
        for p in procs:
            p.wait()
        for f in logs:
            f.close()
    tails = []
    for r, p in enumerate(procs):
        with open(os.path.join(tmp, f"rank{r}.log")) as f:
            tails.append(f"--- rank {r} (exit {p.returncode}) ---\n" + f.read()[-3000:])
    statuses = []
    for r in range(world):
        path = os.path.join(out, f"status.r{r}.json")
        assert os.path.exists(path), "a rank ended without its status:\n" + "\n".join(tails)
        with open(path) as f:
            statuses.append(json.load(f))
    if any(st.get("preflight") for st in statuses):
        pytest.skip("ranks cannot share the device: " + statuses[0]["preflight"])
    for st in statuses:
        for name, status in st["cases"].items():
            assert status == "ok", f"rank {st['rank']} case {name}:\n{status}"
    for p in procs:
        assert p.returncode == 0, "\n".join(tails)
    return out


# world -> ("ok", (cases, expectations, output directory)) | ("skip", reason) | ("fail", what went wrong): the
# outcome of the one launch of that world's ranks.  A failed launch is never repeated in the session: a fault
# that made a rank stop would only happen again.
_RUNS: dict = {}


@pytest.fixture(scope="module", autouse=True)
def _remove_outputs():
    yield
    for kind, value in _RUNS.values():
        if kind == "ok":
            shutil.rmtree(os.path.dirname(value[2]), ignore_errors=True)
    _RUNS.clear()


def _launch_world(world: int) -> tuple[list[dict], dict, str]:
    import torch

    cases = cases_for(world)
    want = {c["name"]: expectations(c) for c in cases}
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    tmp = tempfile.mkdtemp(prefix=f"tav_peer_w{world}_")
    t0 = time.monotonic()
    try:
        out = launch(world, cases, tmp)
    except BaseException:
        shutil.rmtree(tmp, ignore_errors=True)
        raise
    used = max(int(np.load(os.path.join(out, f"{c['name']}.r0.npz"))["device_used_bytes"][0]) for c in cases)
    print(f"\npeer exchange W={world}: {len(cases)} cases in {time.monotonic() - t0:.1f} s, "
          f"device memory in use at most {used / 2**30:.2f} GiB (all ranks, read after every operation)")
    return cases, want, out


def run_world(world: int) -> tuple[list[dict], dict, str]:
    """The ranks of one world over all its cases, launched once per session: (cases, expectations, output
    directory).  The tests after a skipped or failed launch skip or fail from its recorded outcome."""
    if world not in _RUNS:
        try:
            _RUNS[world] = ("ok", _launch_world(world))
        except pytest.skip.Exception as e:
            _RUNS[world] = ("skip", str(e))
            raise
        except (Exception, pytest.fail.Exception) as e:
            _RUNS[world] = ("fail", f"{type(e).__name__}: {e}")
            raise
    kind, value = _RUNS[world]
    if kind == "skip":
        pytest.skip(value)
    if kind == "fail":
        pytest.fail(f"the W={world} ranks failed earlier in this session and are not launched again:\n{value[:3000]}")
    return value


CASE_NAMES = ["bfloat16", "float16", "float32", "slot_reuse", "pipeline", "growth", "fewer_rows_than_ranks",
              "emptied_block", "repair", "split_overflow"]


@pytest.mark.parametrize("name", CASE_NAMES)
@pytest.mark.parametrize("world", [2, 3])
def test_peer_exchange_equals_exact_topk(world, name):
    cases, want, out = run_world(world)
    case = next(c for c in cases if c["name"] == name)
    errors = mismatches(case, want[name], world, out)
    assert not errors, "\n".join(errors[:20])


def test_peer_exchange_eight_ranks():
    cases, want, out = run_world(8)
    errors = mismatches(cases[0], want[cases[0]["name"]], 8, out)
    assert not errors, "\n".join(errors[:20])


# ---------------------------------------------------------------- broken builds
MUTANTS = {1: "tail always zero", 2: "last 16 bytes of the list not published", 3: "repair without the slot copy"}


@pytest.fixture(scope="module")
def mutant_libs():
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc) and not shutil.which(nvcc):
        pytest.skip("nvcc is needed to build the broken variants")
    from typeagent_py_b200 import build as B

    tmp = tempfile.mkdtemp(prefix="tav_group_mutants_")
    procs = {}
    for m in MUTANTS:
        out = os.path.join(tmp, f"libtavec_group_mutant{m}.so")
        cmd = [nvcc, *[f for f in B.NVCC_FLAGS if f != "-Xptxas=-v"], f"-DTAV_GROUP_MUTANT={m}", "-o", out,
               *[os.path.join(B.CSRC, src) for src in B.SOURCES]]
        procs[m] = (subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True), out)
    libs = {}
    for m, (proc, out) in procs.items():
        log = proc.communicate()[0]
        assert proc.returncode == 0, log
        libs[m] = out
    yield libs
    shutil.rmtree(tmp, ignore_errors=True)


def mutant_cases() -> list[dict]:
    return [slot_reuse_case(2), repair_case(2)]


@pytest.mark.parametrize("m", sorted(MUTANTS), ids=[MUTANTS[m].replace(" ", "_") for m in sorted(MUTANTS)])
def test_broken_build_is_caught(mutant_libs, m):
    failed = [w for w, (kind, _) in _RUNS.items() if kind == "fail"]
    if failed:
        pytest.skip(f"the real build failed at W={failed}: its broken variants are not launched")
    cases = mutant_cases()
    want = {c["name"]: expectations(c, check_whole=False) for c in cases}
    tmp = tempfile.mkdtemp(prefix=f"tav_peer_mutant{m}_")
    try:
        out = launch(2, cases, tmp, lib=mutant_libs[m])
        caught = [e for c in cases for e in mismatches(c, want[c["name"]], 2, out)]
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    assert caught, f"the exact checks did not catch: {MUTANTS[m]}"
