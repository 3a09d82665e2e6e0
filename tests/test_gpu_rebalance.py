"""``ShardedVectorBase.rebalance`` on one GPU, bit for bit: W processes (tests/rebalance_ranks.py) share the device and
form a real group over CUDA IPC, so every rank's new block is copied from its peers' row allocations as it would be
across NVLink, and the peer exchange searches the blocks afterwards.

Appends skew the last block and a removal empties the first; then ``rebalance()`` (and ``rebalance(sizes)``) moves
the rows.  On dyadic corpora (tests/exact.py), before and after, every rank's peer-exchange searches (tensor cores
and row scan), filtered, per-query-mask, subset and threshold lookups must equal the exact results over the whole
corpus, and every rank's host mirror (``serialize()``) and device rows (``tav_read_rows``) must equal its new block of
the corpus.  Cases at W = 2 and 3: bf16, fp16 and float32 storage, float32 searched through the fp16 planes with and
without a row beyond the fp16 range that moves to another rank, a ``TAV_NORMALIZE`` index (its normalised rows must move unchanged),
a stage that runs out of memory on one rank (``tav_internal_stage_cap``: every rank raises MemoryError, nothing
changes, and the next rebalance succeeds), and a row mask that must not survive the rows it was set for; one case
at W = 8.  After a rebalance each rank's process holds exactly one row block, its new one, sized to its rows
(``tav_internal_row_bytes`` counts every row allocation and free), and the row blocks its process holds changed by
exactly as much as its index's: the old and staged blocks are freed.  Four broken builds
(``TAV_REBALANCE_MUTANT``) are each caught.
"""

from __future__ import annotations

import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

import tests.test_gpu_peer_exchange as peer
from tests.exact import expected_topk
from tests.peer_ranks import corpus, queries
from tests.rebalance_ranks import lookup_args
from tests.test_sharded_filter_gloo import oracle_arrays, oracle_csr
from tests.test_sharded_query_masks_gloo import as_arrays, as_csr, per_query
from tests.test_sharded_subsets_gloo import oracle_batch_arrays

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "rebalance_ranks.py")
D = 64


def q(seed, b, **kw):
    return dict(seed=seed, b=b, **kw)


def s(key, qs, k, ms=0.0, **kw):
    return dict(op="search", key=key, q=qs, k=k, ms=float(ms), **kw)


def skewed_ops(world: int, n0: int, grow: int, seed: int, big_col=None, k=10, force=None) -> list[dict]:
    """Appends that put ``grow`` rows on the last rank, a removal that empties the first block, then searches,
    lookups and rows before and after ``rebalance()`` and ``rebalance(sizes)``."""
    per = -(-n0 // world)
    kw = {} if big_col is None else dict(big_col=big_col)
    fk = {} if force is None else dict(force=force)
    ops = [dict(op="append", key=f"a{i}", q=q(seed + i, grow // 3), take=grow // 3) for i in range(3)]
    ops += [dict(op="remove", key="empty0", ordinals=list(range(per)))]
    ops += [s("s-before", q(seed + 10, 16, **kw), k, **fk), s("s1-before", q(seed + 11, 1, **kw), k),
            dict(op="rows", key="rows-before"), dict(op="lookups", key="l-before", q=q(seed + 12, 5), seed=seed, k=k,
                                                     ms=0.0),
            dict(op="rebalance", key="rb"),
            s("s-after", q(seed + 10, 16, **kw), k, **fk), s("s1-after", q(seed + 11, 1, **kw), k),
            s("d-after", q(seed + 13, 40, **kw), 33, defer=True, **fk), dict(op="finish", key="f-after", expect="any"),
            dict(op="rows", key="rows-after", same_as="rows-before"),
            dict(op="lookups", key="l-after", q=q(seed + 12, 5), seed=seed, k=k, ms=0.0),
            dict(op="rebalance", key="rb-noop")]
    return ops


def sizes_ops(world: int, n: int, seed: int) -> list[dict]:
    sizes = [0] * world
    sizes[-1 if world == 2 else 1] = n
    return [dict(op="rebalance", key="rs", sizes=sizes), s("s-sizes", q(seed + 20, 16), 10),
            dict(op="rows", key="rows-sizes"), dict(op="lookups", key="l-sizes", q=q(seed + 21, 3), seed=seed + 1,
                                                      k=100, ms=0.5)]


def storage_case(world: int, storage: str) -> dict:
    n0, grow = 3000 * world, 2400 * world
    cspec = dict(n=n0, d=D, seed=40 + world, preset="coarse" if storage == "bfloat16" else "fine")
    ops = skewed_ops(world, n0, grow, 1000) + sizes_ops(world, n0 - (-(-n0 // world)) + grow, 1000)
    return dict(name=storage, storage=storage, corpus=cspec, ops=ops)


def split_case(world: int, big: bool = True) -> dict:
    """float32 through the fp16 planes (tensor cores forced).  With ``big`` the appended rows hold a 2^17 value that
    a rebalance moves off the last rank (whose split searches are then all redone exactly, at finish, while it holds
    that row); without it the last rank's planes, built over its old block, would answer wrongly if they survived."""
    n0, grow = 2000 * world, 1800 * world
    cspec = dict(n=n0 + grow, d=D, seed=60 + world, preset="fine", big=[[n0 + 5, 7]] if big else [])
    ops = skewed_ops(world, n0, grow, 2000, big_col=7 if big else None, force="mma")
    # the appended rows come from the corpus itself here, so that the 2^17 row is among them
    for i, op in enumerate(op for op in ops if op["op"] == "append"):
        op.update(rows=[n0 + i * (grow // 3), n0 + (i + 1) * (grow // 3)])
    return dict(name="split_overflow" if big else "split", storage="float32", corpus=cspec, load=n0, ops=ops)


def normalize_case(world: int) -> dict:
    n0, grow = 1500 * world, 1500 * world
    cspec = dict(n=n0, d=D, seed=70 + world, preset="coarse")
    ops = [dict(op="append", key="a", q=q(7000, grow), take=grow), dict(op="rows", key="rows-before"),
           dict(op="rebalance", key="rb"), dict(op="rows", key="rows-after", same_as="rows-before", normalized=True)]
    return dict(name="normalize", storage="bfloat16", normalize=True, corpus=cspec, ops=ops)


def oom_case(world: int) -> dict:
    n0, grow = 2000 * world, 2000 * world
    cspec = dict(n=n0, d=D, seed=80 + world, preset="coarse")
    ops = [dict(op="append", key="a", q=q(8000, grow), take=grow), dict(op="rows", key="rows-before"),
           dict(op="rebalance", key="rb-oom", cap_rank=world - 1, expect_raise=1),
           dict(op="rows", key="rows-unchanged", same_as="rows-before"), s("s-unchanged", q(8001, 16), 10),
           dict(op="rebalance", key="rb"), dict(op="rows", key="rows-after", same_as="rows-before"),
           s("s-after", q(8001, 16), 10)]
    return dict(name="oom", storage="bfloat16", corpus=cspec, ops=ops)


def mask_case() -> dict:
    """W = 3: blocks of 500, 500 and 1000 rows, then sizes (1000, 500, 500): rank 1 keeps 500 rows, but other ones.
    The row mask set on every rank's index before must not be usable afterwards."""
    cspec = dict(n=1500, d=D, seed=90, preset="coarse")
    ops = [dict(op="append", key="a", q=q(9000, 500), take=500), dict(op="mask", key="mask"),
           dict(op="rebalance", key="rs", sizes=[1000, 500, 500]), dict(op="maskprobe", key="probe", q=q(9001, 1)),
           dict(op="rows", key="rows-after")]
    return dict(name="row_mask", storage="bfloat16", corpus=cspec, ops=ops)


def cases_for(world: int) -> list[dict]:
    if world == 8:
        return [storage_case(8, "bfloat16")]
    out = [storage_case(world, st) for st in ("bfloat16", "float16", "float32")]
    out += [split_case(world), split_case(world, big=False), normalize_case(world), oom_case(world)]
    if world == 3:
        out.append(mask_case())
    return out


# ---------------------------------------------------------------- expectations
def step_corpus(case: dict):
    """Yield (op, the corpus as it stands when the op runs)."""
    cspec = case["corpus"]
    v0 = corpus(cspec)
    cur = v0[: case.get("load", len(v0))]
    for op in case["ops"]:
        if op["op"] == "remove":
            cur = np.delete(cur, op["ordinals"], axis=0)
        elif op["op"] == "append":
            cur = np.concatenate([cur, v0[op["rows"][0]: op["rows"][1]] if "rows" in op
                                  else queries(op["q"], cspec, v0)[: op["take"]]])
        yield op, cur, v0


def lookup_expectations(op, cur, cspec, v0) -> dict:
    qq = queries(op["q"], cspec, v0)
    a = lookup_args(len(cur), len(qq), op["seed"])
    dots = (qq.astype(np.float64) @ cur.astype(np.float64).T).astype(np.float32)
    k, ms = op["k"], op["ms"]
    kk = max(1, min(k, len(cur)))
    return {"allowed": oracle_arrays(dots, kk, ms, allowed=a["allowed"]),
            "masks": as_arrays(per_query(dots, ms, a["masks"]), kk),
            "subset": oracle_arrays(dots, max(1, min(k, len(a["subset"]))), ms, subset=a["subset"]),
            "subsets": oracle_batch_arrays(dots, k, ms, a["subsets"]),
            "ties_low": oracle_arrays(dots, kk, ms, ties_low=True),
            "range": oracle_csr(dots, ms),
            "range_masks": as_csr(per_query(dots, ms, a["masks"]))}


def same_bits(g, w):
    g, w = np.asarray(g), np.asarray(w)
    if g.dtype == np.float32:
        g, w = g.view(np.uint32), w.view(np.uint32)
    return g.shape == w.shape and bool((g == w).all())


def rebalance_mismatches(case: dict, world: int, out: str) -> list[str]:
    """Every way the ranks' rebalance outputs of ``case`` differ from the expectation."""
    from typeagent_py_b200.sharded import shard_bounds

    got = [np.load(os.path.join(out, f"{case['name']}.r{r}.npz")) for r in range(world)]
    errors = []
    for op, cur, v0 in step_corpus(case):
        key = op["key"]
        if op["op"] == "rebalance":
            sizes = op.get("sizes")
            raised = op.get("expect_raise", 0)
            want = shard_bounds(len(cur), world) if sizes is None else list(zip(np.cumsum([0] + sizes)[:-1],
                                                                               np.cumsum(sizes)))
            for r, g in enumerate(got):
                if int(g[key + ".raised"][0]) != raised:
                    errors.append(f"rank {r} {key}: raised {int(g[key + '.raised'][0])}, expected {raised}")
                    continue
                if not raised and [tuple(b) for b in g[key + ".blocks"].tolist()] != [tuple(map(int, b)) for b in want]:
                    errors.append(f"rank {r} {key}: blocks {g[key + '.blocks'].tolist()} != {want}")
                (index0, process0), (index1, process1) = g[key + ".row_bytes"].tolist()
                lo, hi = g[key + ".blocks"][r].tolist()
                row = D * (4 if case["storage"] == "float32" else 2)
                if not raised and index1 != max((hi - lo) * row, 256):
                    errors.append(f"rank {r} {key}: the index holds {index1} bytes of rows for {hi - lo} rows")
                if process1 - process0 != index1 - index0:
                    errors.append(f"rank {r} {key}: the process's row blocks changed by {process1 - process0} bytes, "
                                  f"its index's by {index1 - index0}: a replaced or staged block was not freed")
            if not raised and len({int(g[key + ".moved"][0]) for g in got}) != 1:
                errors.append(f"{key}: ranks returned different moved counts")
        elif op["op"] == "rows":
            for r, g in enumerate(got):
                lo, hi = g[key + ".range"].tolist()
                if not same_bits(g[key + ".mirror"], cur[lo:hi]):
                    errors.append(f"rank {r} {key}: serialize() differs from rows [{lo}, {hi})")
                if not op.get("normalized") and "normalize" not in case and not same_bits(g[key + ".device"],
                                                                                          cur[lo:hi]):
                    errors.append(f"rank {r} {key}: tav_read_rows differs from rows [{lo}, {hi})")
            if op.get("same_as"):
                a = np.concatenate([g[op["same_as"] + ".device"] for g in got])
                b = np.concatenate([g[key + ".device"] for g in got])
                if not same_bits(a, b):
                    errors.append(f"{key}: the device rows, in global order, changed since {op['same_as']}")
        elif op["op"] == "lookups":
            want = lookup_expectations(op, cur, case["corpus"], v0)
            for r, g in enumerate(got):
                for name, arrays in want.items():
                    if not all(same_bits(g[f"{key}.{name}.{i}"], w) for i, w in enumerate(arrays)):
                        errors.append(f"rank {r} {key}: {name} differs from the exact result")
        elif op["op"] == "maskprobe":
            for r, g in enumerate(got):
                if int(g[key + ".rc"][0]) != -5:  # TAV_ERR_STATE: no current row mask
                    errors.append(f"rank {r} {key}: a search with the row mask of the old rows returned "
                                  f"{int(g[key + '.rc'][0])}")
    return errors


def search_expectations(case: dict) -> dict:
    out = {}
    for op, cur, v0 in step_corpus(case):
        if op["op"] == "search":
            qq = queries(op["q"], case["corpus"], v0)
            k = max(1, min(op["k"], len(cur)))
            dots = (qq.astype(np.float64) @ cur.astype(np.float64).T).astype(np.float32)
            out[op["key"]] = expected_topk(dots, k, np.float32(op["ms"]))
    return out


def all_mismatches(case, world, out):
    return peer.mismatches(case, search_expectations(case), world, out) + rebalance_mismatches(case, world, out)


# ---------------------------------------------------------------- launching the ranks
def launch(world, cases, tmp, lib=None):
    saved, peer.WORKER = peer.WORKER, WORKER
    try:
        return peer.launch(world, cases, tmp, lib=lib)
    finally:
        peer.WORKER = saved


_RUNS: dict = {}


@pytest.fixture(scope="module", autouse=True)
def _remove_outputs():
    yield
    for kind, value in _RUNS.values():
        if kind == "ok":
            shutil.rmtree(os.path.dirname(value[1]), ignore_errors=True)
    _RUNS.clear()


def run_world(world: int):
    """The ranks of one world over all its cases, launched once per session: (cases, output directory)."""
    if world not in _RUNS:
        import torch

        cases = cases_for(world)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        tmp = tempfile.mkdtemp(prefix=f"tav_rebalance_w{world}_")
        try:
            _RUNS[world] = ("ok", (cases, launch(world, cases, tmp)))
        except pytest.skip.Exception as e:
            _RUNS[world] = ("skip", str(e))
            shutil.rmtree(tmp, ignore_errors=True)
            raise
        except (Exception, pytest.fail.Exception) as e:
            _RUNS[world] = ("fail", f"{type(e).__name__}: {e}")
            shutil.rmtree(tmp, ignore_errors=True)
            raise
    kind, value = _RUNS[world]
    if kind == "skip":
        pytest.skip(value)
    if kind == "fail":
        pytest.fail(f"the W={world} ranks failed earlier in this session and are not launched again:\n{value[:3000]}")
    return value


CASE_NAMES = ["bfloat16", "float16", "float32", "split_overflow", "split", "normalize", "oom"]


@pytest.mark.parametrize("name", CASE_NAMES + ["row_mask"])
@pytest.mark.parametrize("world", [2, 3])
def test_rebalance_equals_exact(world, name):
    cases, out = run_world(world)
    case = next((c for c in cases if c["name"] == name), None)
    if case is None:
        pytest.skip(f"the {name} case needs a rank whose block keeps its size: W = 3 only")
    errors = all_mismatches(case, world, out)
    assert not errors, "\n".join(errors[:20])


def test_rebalance_eight_ranks():
    cases, out = run_world(8)
    errors = all_mismatches(cases[0], 8, out)
    assert not errors, "\n".join(errors[:20])


# ---------------------------------------------------------------- broken builds
MUTANTS = {1: "two pieces laid out swapped", 2: "fp16 planes kept at commit", 3: "row mask kept at commit",
           4: "old rows not freed at commit"}


@pytest.fixture(scope="module")
def mutant_libs():
    """The broken libraries: tav_api.cu compiled once per variant, linked with the other translation units,
    which are compiled once."""
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc) and not shutil.which(nvcc):
        pytest.skip("nvcc is needed to build the broken variants")
    from typeagent_py_b200 import build as B

    flags = [f for f in B.NVCC_FLAGS if f not in ("-Xptxas=-v", "-shared", "-cudart", "static")]
    tmp = tempfile.mkdtemp(prefix="tav_rebalance_mutants_")
    jobs = {}
    for src in B.SOURCES:
        defines = [f"-DTAV_REBALANCE_MUTANT={m}" for m in MUTANTS] if src == "tav_api.cu" else [None]
        for d in defines:
            obj = os.path.join(tmp, src + (d.rsplit("=", 1)[1] if d else "") + ".o")
            cmd = [nvcc, *flags, *([d] if d else []), "-c", os.path.join(B.CSRC, src), "-o", obj]
            jobs[obj] = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    for obj, proc in jobs.items():
        log = proc.communicate()[0]
        assert proc.returncode == 0, log
    common = [os.path.join(tmp, s + ".o") for s in B.SOURCES if s != "tav_api.cu"]
    libs = {}
    for m in MUTANTS:
        lib = os.path.join(tmp, f"libtavec_rebalance_mutant{m}.so")
        proc = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-cudart", "static",
                               "-o", lib, os.path.join(tmp, f"tav_api.cu{m}.o"), *common], capture_output=True, text=True)
        assert proc.returncode == 0, proc.stdout + proc.stderr
        libs[m] = lib
    yield libs
    shutil.rmtree(tmp, ignore_errors=True)


@pytest.mark.parametrize("m", sorted(MUTANTS), ids=[MUTANTS[m].replace(" ", "_") for m in sorted(MUTANTS)])
def test_broken_build_is_caught(mutant_libs, m):
    failed = [w for w, (kind, _) in _RUNS.items() if kind == "fail"]
    if failed:
        pytest.skip(f"the real build failed at W={failed}: its broken variants are not launched")
    cases = [storage_case(3, "bfloat16"), split_case(3, big=False), mask_case()]
    tmp = tempfile.mkdtemp(prefix=f"tav_rebalance_mutant{m}_")
    try:
        out = launch(3, cases, tmp, lib=mutant_libs[m])
        caught = [e for c in cases for e in all_mismatches(c, 3, out)]
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    assert caught, f"the exact checks did not catch: {MUTANTS[m]}"
