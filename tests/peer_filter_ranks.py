"""One rank of a ``ShardedVectorBase(exchange="peer")`` group running filtered and subset lookups: the worker that
tests/test_gpu_peer_filtered.py launches W times on one GPU, as tests/peer_ranks.py does for plain lookups (same
spec, lockstep and shutdown; see there).

    python tests/peer_filter_ranks.py SPEC.json RANK

A search operation may carry ``filters``, rebuilt here and in the test by ``filters`` from seeds: ``allowed`` (one
row mask), ``masks`` (one mask per query), ``subset`` (one subset with duplicates and negative ordinals),
``subsets`` (per-query subsets, optionally all inside one block) and ``ties``.  ``pred`` runs
``fuzzy_lookup_embedding`` with a predicate.  ``fail`` makes one rank's lookup run out of memory and records what
every rank raised (code 0 nothing, 1 MemoryError, 2 RuntimeError): its per-query mask upload
(``tav_internal_qmask_cap``), or with ``alloc`` a cudaMalloc inside its local tensor-core search
(``tav_internal_search_alloc_fail``: a real allocation failure, not sticky).
"""

from __future__ import annotations

import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.peer_ranks import Rank, main as _main  # noqa: E402


def filters(spec: dict, n: int, b: int) -> dict:
    """The search_arrays keyword arguments of a filter spec over a corpus of n rows and b queries."""
    rng = np.random.default_rng(spec["seed"])
    out = {"ties_low_first": bool(spec.get("ties", False))}
    if spec.get("allowed"):
        out["allowed"] = rng.random(n) < 0.6
    if spec.get("masks"):
        out["allowed"] = rng.random((b, n)) < 0.5
    if spec.get("subset"):
        edges = [e for c in spec.get("edges", []) for e in range(c - 3, c + 3)]
        base = rng.permutation(n)[: n // 4]
        out["subset"] = np.concatenate([base, edges, edges, [-1, -n, 0, n - 1, -2]]).astype(np.int64)
    if spec.get("subsets"):
        lo, hi = spec.get("within", [0, n])
        out["subsets"] = [rng.integers(lo, hi, size=0 if i % 5 == 3 else 30 + 11 * i).astype(np.int64)
                          - (n if i % 4 == 1 else 0) for i in range(b)]
    return out


def predicate_of(spec: dict):
    m = int(spec["mod"])
    return lambda i: i % m != 1


def internal(name, argtypes):
    from typeagent_py_b200 import _capi

    fn = getattr(_capi.load(), name)
    fn.restype, fn.argtypes = C.c_int, argtypes
    return fn


def code_of(e) -> int:
    return 0 if e is None else 1 if isinstance(e, MemoryError) else 2


class FilterRank(Rank):
    _made: dict = {}

    def stage(self, op, cspec, v):
        if op["op"] in ("search", "raise", "fail", "pred"):
            from tests.peer_ranks import queries

            q = queries(op["q"], cspec, v)
            f = dict(op.get("filters", {"seed": 0}))
            # one object per mask or subset spec, so that a later lookup with it finds it uploaded (same key)
            ties = f.pop("ties", False)
            key = (repr(sorted(f.items())), len(v), len(q) if f.get("masks") or f.get("subsets") else -1)
            if key not in self._made:
                self._made[key] = filters(f, len(v), len(q))
            return q, dict(self._made[key], ties_low_first=bool(ties))
        return super().stage(op, cspec, v)

    def act(self, sh, op, staged, results, outputs, side) -> None:
        kind, key = op["op"], op["key"]
        if kind == "pred":
            q, _ = staged
            hits = sh.fuzzy_lookup_embedding(q[0], op["k"], op["ms"], predicate=predicate_of(op["pred"]))
            results[key + ".items"] = np.array([[h.item for h in hits]], np.int64)
            results[key + ".scores"] = np.array([[h.score for h in hits]], np.float32)
            results[key + ".counts"] = np.array([len(hits)], np.int32)
        elif kind == "search":
            q, f = staged
            outputs[key] = (q,) + tuple(sh.search_tensors(q, op["k"], op["ms"], defer_check=op.get("defer", False),
                                                          **f))
        elif kind == "raise":
            q, f = staged
            try:
                sh.search_tensors(q, op["k"], op["ms"], defer_check=True, **f)
                results[key + ".raised"] = np.array([0], np.int64)
            except RuntimeError as e:
                results[key + ".raised"] = np.array([1 if "outstanding" in str(e) else 2], np.int64)
        elif kind == "fail":
            self.fail(sh, op, staged, results)
        else:
            super().act(sh, op, staged, results, outputs, side)

    def fail(self, sh, op, staged, results) -> None:
        """One rank's per-query mask allocation fails.  ``agree``: through the upload agreement (every rank raises
        before anything is published); otherwise the agreement is bypassed, so the failing rank publishes its
        failure in the slot's status word and the others learn it from the merge (``defer``: at finish).  With
        ``alloc`` the failing allocation is one inside the local search itself (after the mask upload)."""
        from typeagent_py_b200 import _capi

        q, f = staged
        ix = sh._engine.base._ensure_device()[1]
        if op.get("alloc"):
            hook = internal("tav_internal_search_alloc_fail", [C.c_void_p, C.c_int])
            on, off = 1, 0
        else:
            hook = internal("tav_internal_qmask_cap", [C.c_void_p, C.c_int64])
            on, off = 0, -1
        if self.rank == op["cap_rank"]:
            _capi.check(hook(ix, on))
        agree = sh._agree_mask
        if not op.get("agree"):
            sh._agree_mask = lambda mask, n_queries: None
        search_error = finish_error = None
        try:
            sh.search_tensors(q, op["k"], op["ms"], defer_check=op.get("defer", False), **f)
        except Exception as e:  # noqa: BLE001
            search_error = e
        try:
            sh.finish()
        except Exception as e:  # noqa: BLE001
            finish_error = e
        sh._agree_mask = agree
        _capi.check(hook(ix, off))
        results[op["key"] + ".codes"] = np.array([code_of(search_error), code_of(finish_error)], np.int64)


if __name__ == "__main__":
    import tests.peer_ranks as P

    P.Rank = FilterRank
    sys.exit(_main(sys.argv[1:]))
