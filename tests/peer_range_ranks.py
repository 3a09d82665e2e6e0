"""One rank of a ``ShardedVectorBase(exchange="peer")`` group running threshold searches through the range inbox:
the worker that tests/test_gpu_peer_range.py launches W times on one GPU, as tests/peer_ranks.py does for plain
lookups (same spec, lockstep and shutdown; see there).

    python tests/peer_range_ranks.py SPEC.json RANK

Operations, besides those of tests/peer_ranks.py (deferred top-k ``search`` and ``finish``):
  * ``range``: ``search_range`` with the operation's ``filters`` (rebuilt here and in the test by
    tests/peer_filter_ranks.py ``filters``); records offsets, items and scores, the rounds the search took and the
    range inbox's capacity and bytes afterwards (``tav_internal_range_bytes``: this group's and the process's);
  * ``fuzzy0``: ``fuzzy_lookup_embedding(max_hits=0)`` of the first query;
  * ``arrays``: ``search_arrays`` with ``k`` and the filters (the threshold routes: k >= rows > 8192, per-query
    subsets with k > 2048);
  * ``rfail``: one rank's per-query mask upload fails (``tav_internal_qmask_cap``) with the upload agreement
    bypassed, so that its local search fails and publishes status 1;
  * ``gfail``: one rank's range inbox may not grow (``tav_internal_range_cap``) and the search needs a grow;
  * ``ofail``: one rank cannot allocate the merged result's device buffers (after the rounds); the other ranks
    record their results.
The failures record what the rank raised (code 0 nothing, 1 MemoryError, 2 RuntimeError).  A case may set
``retain``: the engine's ``RANGE_RETAIN_BYTES``.
"""

from __future__ import annotations

import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.peer_filter_ranks import code_of, filters, internal  # noqa: E402
from tests.peer_ranks import Rank, main as _main  # noqa: E402

RANGE_OPS = ("range", "fuzzy0", "arrays", "rfail", "gfail", "ofail")


class NoEmpty:
    """torch as the engine sees it, except that ``empty`` (the output buffers of a search) fails."""

    def __init__(self, torch):
        self._torch = torch

    def __getattr__(self, name):
        return getattr(self._torch, name)

    def empty(self, *a, **kw):
        raise MemoryError("the output buffers could not be allocated")


def inbox_bytes(sh) -> tuple[int, int]:
    """(this group's range inbox bytes, range inbox bytes of the process)."""
    group, process = C.c_int64(0), C.c_int64(0)
    if sh._engine._group is not None:
        fn = internal("tav_internal_range_bytes", [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)])
        fn(sh._engine._group, C.byref(group), C.byref(process))
    return group.value, process.value


class RangeRank(Rank):
    _made: dict = {}

    def run_case(self, case: dict) -> bool:
        self._retain = case.get("retain")
        return super().run_case(case)

    def stage(self, op, cspec, v):
        if op["op"] in RANGE_OPS:
            from tests.peer_ranks import queries

            q = queries(op["q"], cspec, v)
            f = dict(op.get("filters", {"seed": 0}))
            ties = f.pop("ties", False)
            rows = op.get("rows", len(v))  # the rows the filters cover (after a removal: those left)
            key = (repr(sorted(f.items())), rows, len(q) if f.get("masks") or f.get("subsets") else -1)
            if key not in self._made:  # one object per mask spec, so that a later lookup finds it uploaded
                self._made[key] = filters(f, rows, len(q))
            return q, dict(self._made[key], ties_low_first=bool(ties))
        return super().stage(op, cspec, v)

    def act(self, sh, op, staged, results, outputs, side) -> None:
        kind, key = op["op"], op["key"]
        if self._retain is not None:
            sh._engine.RANGE_RETAIN_BYTES = int(self._retain)
        if kind == "range":
            q, f = staged
            o, i, s = sh.search_range(q, op["ms"], **f)
            results[key + ".offsets"], results[key + ".items"], results[key + ".scores"] = o, i, s
            results[key + ".rounds"] = np.array([sh._engine.last_range_rounds], np.int64)
            results[key + ".inbox"] = np.array([sh._engine.range_capacity()[1], *inbox_bytes(sh)], np.int64)
        elif kind == "fuzzy0":
            q, _ = staged
            hits = sh.fuzzy_lookup_embedding(q[0], 0, op["ms"])
            results[key + ".offsets"] = np.array([0, len(hits)], np.int64)
            results[key + ".items"] = np.array([h.item for h in hits], np.int64)
            results[key + ".scores"] = np.array([h.score for h in hits], np.float32)
        elif kind == "arrays":
            q, f = staged
            results[key + ".items"], results[key + ".scores"], results[key + ".counts"] = sh.search_arrays(
                q, op["k"], op["ms"], **f)
        elif kind in ("rfail", "gfail", "ofail"):
            self.fail(sh, op, staged, results)
        else:
            super().act(sh, op, staged, results, outputs, side)

    def fail(self, sh, op, staged, results) -> None:
        from typeagent_py_b200 import _capi

        q, f = staged
        capped = self.rank == op["cap_rank"]
        if op["op"] == "ofail":
            eng = sh._engine
            torch, error = eng.torch, None
            if capped:
                eng.torch = NoEmpty(torch)
            try:
                got = sh.search_range(q, op["ms"], **f)
                for name, a in zip(("offsets", "items", "scores"), got):
                    results[f"{op['key']}.{name}"] = a
            except Exception as e:  # noqa: BLE001
                error = e
            eng.torch = torch
            results[op["key"] + ".codes"] = np.array([code_of(error)], np.int64)
            return
        if op["op"] == "rfail":
            hook, target, on, off = internal("tav_internal_qmask_cap", [C.c_void_p, C.c_int64]), \
                sh._engine.base._ensure_device()[1], 0, -1
        else:
            hook, target, on, off = internal("tav_internal_range_cap", [C.c_void_p, C.c_int64]), \
                sh._engine._group, inbox_bytes(sh)[0], -1
        if capped:
            _capi.check(hook(target, on))
        agree = sh._agree_mask
        sh._agree_mask = lambda mask, n_queries: None
        error = None
        try:
            sh.search_range(q, op["ms"], **f)
        except Exception as e:  # noqa: BLE001
            error = e
        sh._agree_mask = agree
        if capped:
            _capi.check(hook(target, off))
        results[op["key"] + ".codes"] = np.array([code_of(error)], np.int64)
        results[op["key"] + ".inbox"] = np.array([sh._engine.range_capacity()[1], *inbox_bytes(sh)], np.int64)


if __name__ == "__main__":
    import tests.peer_ranks as P

    P.Rank = RangeRank
    sys.exit(_main(sys.argv[1:]))
