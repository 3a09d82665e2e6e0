"""One rank of a ``ShardedVectorBase`` group that rebalances: the worker tests/test_gpu_rebalance.py launches W times,
every process on the same GPU (or ``rank % device_count``).

    python tests/rebalance_ranks.py SPEC.json RANK

It is tests/peer_ranks.py's worker (preflight, warm-up, lockstep status words before every operation and after
every case, ``close()`` at the end of a case) with the operations of a rebalance added:
  * ``rebalance``: ``rebalance(sizes)``, its return value, and the bytes of the rank's row allocations and of
    every row block the process holds (``tav_internal_row_bytes``) before and after it; with ``cap_rank`` that
    rank's stage is capped at 0 bytes (``tav_internal_stage_cap``), the call must raise, and what it raised is
    recorded;
  * ``lookups``: the filtered, per-query-mask, subset and threshold lookups of ``lookup_args``;
  * ``rows``: the rank's block, its host mirror (``serialize()``) and its device rows (``tav_read_rows``);
  * ``search`` with ``force``: the search path forced for that search only (``VectorBase.force_path``);
  * ``mask`` / ``maskprobe``: an all-ones row mask set on the rank's index, then a ``tav_search`` with
    ``TAV_USE_ROW_MASK`` and no new mask, whose return code is recorded (the rows changed: it must be refused).
The worker asserts nothing: the test compares every output with the exact expectation.
"""

from __future__ import annotations

import ctypes as C
import json
import os
import sys
import traceback

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.peer_ranks import Rank, corpus, queries  # noqa: E402


def lookup_args(n: int, b: int, seed: int) -> dict:
    """The row mask, per-query masks, subset and per-query subsets of a ``lookups`` operation over n rows."""
    rng = np.random.default_rng(seed)
    return dict(allowed=rng.random(n) < 0.5, masks=rng.random((b, n)) < 0.6,
                subset=np.concatenate([rng.permutation(n)[: n // 3], [0, n - 1, -1, 0]]).astype(np.int64),
                subsets=[rng.permutation(n)[: 40 + 7 * i] for i in range(b)])


def internal(name, argtypes):
    from typeagent_py_b200 import _capi

    fn = getattr(_capi.load(), name)
    fn.restype, fn.argtypes = C.c_int, argtypes
    return fn


class RebalanceRank(Rank):
    def act_rebalance(self, sh, op, staged, results):
        from typeagent_py_b200 import _capi

        kind, key = op["op"], op["key"]
        if kind == "rebalance":
            cap = op.get("cap_rank")
            ix = sh._engine.base._ensure_device()[1]
            if cap is not None and cap == self.rank:
                _capi.check(internal("tav_internal_stage_cap", [C.c_void_p, C.c_int64])(ix, 0))
            row_bytes = internal("tav_internal_row_bytes", [C.c_void_p, C.c_void_p, C.c_void_p])

            def held():
                index, process = C.c_int64(0), C.c_int64(0)
                _capi.check(row_bytes(ix, C.byref(index), C.byref(process)))
                return [index.value, process.value]

            before = held()
            try:
                results[key + ".moved"] = np.array([sh.rebalance(op.get("sizes"))], np.int64)
                results[key + ".raised"] = np.array([0], np.int64)
            except MemoryError:
                results[key + ".raised"] = np.array([1], np.int64)
            except RuntimeError:
                results[key + ".raised"] = np.array([2], np.int64)
            finally:
                if cap is not None and cap == self.rank:
                    _capi.check(internal("tav_internal_stage_cap", [C.c_void_p, C.c_int64])(ix, -1))
            results[key + ".row_bytes"] = np.array([before, held()], np.int64)
            results[key + ".blocks"] = np.array(sh.blocks, np.int64).reshape(-1, 2)
        elif kind == "lookups":
            n = len(sh)
            a = lookup_args(n, len(staged), op["seed"])
            k, ms = op["k"], op["ms"]
            out = {
                "allowed": sh.search_arrays(staged, k, ms, allowed=a["allowed"]),
                "masks": sh.search_arrays(staged, k, ms, allowed=a["masks"]),
                "subset": sh.search_arrays(staged, k, ms, subset=a["subset"]),
                "subsets": sh.search_arrays(staged, k, ms, subsets=a["subsets"]),
                "ties_low": sh.search_arrays(staged, k, ms, ties_low_first=True),
                "range": sh.search_range(staged, ms),
                "range_masks": sh.search_range(staged, ms, allowed=a["masks"]),
            }
            for name, arrays in out.items():
                for i, arr in enumerate(arrays):
                    results[f"{key}.{name}.{i}"] = np.asarray(arr)
        elif kind == "rows":
            lo, hi = sh.local_range
            base = sh._engine.base
            results[key + ".range"] = np.array([lo, hi], np.int64)
            results[key + ".mirror"] = np.array(base.serialize(), np.float32).reshape(hi - lo, sh._embedding_size)
            lib, ix = base._ensure_device()
            dev = np.zeros((hi - lo, max(sh._embedding_size, 1)), np.float32)
            if hi > lo:
                _capi.check(lib.tav_read_rows(ix, 0, hi - lo, dev.ctypes.data_as(C.POINTER(C.c_float)), None))
            results[key + ".device"] = dev
        elif kind == "mask":
            lib, ix = sh._engine.base._ensure_device()
            n = len(sh._engine.base)
            words = np.full((n + 31) // 32, 0xFFFFFFFF, np.uint32)
            _capi.check(lib.tav_set_row_mask(ix, words.ctypes.data_as(C.c_void_p), n, 0, None))
        elif kind == "maskprobe":
            lib, ix = sh._engine.base._ensure_device()
            q = np.ascontiguousarray(staged[:1].cpu().numpy())
            items, scores, counts = np.zeros(4, np.int64), np.zeros(4, np.float32), np.zeros(1, np.int32)
            rc = lib.tav_search(ix, q.ctypes.data_as(C.c_void_p), 1, 4, C.c_float(0.0),
                                _capi.TAV_USE_ROW_MASK | _capi.TAV_FORCE_SCAN, None, 0, 0,
                                items.ctypes.data_as(C.c_void_p), scores.ctypes.data_as(C.c_void_p),
                                counts.ctypes.data_as(C.c_void_p), None)
            results[key + ".rc"] = np.array([rc], np.int64)

    def stage(self, op, cspec, v):
        if op["op"] == "append" and "rows" in op:
            return v[op["rows"][0]: op["rows"][1]]
        if op["op"] in ("lookups",):
            return queries(op["q"], cspec, v)
        if op["op"] == "maskprobe":
            return super().stage(dict(op, op="search"), cspec, v)
        return super().stage(op, cspec, v)

    def act(self, sh, op, staged, results, outputs, side):
        if op["op"] in ("rebalance", "lookups", "rows", "mask", "maskprobe"):
            return self.act_rebalance(sh, op, staged, results)
        sh._engine.base.force_path = op.get("force")  # a search may force the tensor cores
        try:
            return super().act(sh, op, staged, results, outputs, side)
        finally:
            sh._engine.base.force_path = None

    def run_case(self, case: dict) -> bool:
        """peer_ranks' case loop; the index may be a TAV_NORMALIZE one."""
        import typeagent_py_b200 as tab
        from oracle import vectorbase_oracle as O
        from typeagent_py_b200.sharded import ShardedVectorBase

        torch = self.torch
        cspec = case["corpus"]
        results, outputs, error = {}, {}, ""
        sh = None
        try:
            v = corpus(cspec)
            settings = tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel())
            sh = ShardedVectorBase(settings, device=self.device, storage_dtype=case["storage"], exchange="peer")
            if case.get("normalize"):
                sh._engine.base = tab.VectorBase(settings, device=self.device, storage_dtype=case["storage"],
                                                 normalize=True)
            sh.deserialize(v[: case.get("load", len(v))])
            side = torch.cuda.Stream(device=self.device)
        except Exception:  # noqa: BLE001
            error = traceback.format_exc()
        for op in case["ops"]:
            staged = None
            if not error:
                try:
                    staged = self.stage(op, cspec, v)
                except Exception:  # noqa: BLE001
                    error = traceback.format_exc()
            if not self.agree(not error, op["key"]):
                error = error or "another rank failed"
                break
            try:
                self.act(sh, op, staged, results, outputs, side)
            except Exception:  # noqa: BLE001
                error = traceback.format_exc()
        if self.agree(not error, "finish") and sh is not None and sh._pending:
            try:
                sh.finish()
            except Exception:  # noqa: BLE001
                error = traceback.format_exc()
        try:
            torch.cuda.synchronize()
            if not error:
                for key, (_, items, scores, counts) in outputs.items():
                    results[key + ".items"] = items.cpu().numpy()
                    results[key + ".scores"] = scores.cpu().numpy()
                    results[key + ".counts"] = counts.cpu().numpy()
        except Exception:  # noqa: BLE001
            error = error or traceback.format_exc()
        outputs.clear()
        if sh is not None:
            try:
                sh.close()
            except Exception:  # noqa: BLE001
                error = error or traceback.format_exc()
        else:
            self.dist.barrier()
            self.dist.barrier()
        del sh
        np.savez(os.path.join(self.out, f"{case['name']}.r{self.rank}.npz"), **results)
        self.status["cases"][case["name"]] = error or "ok"
        return self.agree(not error, case["name"])


def main(argv) -> int:
    from datetime import timedelta

    with open(argv[0]) as f:
        spec = json.load(f)
    rank = int(argv[1])
    if spec.get("lib"):
        from typeagent_py_b200 import _capi

        _capi.LIB_PATH = spec["lib"]
    import torch.distributed as dist

    dist.init_process_group("gloo", init_method=f"file://{spec['store']}", rank=rank, world_size=spec["world"],
                            timeout=timedelta(seconds=spec.get("timeout", 300)))
    r = RebalanceRank(spec, rank)
    try:
        if not r.preflight():
            return 0
        r.warm_up()
        for case in spec["cases"]:
            if not r.run_case(case):
                break
    finally:
        r.write_status()
        dist.barrier()
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
