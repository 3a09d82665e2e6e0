"""One rank of a ``ShardedVectorBase`` group with ``exchange="peer"``: the worker that
tests/test_gpu_peer_exchange.py launches W times, every process on the same GPU (or ``rank % device_count``).

    python tests/peer_ranks.py SPEC.json RANK

CUDA IPC maps one process's device memory into another on the same device, so W processes sharing one GPU form
a real group: every rank's publish kernel stores into its peers' exchange regions and its merge kernel spins on
their flags, exactly as across NVLink.  The kernels of the W contexts run in turn (the default compute mode
time-slices contexts), so a spinning merge yields to its peer's publish.

The spec (JSON, written by the test) names the world, the gloo file store, the output directory, optionally
another build of libtavec, and a list of cases.  A case is a corpus (rebuilt here from seeds by ``corpus``) and
a list of operations on one ``ShardedVectorBase``.  The worker asserts nothing: it writes every output to
``<out>/<case>.r<rank>.npz`` and a status file, and the test compares them with the exact expectation.

The worker keeps the ranks in lockstep so that a failure cannot leave a kernel spinning on a rank that stopped:
  * preflight: context, an allocation and a tav_group connected over IPC, then a status word from every rank;
    if any rank failed (an exclusive-process device, no IPC) every rank stops and the test skips;
  * before every group search the ranks exchange a status word, which is also the barrier: inputs are staged
    before it, and nothing between the search and the next exchange depends on the rank;
  * after every case a status word again, and all ranks stop together if one failed;
  * shutdown with ``ShardedVectorBase.close()``: synchronise, barrier, destroy the index and its group, barrier.
"""

from __future__ import annotations

import json
import os
import sys
import traceback

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.exact import dyadic_corpus, preset  # noqa: E402

BIG = np.float32(2.0 ** 17)  # exact in float32, beyond the fp16 range (65504)


# ---------------------------------------------------------------- inputs (shared with the test)
def corpus(spec: dict) -> np.ndarray:
    """float32 [n, d] of a case: a dyadic corpus (tests/exact.py) with
    ``dup`` [[dst, src], ...] row copies, ``copies`` [src, lo, hi]: rows [lo, hi) copies of row src, and ``big``
    [[row, col], ...]: rows whose only non-zero entry is 2^17 in column col."""
    amp, exp = preset(spec["preset"], spec["d"])
    v, _, _ = dyadic_corpus(spec["n"], spec["d"], 1, amp, exp, seed=spec["seed"],
                            dup=[tuple(p) for p in spec.get("dup", [])])
    if spec.get("copies"):
        src, lo, hi = spec["copies"]
        v[lo:hi] = v[src]
    for row, col in spec.get("big", []):
        v[row] = 0
        v[row, col] = BIG
    return v


def queries(spec: dict, cspec: dict, v: np.ndarray) -> np.ndarray:
    """float32 [b, d] dyadic queries of the corpus's preset, drawn from ``seed``.  ``favour``: every other query
    is row ``favour`` itself; ``against``: queries whose dot with row ``against`` is positive are negated (that
    row then scores below 0.5); ``big_col``: column big_col of every query is +amp * 2^-exp, so that a 2^17 row
    in that column scores 1.0."""
    amp, exp = preset(cspec["preset"], cspec["d"])
    rng = np.random.default_rng(spec["seed"])
    q = rng.integers(-amp, amp + 1, size=(spec["b"], cspec["d"])).astype(np.float32) * np.float32(2.0 ** -exp)
    if spec.get("against") is not None:
        dots = q.astype(np.float64) @ v[spec["against"]].astype(np.float64)
        q[dots > 0] *= -1
    if spec.get("favour") is not None:
        q[::2] = v[spec["favour"]]
    if spec.get("big_col") is not None:
        q[:, spec["big_col"]] = np.float32(amp * 2.0 ** -exp)
    return np.ascontiguousarray(q)


# ---------------------------------------------------------------- the rank
class Rank:
    def __init__(self, spec: dict, rank: int):
        import torch
        import torch.distributed as dist

        self.torch, self.dist = torch, dist
        self.spec, self.rank, self.world = spec, rank, spec["world"]
        self.device = rank % max(torch.cuda.device_count(), 1)
        self.out = spec["out"]
        self.status: dict = {"rank": rank, "device": self.device, "cases": {}}

    def agree(self, ok: bool, what: str) -> bool:
        """Every rank's status word; True when all ranks are fine.  Also the barrier before a group search."""
        got = [None] * self.world
        self.dist.all_gather_object(got, (bool(ok), what))
        return all(g[0] for g in got)

    def write_status(self) -> None:
        with open(os.path.join(self.out, f"status.r{self.rank}.json"), "w") as f:
            json.dump(self.status, f)

    def preflight(self) -> bool:
        import ctypes as C

        from typeagent_py_b200 import _capi

        torch = self.torch
        err, handle, group = "", b"", None
        try:
            torch.cuda.set_device(self.device)
            x = torch.ones(1 << 20, device=f"cuda:{self.device}")
            torch.cuda.synchronize()
            del x
            lib = _capi.load()
            group = C.c_void_p()
            _capi.check(lib.tav_group_create(self.device, self.rank, self.world, 16, 16, 2, C.byref(group)))
            buf = C.create_string_buffer(lib.tav_group_handle_bytes())
            _capi.check(lib.tav_group_local_handle(group, buf))
            handle = bytes(buf.raw)
        except Exception as e:  # noqa: BLE001
            err = f"rank {self.rank}: {type(e).__name__}: {e}"
        got = [None] * self.world
        self.dist.all_gather_object(got, (err, handle))
        errors = [g[0] for g in got if g[0]]
        if not errors:
            try:
                _capi.check(lib.tav_group_connect(group, b"".join(g[1] for g in got)))
            except Exception as e:  # noqa: BLE001
                err = f"rank {self.rank}: {type(e).__name__}: {e}"
            got = [None] * self.world
            self.dist.all_gather_object(got, err)
            errors = [g for g in got if g]
        self.dist.barrier()
        if group is not None and group.value:
            _capi.load().tav_group_destroy(group)
        self.dist.barrier()
        self.status["preflight"] = "; ".join(errors)
        return not errors

    def warm_up(self) -> None:
        """One plain local search per storage type, so that module loading does not happen while a peer spins."""
        import typeagent_py_b200 as tab
        from oracle import vectorbase_oracle as O

        for storage in ("float32", "bfloat16", "float16"):
            one = tab.VectorBase(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()), device=self.device,
                                 storage_dtype=storage)
            one.add_embeddings(None, np.ones((4096, 64), np.float32))
            one.search_arrays(np.ones((16, 64), np.float32), 10, 0.0)
            one.search_arrays(np.ones((1, 64), np.float32), 10, 0.0)
            del one
        self.torch.cuda.synchronize()

    def stage(self, op: dict, cspec: dict, v: np.ndarray):
        """What an operation needs before the ranks agree to run it: its queries on the device."""
        if op["op"] in ("search", "raise"):
            q = self.torch.from_numpy(queries(op["q"], cspec, v)).to(f"cuda:{self.device}")
            self.torch.cuda.synchronize()
            return q
        if op["op"] == "append":
            return queries(op["q"], cspec, v)[: op["take"]]
        return None

    def act(self, sh, op: dict, staged, results: dict, outputs: dict, side) -> None:
        torch = self.torch
        kind, key = op["op"], op["key"]
        if kind == "remove":
            sh.remove_embeddings(np.asarray(op["ordinals"], np.int64))
        elif kind == "append":
            sh.add_embeddings(None, staged)
        elif kind == "finish":
            results[key + ".finish"] = np.array([sh.finish()], np.int64)
        else:
            stream = side if op.get("stream") else torch.cuda.current_stream(self.device)
            with torch.cuda.stream(stream):
                if kind == "raise":  # a search the group must refuse, the same way on every rank
                    try:
                        sh.search_tensors(staged, op["k"], op["ms"], defer_check=True)
                        results[key + ".raised"] = np.array([0], np.int64)
                    except RuntimeError as e:
                        results[key + ".raised"] = np.array([1 if "outstanding" in str(e) else 2], np.int64)
                else:
                    outputs[key] = (staged,) + tuple(sh.search_tensors(staged, op["k"], op["ms"],
                                                                       defer_check=op.get("defer", False)))

    def run_case(self, case: dict) -> bool:
        """The case's operations in lockstep; its outputs to ``<out>/<case>.r<rank>.npz``.  False when some rank
        failed (all ranks return False together)."""
        import typeagent_py_b200 as tab
        from oracle import vectorbase_oracle as O
        from typeagent_py_b200.sharded import ShardedVectorBase

        torch = self.torch
        cspec = case["corpus"]
        results, outputs, error = {}, {}, ""
        sh, used = None, 0
        try:
            v = corpus(cspec)
            sh = ShardedVectorBase(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()), device=self.device,
                                   storage_dtype=case["storage"], exchange="peer")
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
            if not self.agree(not error, op["key"]):  # the barrier before the operation
                error = error or "another rank failed"
                break
            try:
                self.act(sh, op, staged, results, outputs, side)
                # device memory in use after every operation (all ranks' contexts): its allocations are made by
                # the host calls, so this sees each one that outlives the operation
                free, total = torch.cuda.mem_get_info(self.device)
                used = max(used, total - free)
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
                results["device_used_bytes"] = np.array([used], np.int64)
        except Exception:  # noqa: BLE001
            error = error or traceback.format_exc()
        outputs.clear()
        # collective, in a fixed order: nobody frees a region that a peer may still publish into
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
    r = Rank(spec, rank)
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
