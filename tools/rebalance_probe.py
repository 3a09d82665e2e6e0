"""Time ``ShardedVectorBase.rebalance`` on one GPU shared by W rank processes, against the status quo.

    python tools/rebalance_probe.py [--world 2] [--rows 10000000] [--dim 768] [--load 2000000] [--out FILE]

Every rank builds a skewed bf16 index: ``--load`` rows spread evenly by ``load_local_shard``, then the rest appended,
so that they all sit on the last rank, and the device rows brought up to date.  Then one ``rebalance()``, its phases
timed on every rank (host clock; every phase ends synchronised):
  * export: ``rows_export`` (the IPC handle of the rank's rows);
  * stage: ``rows_stage`` (allocate the new block, copy the pieces from the ranks' rows, synchronise);
  * mirror: the float32 host mirrors of the moved rows over the process group (``all_to_all_single``, gloo here);
  * commit: ``rows_commit`` (swap in the new rows, free the old ones, replace the mirror);
  * total: the whole call, collectives included.
Moved bytes are the rows that changed rank, in the storage dtype, over the slowest rank's stage.  Peak memory: the
bytes of every rank's row blocks right after its stage (old and new block both held; ``tav_internal_row_bytes``), and
the device memory in use then (all ranks' contexts, and whatever else runs on the device).

The status quo in the same session, after the rebalanced index is closed: ``deserialize`` of the global float32
array on every rank of a fresh index, then its rows brought to the device.  The global array is held in host
memory, so each rank's part of it is a view, as ``deserialize`` slices it; only that part is materialised.  Times
are the slowest rank's.  One run of each; the card's name and power limit are printed with the numbers.  The ranks
share one GPU, so the peer copies are device-to-device copies; copies between GPUs over NVLink are not measured.
"""

from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

CHUNK = 1 << 20  # rows generated per seed


def rows_of(lo: int, hi: int, dim: int) -> np.ndarray:
    """Global rows [lo, hi) as float32, exact in bf16: chunk c of CHUNK rows from seed c."""
    out = np.empty((hi - lo, dim), np.float32)
    for c in range(lo // CHUNK, -(-hi // CHUNK)):
        a, b = max(lo, c * CHUNK), min(hi, (c + 1) * CHUNK)
        gen = np.random.default_rng(1000 + c).integers(-127, 128, size=(CHUNK, dim), dtype=np.int8)
        out[a - lo: b - lo] = gen[a - c * CHUNK: b - c * CHUNK].astype(np.float32) * np.float32(1 / 128)
    return out


class GlobalRows:
    """The global array as ``deserialize`` reads it, for one rank: its shape, and this rank's block as a view."""

    def __init__(self, n: int, dim: int, lo: int, hi: int):
        self.shape, self.ndim = (n, dim), 2
        self._lo, self._block = lo, rows_of(lo, hi, dim)

    def __len__(self):
        return self.shape[0]

    def __getitem__(self, sl):
        return self._block[sl.start - self._lo: sl.stop - self._lo]


def rank_main(args) -> None:
    import torch
    import torch.distributed as dist

    import typeagent_py_b200 as tab
    from oracle import vectorbase_oracle as O
    from typeagent_py_b200 import _capi
    from typeagent_py_b200.sharded import ShardedVectorBase, shard_bounds

    rank, world, n, d = args.rank, args.world, args.rows, args.dim
    dist.init_process_group("gloo", init_method=f"file://{args.store}", rank=rank, world_size=world)
    torch.cuda.set_device(0)
    lib = _capi.load()
    row_bytes = lib.tav_internal_row_bytes
    row_bytes.restype, row_bytes.argtypes = C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]
    settings = tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel())

    def used() -> int:
        free, total = torch.cuda.mem_get_info(0)
        return total - free

    # ---- the skewed index
    sh = ShardedVectorBase(settings, device=0, storage_dtype="bfloat16")
    lo, hi = shard_bounds(args.load, world)[rank]
    sh.load_local_shard(rows_of(lo, hi, d), args.load)
    zeros = np.zeros(d, np.float32)
    for a in range(args.load, n, 4 * CHUNK):
        b = min(n, a + 4 * CHUNK)
        sh.add_embeddings(None, rows_of(a, b, d) if rank == world - 1 else np.broadcast_to(zeros, (b - a, d)))
    eng = sh._engine
    eng.base._ensure_device()
    torch.cuda.synchronize()
    dist.barrier()

    times, peak = {}, {}

    def timed(name, fn, after=None):
        def run(*a, **k):
            t0 = time.perf_counter()
            out = fn(*a, **k)
            torch.cuda.synchronize()
            times[name] = times.get(name, 0.0) + time.perf_counter() - t0
            if after:
                after()
            return out
        return run

    def after_stage():
        index, process = C.c_int64(0), C.c_int64(0)
        _capi.check(row_bytes(eng.base._ix, C.byref(index), C.byref(process)))
        peak.update(row_bytes=index.value, device_used=used())

    eng.rows_export = timed("export", eng.rows_export)
    eng.rows_stage = timed("stage", eng.rows_stage, after_stage)
    sh._exchange_mirror = timed("mirror", sh._exchange_mirror)
    eng.rows_commit = timed("commit", eng.rows_commit)
    blocks_before = sh.blocks
    t0 = time.perf_counter()
    moved = sh.rebalance()
    times["total"] = time.perf_counter() - t0
    mine = {"rank": rank, "times": times, "peak": peak, "moved": moved, "blocks_before": blocks_before,
            "blocks_after": sh.blocks}
    sh.close()
    del sh, eng
    torch.cuda.synchronize()
    torch.cuda.empty_cache()

    # ---- the status quo: deserialize of the global array on a fresh index, rows to the device
    lo, hi = shard_bounds(n, world)[rank]
    data = GlobalRows(n, d, lo, hi)
    fresh = ShardedVectorBase(settings, device=0, storage_dtype="bfloat16")
    dist.barrier()
    t0 = time.perf_counter()
    fresh.deserialize(data)
    fresh._engine.base._ensure_device()
    torch.cuda.synchronize()
    mine["deserialize_s"] = time.perf_counter() - t0
    fresh.close()
    got = [None] * world
    dist.all_gather_object(got, mine)
    if rank == 0:
        slowest = {k: max(g["times"].get(k, 0.0) for g in got) for k in ("export", "stage", "mirror", "commit", "total")}
        moved_bytes = got[0]["moved"] * d * 2
        report = {
            "gpu": args.gpu, "world": world, "rows": n, "dim": d, "storage": "bfloat16",
            "blocks_before": got[0]["blocks_before"], "blocks_after": got[0]["blocks_after"],
            "rows_moved": got[0]["moved"], "bytes_moved": moved_bytes,
            "rebalance_s": slowest, "moved_GB_per_s_over_stage": moved_bytes / slowest["stage"] / 1e9,
            "row_blocks_after_stage_bytes": [g["peak"].get("row_bytes", 0) for g in got],
            "device_used_after_stage_bytes": max(g["peak"].get("device_used", 0) for g in got),
            "deserialize_s": max(g["deserialize_s"] for g in got),
        }
        text = json.dumps(report)
        print(text)
        if args.out:
            with open(args.out, "w") as f:
                f.write(text + "\n")
    dist.barrier()
    dist.destroy_process_group()


def main() -> int:
    p = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    p.add_argument("--world", type=int, default=2)
    p.add_argument("--rows", type=int, default=10_000_000)
    p.add_argument("--dim", type=int, default=768)
    p.add_argument("--load", type=int, default=2_000_000, help="rows spread evenly before the appends")
    p.add_argument("--out", default=None)
    p.add_argument("--rank", type=int, default=None, help=argparse.SUPPRESS)
    p.add_argument("--store", default=None, help=argparse.SUPPRESS)
    p.add_argument("--gpu", default=None, help=argparse.SUPPRESS)
    args = p.parse_args()
    if args.rank is not None:
        rank_main(args)
        return 0
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip().splitlines()
    except FileNotFoundError:
        gpu = []
    if not gpu:
        raise SystemExit("no GPU: this probe measures on an H100")
    tmp = tempfile.mkdtemp(prefix="tav_rebalance_probe_")
    cmd = [sys.executable, os.path.abspath(__file__), "--world", str(args.world), "--rows", str(args.rows), "--dim",
           str(args.dim), "--load", str(args.load), "--store", os.path.join(tmp, "store"), "--gpu", gpu[0]]
    if args.out:
        cmd += ["--out", os.path.abspath(args.out)]
    procs = [subprocess.Popen(cmd + ["--rank", str(r)], cwd=ROOT) for r in range(args.world)]
    try:
        codes = [p.wait() for p in procs]
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
                p.wait()
        shutil.rmtree(tmp, ignore_errors=True)
    return max(codes)


if __name__ == "__main__":
    sys.exit(main())
