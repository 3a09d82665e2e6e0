#!/usr/bin/env python3
"""Filtered and subset lookups of ``ShardedVectorBase`` through the peer exchange against the process-group
exchange (``_exchange_topk``: packed all-gather + ``tav_merge_topk_ordered``), W rank processes on ONE GPU.

    python tools/peer_filter_probe.py [--world 2] [--rows 1000000] [--dim 256] [--batch 16] [--k 10] [--reps 30]

Both groups run over gloo with the ranks sharing cuda:0 (the peer exchange's CUDA IPC works between processes on
one device; NCCL does not run two ranks on one GPU), so the process-group exchange here is gloo's, through host
memory, and the peer exchange's publish and merge run between contexts that share the GPU.  What this measures is
the protocol's overhead on one GPU (host checks, mask agreement, launches, the waits), not NVLink: on 2 or more
GPUs the exchange is not measured by this script.

Per lookup kind (row mask, per-query masks, ties low-first, one subset, per-query subsets), rank 0 prints one JSON
line with the median host wall time of a synchronous ``search_arrays`` for each exchange, the median device span
(CUDA events on the current stream around the call) and, for the peer exchange, the wall time per lookup of 8
deferred ``search_tensors`` calls and one ``finish()``.  The card's name and power limit are in every line.
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card() -> dict:
    import torch

    out = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        out["power_limit"] = q.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out["power_limit"] = "unknown"
    return out


def kinds(n: int, b: int, rng) -> dict:
    """Lookup kind -> search_arrays keyword arguments (one object each, so that masks are uploaded once)."""
    return {
        "row_mask": dict(allowed=rng.random(n) < 0.5),
        "query_masks": dict(allowed=rng.random((b, n)) < 0.5),
        "ties_low_first": dict(ties_low_first=True),
        "subset": dict(subset=rng.permutation(n)[: n // 8].astype(np.int64)),
        "subsets": dict(subsets=[rng.permutation(n)[:2000].astype(np.int64) for _ in range(b)]),
    }


def rank_main(rank: int, args, store: str) -> None:
    import torch
    import torch.distributed as dist

    import typeagent_py_b200 as tab
    from oracle import vectorbase_oracle as O
    from typeagent_py_b200.sharded import ShardedVectorBase

    torch.cuda.set_device(0)
    dist.init_process_group("gloo", init_method=f"file://{store}", rank=rank, world_size=args.world)
    rng = np.random.default_rng(7)
    v = rng.standard_normal((args.rows, args.dim)).astype(np.float32)
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    q = np.ascontiguousarray(v[rng.integers(0, args.rows, args.batch)])
    settings = tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel())
    info = card() if rank == 0 else {}
    lookups = kinds(args.rows, args.batch, rng)
    groups = {}
    for exchange in ("peer", "nccl"):
        sh = ShardedVectorBase(settings, device=0, storage_dtype="bfloat16", exchange=exchange)
        sh.deserialize(v)
        groups[exchange] = sh
    for name, kw in lookups.items():
        row = dict(kind=name, world=args.world, rows=args.rows, dim=args.dim, batch=args.batch, k=args.k,
                   storage="bfloat16", **info)
        for exchange, sh in groups.items():
            try:
                wall, span = [], []
                for i in range(args.reps + 5):
                    dist.barrier()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    t0 = time.perf_counter()
                    e0.record()
                    sh.search_arrays(q, args.k, 0.0, **kw)
                    e1.record()
                    e1.synchronize()
                    if i >= 5:
                        wall.append((time.perf_counter() - t0) * 1e3)
                        span.append(e0.elapsed_time(e1))
                row[f"{exchange}_wall_ms"] = float(np.median(wall))
                row[f"{exchange}_device_span_ms"] = float(np.median(span))
            except Exception as e:  # noqa: BLE001  (recorded, not hidden: the line says which exchange failed)
                row[f"{exchange}_error"] = f"{type(e).__name__}: {e}"[:200]
        sh = groups["peer"]
        qd = torch.from_numpy(q).cuda()
        deferred = []
        for i in range(max(1, args.reps // 8) + 1):
            dist.barrier()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(8):
                sh.search_tensors(qd, args.k, 0.0, defer_check=True, **kw)
            sh.finish()
            torch.cuda.synchronize()
            if i:
                deferred.append((time.perf_counter() - t0) * 1e3 / 8)
        row["peer_deferred_wall_ms_per_lookup"] = float(np.median(deferred))
        if rank == 0:
            print(json.dumps(row), flush=True)
    for sh in groups.values():
        sh.close()
    dist.barrier()
    dist.destroy_process_group()


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=2)
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=256)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    import torch
    import torch.multiprocessing as mp

    if not torch.cuda.is_available():
        print("peer_filter_probe: no CUDA device", file=sys.stderr)
        return 1
    with tempfile.TemporaryDirectory() as tmp:
        os.environ.setdefault("GLOO_SOCKET_IFNAME", "lo")
        mp.spawn(rank_main, args=(args, os.path.join(tmp, "store")), nprocs=args.world, join=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
