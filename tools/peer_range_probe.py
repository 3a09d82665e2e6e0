#!/usr/bin/env python3
"""Threshold searches of ``ShardedVectorBase`` through the peer exchange (the group's range inbox) against the
process-group exchange (offsets and hits all-gathered, then ``tav_merge_range``), W rank processes on ONE GPU.

    python tools/peer_range_probe.py [--world 2] [--reps 10]

Both groups run over gloo with the ranks sharing cuda:0 (CUDA IPC works between processes on one device; NCCL does
not run two ranks on one GPU), so the process-group exchange here is gloo's, through host memory, and the peer
exchange's publish, wait and merge run between contexts that share the GPU.  What this measures is the protocol's
cost on one GPU (the local search, the rounds, the waits, the merge, the host copy of the result), not NVLink: on 2
or more GPUs the exchange is not measured by this script.

Cases: 1M x 256 bf16 rows, 64 queries, min_score 0.6 (few hits); 1M x 768 float32 rows, one query, min_score 0
(every row); and that second search on an inbox reset to its smallest size before every call, so that each call
grows it (two rounds and a reserve).  Rank 0 prints one JSON line per case with the median host wall time of a
synchronous ``search_range`` for each exchange, the hits, the rounds of the last peer call, and the card's name and
power limit.
"""

from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.peer_filter_probe import card  # noqa: E402

CASES = [dict(name="few_hits", rows=1_000_000, dim=256, storage="bfloat16", batch=64, min_score=0.6),
         dict(name="every_row", rows=1_000_000, dim=768, storage="float32", batch=1, min_score=0.0),
         dict(name="every_row_grows", rows=1_000_000, dim=768, storage="float32", batch=1, min_score=0.0, grow=True)]


def rank_main(rank: int, args, store: str) -> None:
    import torch
    import torch.distributed as dist

    import typeagent_py_b200 as tab
    from oracle import vectorbase_oracle as O
    from typeagent_py_b200.sharded import RANGE_MIN_HITS, ShardedVectorBase

    torch.cuda.set_device(0)
    dist.init_process_group("gloo", init_method=f"file://{store}", rank=rank, world_size=args.world)
    settings = tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel())
    info = card() if rank == 0 else {}
    built = {}
    for case in CASES:
        shape = (case["rows"], case["dim"], case["storage"])
        if shape not in built:
            for sh in built.values():
                for s in sh.values():
                    s.close()
            built.clear()
            rng = np.random.default_rng(7)
            v = rng.standard_normal(shape[:2], dtype=np.float32)
            v /= np.linalg.norm(v, axis=1, keepdims=True)
            groups = {}
            for exchange in ("peer", "nccl"):
                sh = ShardedVectorBase(settings, device=0, storage_dtype=case["storage"], exchange=exchange)
                sh.deserialize(v)
                groups[exchange] = sh
            built[shape] = groups
            q = np.ascontiguousarray(v[rng.integers(0, case["rows"], 64)])
            del v
        groups = built[shape]
        qq = q[: case["batch"]]
        row = dict(case=case["name"], world=args.world, **{k: case[k] for k in ("rows", "dim", "storage", "batch",
                                                                                 "min_score")}, **info)
        for exchange, sh in groups.items():
            wall, hits = [], 0
            try:
                for i in range(args.reps + 2):
                    if case.get("grow") and exchange == "peer":  # back to the smallest inbox: the call grows it
                        eng = sh._engine
                        eng._range_reserve(dist, None, args.world, eng.range_capacity()[0] or 64, RANGE_MIN_HITS)
                        eng._range_cap_hint = RANGE_MIN_HITS
                    dist.barrier()
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    o, _, _ = sh.search_range(qq, case["min_score"])
                    if i >= 2:
                        wall.append((time.perf_counter() - t0) * 1e3)
                    hits = int(o[-1])
                row[f"{exchange}_wall_ms"] = round(float(np.median(wall)), 3)
                row["hits"] = hits
                if exchange == "peer":
                    row["peer_rounds"] = sh._engine.last_range_rounds
            except Exception as e:  # noqa: BLE001  (recorded, not hidden: the line says which exchange failed)
                row[f"{exchange}_error"] = f"{type(e).__name__}: {e}"[:200]
        row["process_group"] = "gloo (host memory)"
        if rank == 0:
            print(json.dumps(row), flush=True)
    for groups in built.values():
        for sh in groups.values():
            sh.close()
    dist.barrier()
    dist.destroy_process_group()


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=2)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    import torch
    import torch.multiprocessing as mp

    if not torch.cuda.is_available():
        print("peer_range_probe: no CUDA device", file=sys.stderr)
        return 1
    with tempfile.TemporaryDirectory() as tmp:
        os.environ.setdefault("GLOO_SOCKET_IFNAME", "lo")
        mp.spawn(rank_main, args=(args, os.path.join(tmp, "store")), nprocs=args.world, join=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
