"""Sharded threshold-search probe: what ``ShardedVectorBase.search_range`` and its merge kernel cost.

    python tools/sharded_range_probe.py [--reps 5] [--json OUT]                       # one GPU
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \\
        --master-port 29518 tools/sharded_range_probe.py                               # N GPUs

Reports, in one run (rank 0 prints one JSON line): the card's name and power limit, then
  (i)  ``tav_merge_range`` alone on one GPU: W = 8 synthetic sorted lists of 1.25M hits each (one query),
       64 queries of 20k hits each over 8 lists, and 64 skewed queries over 8 lists (one of 1M hits, 63 of ~100);
       kernel time from CUDA events (median of --reps), and the bytes
       it reads and writes (every input hit once, every output hit once: 24 B per hit) over that time, against
       the 3.35 TB/s data-sheet HBM3 bandwidth;
  (ii) ``search_range`` end to end at the GPU count of the launch: 1M x 768 float32 with one query at min_score
       0.85 / 0.5 / 0.0, and 10M x 768 bfloat16 with 64 queries at min_score 0.6 (rows unit-norm Gaussian,
       queries with neighbours, seeded) — total wall time of the call, and the same stages run one by one with a
       synchronisation after each: local range search, offsets exchange, payload exchange (fetch + all-gather),
       merge; plus the bytes each rank receives in the payload exchange (world x padded total x 12).
With one GPU the sharded search returns the local result: no exchange and no merge run ("not run: world 1").
Writes nothing unless ``--json`` is given.
"""

from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.range_probe import HBM_TBPS, NOT_MEASURED, card, unit_rows  # noqa: E402


def merge_alone(w, per_query, reps, seed):
    """tav_merge_range over W synthetic lists holding per_query[q] hits of query q each: median kernel ms, bytes."""
    import torch

    from typeagent_py_b200 import _capi

    g = torch.Generator(device="cuda").manual_seed(seed)
    counts = torch.tensor(per_query, dtype=torch.int64, device="cuda")
    b, n = len(per_query), int(sum(per_query))
    seg = torch.repeat_interleave(torch.arange(b, device="cuda", dtype=torch.float64), counts)
    scores, items = [], []
    for lst in range(w):
        s = torch.rand(n, generator=g, device="cuda")
        order = torch.argsort(seg * 2 + (1 - s.double()))  # by query, then score descending
        scores.append(s[order])
        # distinct items, descending inside each list so that equal scores are already in the library's order
        items.append(lst * n + (n - 1) - torch.arange(n, device="cuda", dtype=torch.int64))
    scores, items = torch.stack(scores).contiguous(), torch.stack(items).contiguous()
    offsets = torch.cat([torch.zeros(1, dtype=torch.int64, device="cuda"), counts.cumsum(0)]).repeat(w, 1).contiguous()
    out_o = torch.empty(b + 1, dtype=torch.int64, device="cuda")
    out_i = torch.empty(w * n, dtype=torch.int64, device="cuda")
    out_s = torch.empty(w * n, dtype=torch.float32, device="cuda")
    lib = _capi.load()
    stream = torch.cuda.current_stream().cuda_stream

    def run():
        _capi.check(lib.tav_merge_range(0, w, b, C.c_void_p(offsets.data_ptr()), b + 1, C.c_void_p(items.data_ptr()),
                                        n, C.c_void_p(scores.data_ptr()), n, 0, C.c_void_p(out_o.data_ptr()),
                                        C.c_void_p(out_i.data_ptr()), C.c_void_p(out_s.data_ptr()),
                                        C.c_void_p(stream)))

    run()
    torch.cuda.synchronize()
    # check once: every query's output is its lists' scores in descending order
    oo = out_o.cpu()
    assert int(oo[-1]) == w * n
    for q in {0, b - 1}:
        lo, hi = int(oo[q]), int(oo[q + 1])
        part = torch.cat([scores[lst, int(offsets[0, q]):int(offsets[0, q + 1])] for lst in range(w)])
        assert torch.equal(out_s[lo:hi], part.sort(descending=True)[0])
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    times.sort()
    ms = times[len(times) // 2]
    moved = 2 * 12 * w * n + 8 * (w + 1) * (b + 1)
    tbps = moved / (ms * 1e-3) / 1e12
    return {"lists": w, "queries": b, "hits_per_list_largest_query": max(per_query),
            "hits_per_list_smallest_query": min(per_query), "hits": w * n, "kernel_ms": ms, "bytes": moved,
            "TBps": tbps, "share_of_3.35TBps": tbps / HBM_TBPS}


def staged(sh, q, ms):
    """search_range's steps one by one (as ShardedVectorBase.search_range runs them), synchronised after each."""
    import torch

    from typeagent_py_b200.sharded import offsets_with_status, pack_range_payload, range_pad

    eng, dist, world = sh._engine, sh._dist, sh.world
    b = len(q)
    t = {}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    local = eng.range_local(q, ms, sh.local_range[0], False)
    offsets = local.offsets
    t["local_range_search_ms"] = (time.perf_counter() - t0) * 1e3
    t1 = time.perf_counter()
    mine = torch.from_numpy(offsets_with_status(offsets, False)).to(eng.comm_device())
    offsets_all = torch.empty((world, b + 2), dtype=torch.int64, device=eng.comm_device())
    dist.all_gather_into_tensor(offsets_all.view(-1), mine)
    host = offsets_all.cpu().numpy()
    t["offsets_exchange_ms"] = (time.perf_counter() - t1) * 1e3
    totals = host[:, b]
    t_pad = range_pad(totals)
    t2 = time.perf_counter()
    send = pack_range_payload(local, t_pad, eng.comm_device())
    payload = torch.empty((world, 12 * t_pad), dtype=torch.uint8, device=eng.comm_device())
    dist.all_gather_into_tensor(payload.view(-1), send)
    torch.cuda.synchronize()
    t["payload_exchange_ms"] = (time.perf_counter() - t2) * 1e3
    t3 = time.perf_counter()
    out = eng.merge_range(offsets_all, payload, world, b, t_pad, int(totals.sum()), False)
    torch.cuda.synchronize()
    t["merge_ms"] = (time.perf_counter() - t3) * 1e3
    t["stages_sum_ms"] = sum(t.values())
    t["payload_bytes_received_per_rank"] = world * t_pad * 12
    del out
    return t


def end_to_end(sh, q, ms, reps):
    import torch

    got = sh.search_range(q, ms)
    walls = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        sh.search_range(q, ms)
        walls.append((time.perf_counter() - t0) * 1e3)
    walls.sort()
    row = {"min_score": ms, "queries": len(q), "hits": int(got[0][-1]), "total_wall_ms": walls[len(walls) // 2]}
    if sh.world > 1:
        stages = [staged(sh, q, ms) for _ in range(reps)]
        stages.sort(key=lambda s: s["stages_sum_ms"])
        row.update(stages[len(stages) // 2])
    else:
        row.update({k: "not run: world 1" for k in ("offsets_exchange_ms", "payload_exchange_ms", "merge_ms",
                                                    "payload_bytes_received_per_rank")})
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--big-rows", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    import torch.distributed as dist

    if not torch.cuda.is_available():
        raise SystemExit("sharded_range_probe needs a CUDA device (no CPU fallback)")
    import typeagent_py_b200 as tab
    from oracle import vectorbase_oracle as O
    from typeagent_py_b200.sharded import ShardedVectorBase, shard_bounds

    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    else:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29519")
        dist.init_process_group("gloo", rank=0, world_size=1)
    report = card()
    report["gpus"] = world
    if rank == 0:
        report["merge_alone"] = [merge_alone(8, [1_250_000], args.reps, seed=1),
                                 merge_alone(8, [2_500] * 64, args.reps, seed=2),
                                 merge_alone(8, [125_000] + [13] * 63, args.reps, seed=3)]
        torch.cuda.empty_cache()
    settings = tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel())
    d = args.dim

    def sharded(n, dtype, seed):
        lo, hi = shard_bounds(n, world)[rank]
        rows = unit_rows(hi - lo, d, dtype, seed=seed + rank)
        sh = ShardedVectorBase(settings, device=local, storage_dtype="float32" if dtype == torch.float32 else "bfloat16")
        sh.load_local_shard(rows, n)
        return sh, rows

    def replicated(x):
        t = torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()
        if world > 1:
            dist.broadcast(t, 0)
        return t.cpu().numpy()

    # 1M x 768 float32, one query with neighbours (rank 0's row 12345)
    sh, rows = sharded(args.rows, torch.float32, seed=1)
    q = unit_rows(1, d, torch.float32, seed=2)
    q = 0.5 * q + 0.5 * rows[12345:12346]
    q = replicated((q / q.norm()).cpu().numpy())
    report["f32_1M_one_query"] = {"rows": args.rows, "dim": d,
                                  "results": [end_to_end(sh, q, ms, args.reps) for ms in (0.85, 0.5, 0.0)]}
    del sh, rows
    torch.cuda.empty_cache()
    # 10M x 768 bfloat16, 64 queries with neighbours
    try:
        sh, rows = sharded(args.big_rows, torch.bfloat16, seed=3)
        qb = unit_rows(64, d, torch.float32, seed=4)
        qb = 0.6 * qb + 0.4 * rows[: 64 * 97: 97].float()
        qb = replicated((qb / qb.norm(dim=1, keepdim=True)).cpu().numpy())
        report["bf16_10M_B64"] = {"rows": args.big_rows, "dim": d, "results": [end_to_end(sh, qb, 0.6, args.reps)]}
        del sh, rows
    except torch.cuda.OutOfMemoryError as e:
        report["bf16_10M_B64"] = {"total_wall_ms": NOT_MEASURED, "why": repr(e)}
    dist.destroy_process_group()
    if rank == 0:
        line = json.dumps(report)
        print(line)
        if args.json:
            with open(args.json, "w") as f:
                f.write(line + "\n")


if __name__ == "__main__":
    main()
