"""Per-query mask probe: what one batched search with a mask per query costs on the GPU, next to no mask, one
shared mask, and the status quo of one masked search per query.

    python tools/query_mask_probe.py [--rows 10000000] [--batch 256] [--k 100] [--reps 3] [--json OUT]

Reports, in one run: the card's name and power limit; at rows x 768 bfloat16 (unit-norm Gaussian rows and
queries, seeded), B queries, top-k: the MAIN kernel time and the whole search's device time (median over reps,
CUDA events inside the library) and the number of queries redone by the exact row scan, for no mask, one
shared mask of density 0.1, and random per-query masks at densities 1, 0.1, 0.01 and 1e-3; the same for
``search_range`` at min_score 0.6; and a few one-query masked searches (the status quo), timed and reported
per query.  Writes nothing unless ``--json`` is given.  Anything not measured is reported as "not measured".
"""

from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.range_probe import card, unit_rows  # noqa: E402


def packed_masks(b, n, density, seed):
    """int32 CUDA tensor [b, ceil(n / 32)]: random per-query masks, bit r of word r // 32 = row r."""
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    words = (n + 31) // 32
    out = torch.empty((b, words), dtype=torch.int32, device="cuda")
    weights = (torch.ones(32, dtype=torch.int64, device="cuda") << torch.arange(32, device="cuda"))
    for q0 in range(0, b, 8):
        bits = torch.zeros((min(8, b - q0), words * 32), dtype=torch.bool, device="cuda")
        bits[:, :n] = torch.rand((len(bits), n), generator=g, device="cuda") < density
        w = (bits.view(len(bits), words, 32).to(torch.int64) * weights).sum(dim=2)
        out[q0:q0 + len(bits)] = (w - ((w >> 31) << 32)).to(torch.int32)  # the low 32 bits as a signed word
    return out


def timed_topk(base, q, k, allowed, reps):
    """(median search ms, median MAIN ms, redone queries of the last run)."""
    rows, redone = [], 0
    for i in range(reps + 1):
        base.search_device(q, k, 0.0, defer_check=True, allowed=allowed)
        redone = base.finish_search()
        t = base.last_timing()
        if i:
            rows.append((t["total_ms"], t["scan_ms"]))
    rows.sort()
    return rows[len(rows) // 2] + (redone,)


def timed_range(base, q, ms, allowed, reps):
    rows, total = [], 0
    for i in range(reps + 1):
        offsets, _, _ = base.search_range(q, ms, allowed=allowed)
        t = base.last_timing()
        total = int(offsets[-1])
        if i:
            rows.append((t["total_ms"], t["scan_ms"]))
    rows.sort()
    return rows[len(rows) // 2] + (total,)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--single", type=int, default=3, help="one-query masked searches timed (status quo)")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch

    import typeagent_py_b200 as tab
    from oracle import vectorbase_oracle as O

    out = card()
    out["shape"] = f"{args.rows} x {args.dim} bfloat16, B = {args.batch}, k = {args.k}"
    rows = unit_rows(args.rows, args.dim, torch.bfloat16, seed=1)
    q = unit_rows(args.batch, args.dim, torch.float32, seed=2)
    base = tab.VectorBase.from_device_tensor(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()), rows)
    base.enable_timing()
    shared = packed_masks(1, args.rows, 0.1, seed=3)[0].cpu().numpy().view(np.uint32)
    cases = [("no mask", None), ("shared mask, density 0.1", shared)]
    for dens in (1.0, 0.1, 0.01, 1e-3):
        cases.append((f"per-query masks, density {dens:g}", dens))
    topk, rng = {}, {}
    qh = q.cpu().numpy()
    for name, m in cases:
        allowed = packed_masks(args.batch, args.rows, m, seed=4) if isinstance(m, float) else m
        total, main_ms, redone = timed_topk(base, q, args.k, allowed, args.reps)
        topk[name] = {"search_ms": round(total, 3), "main_ms": round(main_ms, 3), "redone": redone}
        total, main_ms, hits = timed_range(base, qh, 0.6, allowed, args.reps)
        rng[name] = {"search_ms": round(total, 3), "main_ms": round(main_ms, 3), "hits": hits}
        print(f"{name:34s} top-k {topk[name]}  range(0.6) {rng[name]}", flush=True)
        del allowed
        torch.cuda.empty_cache()
    out["topk"], out["range_min_score_0.6"] = topk, rng

    # status quo: one masked search per query (each query's own mask uploaded as the row mask first)
    masks = packed_masks(args.single, args.rows, 0.1, seed=5)
    per = []
    for b in range(args.single):
        words = masks[b].cpu().numpy().view(np.uint32)
        base.search_device(q[b:b + 1], args.k, 0.0, allowed=words)  # upload + warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        base.search_device(q[b:b + 1], args.k, 0.0, allowed=words)
        torch.cuda.synchronize()
        wall = (time.perf_counter() - t0) * 1e3
        per.append((base.last_timing()["total_ms"], wall))
    out["one_query_masked_search"] = {
        "queries_timed": args.single,
        "device_ms_per_query": [round(d, 3) for d, _ in per],
        "wall_ms_per_query": [round(w, 3) for _, w in per],
        "mask_upload": "not measured",
    }
    print(json.dumps(out, indent=1))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
