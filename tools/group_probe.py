"""Grouped lookups probe: what ``search_groups`` costs next to the plain top-k and next to the exact route without it
(``search_range`` plus a fold of every hit on the host), and what one host query through
``fuzzy_lookup_embedding_grouped`` costs next to ``fuzzy_lookup_embedding``.

    python tools/group_probe.py [--batch 256] [--reps 5] [--json OUT]

Reports, in one run, the card's name and power limit and:
  * 10M x 768 bfloat16 (unit-norm Gaussian rows and queries, seeded), B queries, k = 100, min_score 0:
    ``search_arrays`` against ``search_groups`` with groups of 1 row, 8 contiguous rows, 8 random rows (a random
    assignment to N / 8 groups) and Zipf-sized runs; the queries redone (``last_redone``);
  * the same index and queries at min_score 0.56 (a few thousand hits per query): ``search_range`` plus a numpy fold
    of every hit to its groups' first rows, against ``search_groups`` at that floor;
  * one host query: 10k x 384 float32 at min_score 0.85, 1M x 768 float32 at 0.85 and 0.5, groups of 8 contiguous
    rows, k = 10.
Times are medians over the repetitions after one warm-up of every shape: device time from CUDA events recorded on
the current stream around each call (the calls synchronise), wall time from the host clock.  Writes nothing unless
``--json``.
"""

from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.range_probe import card, unit_rows  # noqa: E402


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def timed(fn, reps):
    """(device ms, wall ms) medians over reps after one warm-up, and the last result."""
    import torch

    out = fn()
    dev, wall = [], []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        a.record()
        out = fn()
        b.record()
        b.synchronize()
        wall.append((time.perf_counter() - t0) * 1e3)
        dev.append(a.elapsed_time(b))
    return round(median(dev), 3), round(median(wall), 3), out


def host_fold(offsets, items, scores, groups):
    """search_range's hits -> every query's groups in the order of their first rows (the exact route without
    grouped lookups)."""
    out = []
    for i in range(len(offsets) - 1):
        it = items[offsets[i]:offsets[i + 1]]
        g = groups[it]
        _, first = np.unique(g, return_index=True)
        keep = np.sort(first)
        out.append((g[keep], scores[offsets[i]:offsets[i + 1]][keep]))
    return out


def layouts(n, seed):
    rng = np.random.default_rng(seed)
    zipf = np.minimum(rng.zipf(1.5, n), 4096)
    runs = np.repeat(np.arange(len(zipf)), zipf)[:n]
    return {"1": np.arange(n, dtype=np.int32), "8 contiguous": (np.arange(n) // 8).astype(np.int32),
            "8 random": rng.integers(0, n // 8, n).astype(np.int32), "zipf": runs.astype(np.int32)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--json")
    args = ap.parse_args()
    import torch

    import typeagent_py_b200 as tab
    from oracle import vectorbase_oracle as O

    res = {**card(), "batch": args.batch, "reps": args.reps, "cells": []}
    print(json.dumps({k: res[k] for k in ("card", "power_limit")}), flush=True)
    settings = tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel())

    n = args.rows
    t = unit_rows(n, 768, torch.bfloat16, 1)
    q = unit_rows(args.batch, 768, torch.float32, 2).cpu().numpy()
    base = tab.VectorBase.from_device_tensor(settings, t)
    dev, wall, _ = timed(lambda: base.search_arrays(q, 100, 0.0), args.reps)
    cell = {"shape": f"{n} x 768 bf16", "call": "search_arrays", "k": 100, "min_score": 0.0, "device_ms": dev,
            "wall_ms": wall}
    res["cells"].append(cell)
    print(json.dumps(cell), flush=True)
    groups = layouts(n, 3)
    for name, g in groups.items():
        gt = torch.from_numpy(g).cuda()
        dev, wall, _ = timed(lambda: base.search_groups(q, 100, gt), args.reps)
        cell = {"shape": f"{n} x 768 bf16", "call": "search_groups", "groups": name, "k": 100, "min_score": 0.0,
                "device_ms": dev, "wall_ms": wall, "last_redone": base.last_redone}
        res["cells"].append(cell)
        print(json.dumps(cell), flush=True)
    g8 = groups["8 contiguous"]
    g8t = torch.from_numpy(g8).cuda()
    dev, wall, r = timed(lambda: host_fold(*base.search_range(q, 0.56), g8), args.reps)
    cell = {"shape": f"{n} x 768 bf16", "call": "search_range + host fold", "groups": "8 contiguous",
            "min_score": 0.56, "device_ms": dev, "wall_ms": wall, "hits": int(sum(len(x[0]) for x in r))}
    res["cells"].append(cell)
    print(json.dumps(cell), flush=True)
    dev, wall, r = timed(lambda: base.search_groups(q, 100, g8t, min_score=0.56), args.reps)
    cell = {"shape": f"{n} x 768 bf16", "call": "search_groups", "groups": "8 contiguous", "k": 100,
            "min_score": 0.56, "device_ms": dev, "wall_ms": wall, "last_redone": base.last_redone}
    res["cells"].append(cell)
    print(json.dumps(cell), flush=True)
    del base, t
    torch.cuda.empty_cache()

    for rows, d, floors in ((10_000, 384, (0.85,)), (1_000_000, 768, (0.85, 0.5))):
        v = unit_rows(rows, d, torch.float32, 4).cpu().numpy()
        one = unit_rows(1, d, torch.float32, 5).cpu().numpy()[0]
        b1 = tab.VectorBase(settings)
        b1.add_embeddings(None, v)
        g = (np.arange(rows) // 8).astype(np.int32)
        for ms in floors:
            for call, fn in (("fuzzy_lookup_embedding", lambda: b1.fuzzy_lookup_embedding(one, 10, ms)),
                             ("fuzzy_lookup_embedding_grouped",
                              lambda: b1.fuzzy_lookup_embedding_grouped(one, g, 10, ms))):
                dev, wall, _ = timed(fn, max(args.reps, 20))
                cell = {"shape": f"{rows} x {d} f32", "call": call, "k": 10, "min_score": ms, "device_ms": dev,
                        "wall_ms": wall}
                res["cells"].append(cell)
                print(json.dumps(cell), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
