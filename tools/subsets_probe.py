"""Per-query subsets probe: what one batched lookup costs when every query scores only its own candidate ordinals,
next to the two other ways of getting the same hits: a loop of one-query subset lookups, and one batched search
with a per-query row mask (2-D ``allowed=``, which cannot express repeated ordinals; the subsets here have none).

    python tools/subsets_probe.py [--batch 256] [--reps 3] [--json OUT]

Reports, in one run, the card's name and power limit and, for 10M x 768 bfloat16 and 1M x 768 float32 (unit-norm
Gaussian rows and queries, seeded), B queries with subsets of 1000, 4096 and 65536 distinct uniform ordinals each:
  * the batched call (``search_arrays(subsets=)`` for k = 10 and 100, ``search_range(subsets=)``) at min_score 0
    and 0.85: device time (CUDA events inside the library: the gather kernel and the whole call) and wall time,
    medians over reps;
  * the ordinal upload: a host-to-device copy of the same int64 ordinals timed on its own, and its share of the
    batched call's wall time;
  * gathered row bytes over the gather kernel's time, against the data sheet's 3.35 TB/s;
  * at min_score 0: the same batch as a loop of one-query ``search_arrays(subset=)`` calls (wall), and as one
    search with per-query masks (device and wall, masks uploaded beforehand).
Writes nothing unless ``--json`` is given.
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

HBM_TBS = 3.35


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def subset_masks(subsets, n):
    """int32 CUDA tensor [B, ceil(n / 32)] with the bits of each query's (distinct) ordinals set."""
    import torch

    words = (n + 31) // 32
    w = torch.zeros(len(subsets) * words, dtype=torch.int64, device="cuda")
    for b, s in enumerate(subsets):
        idx = torch.from_numpy(s).cuda()
        w.index_put_((b * words + (idx >> 5),), torch.ones_like(idx) << (idx & 31), accumulate=True)
    w = w.view(len(subsets), words)
    return (w - ((w >> 31) << 32)).to(torch.int32).contiguous()  # the low 32 bits as signed words


def upload_ms(ordinals, reps):
    import torch

    out = []
    for _ in range(reps + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        torch.from_numpy(ordinals).cuda()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
    return median(out[1:])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch

    import typeagent_py_b200 as tab
    from oracle import vectorbase_oracle as O

    out = card()
    out["batch"] = args.batch
    out["cases"] = []
    d = 768
    for n, dtype, name in ((10_000_000, torch.bfloat16, "bfloat16"), (1_000_000, torch.float32, "float32")):
        rows = unit_rows(n, d, dtype, seed=1)
        qd = unit_rows(args.batch, d, torch.float32, seed=2)
        q = qd.cpu().numpy()
        base = tab.VectorBase.from_device_tensor(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()), rows)
        base.enable_timing()
        elem = 2 if dtype == torch.bfloat16 else 4
        rng = np.random.default_rng(3)
        for m in (1000, 4096, 65536):
            subsets = [rng.permutation(np.unique(rng.integers(n, size=m + m * m // n + 64)))[:m]
                       for _ in range(args.batch)]
            ordinals = np.concatenate(subsets)
            up = upload_ms(ordinals, args.reps)
            gathered = len(ordinals) * d * elem
            masks = subset_masks(subsets, n)
            for ms in (0.0, 0.85):
                for k in (10, 100, None):  # None: the threshold form
                    dev, gather, wall = [], [], []
                    for i in range(args.reps + 1):
                        t0 = time.perf_counter()
                        if k is None:
                            base.search_range(q, ms, subsets=subsets)
                        else:
                            base.search_arrays(q, k, ms, subsets=subsets)
                        w = (time.perf_counter() - t0) * 1e3
                        t = base.last_timing()
                        if i:
                            dev.append(t["total_ms"])
                            gather.append(t["scan_ms"])
                            wall.append(w)
                    case = {"corpus": f"{n} x {d} {name}", "subset": m, "k": k if k else "range", "min_score": ms,
                            "device_ms": round(median(dev), 3), "gather_ms": round(median(gather), 3),
                            "wall_ms": round(median(wall), 3), "upload_ms": round(up, 3),
                            "upload_share_of_wall": round(up / median(wall), 3),
                            "gather_TBs": round(gathered / median(gather) / 1e9, 3),
                            "gather_share_of_3.35TBs": round(gathered / median(gather) / 1e9 / HBM_TBS, 3)}
                    if ms == 0.0 and k is not None:
                        t0 = time.perf_counter()
                        for b in range(args.batch):
                            base.search_arrays(q[b:b + 1], k, ms, subset=subsets[b])
                        case["loop_wall_ms"] = round((time.perf_counter() - t0) * 1e3, 3)
                        mdev, mwall = [], []
                        for i in range(args.reps + 1):
                            torch.cuda.synchronize()
                            t0 = time.perf_counter()
                            base.search_device(qd, k, ms, allowed=masks)
                            torch.cuda.synchronize()
                            if i:
                                mwall.append((time.perf_counter() - t0) * 1e3)
                                mdev.append(base.last_timing()["total_ms"])
                        case["masks_device_ms"] = round(median(mdev), 3)
                        case["masks_wall_ms"] = round(median(mwall), 3)
                    print(json.dumps(case), flush=True)
                    out["cases"].append(case)
            del masks
            torch.cuda.empty_cache()
        del base, rows
        torch.cuda.empty_cache()
    print(json.dumps(out, indent=1))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
