"""Per-query subsets from device tensors probe: what the batched subset lookup costs when the candidate lists are
already on the GPU (``search_device`` / ``search_range_device`` with ``subsets=``), next to the host-CSR form
(``search_arrays`` / ``search_range`` with ``subsets=``) on the same index and the same candidates.

    python tools/subsets_device_probe.py [--batch 256] [--reps 5] [--json OUT]

Reports, in one run, the card's name and power limit and, for 10M x 768 bfloat16 and 1M x 768 float32 (unit-norm
Gaussian rows and queries, seeded), B queries with subsets of 1000, 4096 and 65536 distinct uniform ordinals each,
k = 10, k = 100 and the threshold form, at min_score 0 and 0.85, three forms alternated within every repetition:
  * host: the host-CSR call, from B numpy arrays of ordinals (what a caller holding host lists pays);
  * sync: the device call without ``defer_check`` (it synchronises once to read the device checks' status);
  * deferred: the device call with ``defer_check=True`` and its ``finish_search()``.
Each form's device time (CUDA events inside the library, first launch to last result) and wall time (host clock,
the stream synchronised before and after), medians over the repetitions after one warm-up of every shape.  The
warm-up also compares every form's result with the host form's, bit for bit.  Writes nothing unless ``--json``.
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


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--reps", type=int, default=5)
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
        rng = np.random.default_rng(3)
        for m in (1000, 4096, 65536):
            subsets = [rng.permutation(np.unique(rng.integers(n, size=m + m * m // n + 64)))[:m]
                       for _ in range(args.batch)]
            ordinals = torch.from_numpy(np.concatenate(subsets)).cuda()
            offsets = torch.arange(0, (args.batch + 1) * m, m, dtype=torch.int64, device="cuda")
            csr = (offsets, ordinals)
            r_out = (torch.empty(args.batch + 1, dtype=torch.int64, device="cuda"),
                     torch.empty(ordinals.numel(), dtype=torch.int64, device="cuda"),
                     torch.empty(ordinals.numel(), dtype=torch.float32, device="cuda"))
            for ms in (0.0, 0.85):
                for k in (10, 100, None):  # None: the threshold form

                    def host():
                        if k is None:
                            return base.search_range(q, ms, subsets=subsets)
                        return base.search_arrays(q, k, ms, subsets=subsets)

                    def device(defer):
                        if k is None:
                            got = base.search_range_device(qd, ms, out=r_out, subsets=csr, defer_check=defer)
                        else:
                            got = base.search_device(qd, k, ms, subsets=csr, defer_check=defer)
                        if defer:
                            base.finish_search()
                        return got

                    forms = {"host": host, "sync": lambda: device(False), "deferred": lambda: device(True)}
                    dev = {f: [] for f in forms}
                    wall = {f: [] for f in forms}
                    for i in range(args.reps + 1):
                        res = {}
                        for f, call in forms.items():
                            torch.cuda.synchronize()
                            t0 = time.perf_counter()
                            res[f] = call()
                            torch.cuda.synchronize()
                            w = (time.perf_counter() - t0) * 1e3
                            if i:
                                wall[f].append(w)
                                dev[f].append(base.last_timing()["total_ms"])
                        if i == 0:  # the same result from every form
                            h = res["host"]
                            for f in ("sync", "deferred"):
                                g = tuple(t.cpu().numpy() for t in res[f])
                                if k is None:
                                    same = (np.array_equal(g[0], h[0]) and np.array_equal(g[1][:h[0][-1]], h[1])
                                            and np.array_equal(g[2][:h[0][-1]].view(np.uint32), h[2].view(np.uint32)))
                                else:
                                    kk = h[0].shape[1]
                                    same = (np.array_equal(g[2], h[2]) and np.array_equal(g[0][:, :kk], h[0])
                                            and np.array_equal(g[1][:, :kk].view(np.uint32), h[1].view(np.uint32)))
                                assert same, f"{f} differs from the host form: {name} m={m} k={k} ms={ms}"
                    case = {"corpus": f"{n} x {d} {name}", "subset": m, "k": k if k else "range", "min_score": ms}
                    for f in forms:
                        case[f"{f}_device_ms"] = round(median(dev[f]), 3)
                        case[f"{f}_wall_ms"] = round(median(wall[f]), 3)
                    print(json.dumps(case), flush=True)
                    out["cases"].append(case)
            del ordinals, offsets, csr, r_out
            torch.cuda.empty_cache()
        del base, rows
        torch.cuda.empty_cache()
    print(json.dumps(out, indent=1))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
