"""Probe of the multi-device search (``tav_multi_search``, ``VectorBase(devices=[...])``): the wall time of one lookup
over W = 1, 2, 4 and 8 shards at the benchmark's c3 shape and of a one-query lookup.

    python tools/multi_device_probe.py [--rows 10000000] [--dim 768] [--batch 256] [--k 100] [--reps 10]
                                       [--shards 1,2,4,8] [--json OUT]

Rows are unit-norm Gaussian bfloat16, generated on the device block by block and appended from device memory (no
host mirror), seeded.  With one shard the same lookups also go through ``tav_search`` on that index.  Shard g lives on device g when the machine has W devices or more; otherwise every shard repeats device 0,
and the output says so: shards that share one GPU measure the fan-out's overhead, not a speed-up.  Time: the host
clock around each call (the call synchronises once at its end), the median of ``--reps`` after two warm-ups.  The
card's name and power limit are read in the same run and printed beside every number.  Writes nothing unless
``--json`` is given.
"""

from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info() -> str:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError("nvidia-smi failed: " + out.stderr)
    return out.stdout.strip().splitlines()[0]


def wall_ms(fn, reps) -> float:
    fn()
    fn()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        times.append((time.perf_counter() - t0) * 1e3)
    return round(statistics.median(times), 3)


def build_shards(lib, _capi, devices, rows, dim, seed):
    import torch

    from typeagent_py_b200.multi import even_starts

    starts = even_starts(rows, len(devices))
    shards = []
    chunk = 1 << 20
    for g, dev in enumerate(devices):
        h = C.c_void_p()
        _capi.check(lib.tav_create(dev, dim, _capi.TAV_BF16, 0, starts[g + 1] - starts[g], C.byref(h)))
        shards.append(h)
        gen = torch.Generator(device=f"cuda:{dev}").manual_seed(seed + g)
        for lo in range(starts[g], starts[g + 1], chunk):
            n = min(chunk, starts[g + 1] - lo)
            block = torch.randn((n, dim), generator=gen, device=f"cuda:{dev}", dtype=torch.float32)
            block = (block / block.norm(dim=1, keepdim=True)).to(torch.bfloat16)   # unit-norm rows, as bench.py
            torch.cuda.synchronize(dev)
            _capi.check(lib.tav_append(h, C.c_void_p(block.data_ptr()), n, dim, _capi.TAV_BF16, 1, None))
            torch.cuda.synchronize(dev)
            del block
    return shards, starts


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--shards", default="1,2,4,8")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch

    from typeagent_py_b200 import _capi

    if not torch.cuda.is_available():
        raise SystemExit("multi_device_probe needs a CUDA device")
    lib = _capi.load()
    n_dev = torch.cuda.device_count()
    card = gpu_info()
    rng = np.random.default_rng(7)
    queries = rng.standard_normal((args.batch, args.dim)).astype(np.float32)
    queries /= np.linalg.norm(queries, axis=1, keepdims=True)
    results = []
    for w in [int(s) for s in args.shards.split(",")]:
        devices = list(range(w)) if n_dev >= w else [0] * w
        shared = n_dev < w and w > 1
        shards, starts = build_shards(lib, _capi, devices, args.rows, args.dim, seed=11)
        arr = (C.c_void_p * w)(*[h.value for h in shards])
        m = C.c_void_p()
        _capi.check(lib.tav_multi_create(devices[0], w, arr, C.byref(m)))
        st = np.asarray(starts, np.int64)
        row = {"shards": w, "devices": devices, "shared_gpu": shared, "gpu": card, "rows": args.rows, "dim": args.dim}
        for name, b, k in (("batch", args.batch, args.k), ("one_query", 1, 10)):
            items = np.empty((b, k), np.int64)
            scores = np.empty((b, k), np.float32)
            counts = np.empty(b, np.int32)
            q = np.ascontiguousarray(queries[:b])

            def call():
                _capi.check(lib.tav_multi_search(m, st.ctypes.data_as(C.c_void_p), q.ctypes.data_as(C.c_void_p), b, k,
                                                 C.c_float(0.0), 0, None, 0, items.ctypes.data_as(C.c_void_p),
                                                 scores.ctypes.data_as(C.c_void_p), counts.ctypes.data_as(C.c_void_p)))

            def one_index():
                _capi.check(lib.tav_search(shards[0], q.ctypes.data_as(C.c_void_p), b, k, C.c_float(0.0), 0, None, 0,
                                           0, items.ctypes.data_as(C.c_void_p), scores.ctypes.data_as(C.c_void_p),
                                           counts.ctypes.data_as(C.c_void_p), None))

            row[f"{name}_ms"] = wall_ms(call, args.reps)
            row[f"{name}_shape"] = [b, k]
            if w == 1:  # the same lookup through tav_search on the one index: the fan-out's own cost
                row[f"{name}_tav_search_ms"] = wall_ms(one_index, args.reps)
        lib.tav_multi_destroy(m)
        for h in shards:
            lib.tav_destroy(h)
        results.append(row)
        note = " (shards share one GPU: overhead, not scaling)" if shared else ""
        ref = (f" (tav_search on the one index: {row['batch_tav_search_ms']} / {row['one_query_tav_search_ms']} ms)"
               if w == 1 else "")
        print(f"W={w} devices={devices}: B={args.batch} k={args.k} {row['batch_ms']} ms, "
              f"1 query k=10 {row['one_query_ms']} ms{ref} on {card}{note}", flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
