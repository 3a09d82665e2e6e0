#!/usr/bin/env python3
"""Costs of the sharded filtered and subset lookups on one GPU:

  1. tav_merge_topk_ordered (orders 0..3) against tav_merge_topk: W = 8 lists, B = 256 queries, k = 100, device
     time from CUDA events;
  2. one subset lookup (tav_search with a subset) with and without TAV_ITEMS_AS_POSITIONS, host wall time: the
     single-launch form (one query, 4096 ordinals) and the general form (16 queries, 200k ordinals);
  3. one-rank ShardedVectorBase filtered lookups against VectorBase, host wall time (the per-rank steps, the
     ordered merge and the decode; a one-rank group has no exchange).

    python tools/sharded_filter_probe.py [--rows 2000000] [--dim 768]

Prints one JSON line per measurement.  The exchange over two or more GPUs is not measured here.
"""

from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import socket
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import typeagent_py_b200 as tab  # noqa: E402
from oracle import vectorbase_oracle as O  # noqa: E402
from typeagent_py_b200 import _capi  # noqa: E402
from typeagent_py_b200.sharded import ShardedVectorBase, packed_layout  # noqa: E402


def median_ms(fn, reps=30, warm=5):
    for _ in range(warm):
        fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def merge_probe(w=8, b=256, k=100, reps=200):
    lib = _capi.load()
    dev = torch.device("cuda", 0)
    off_s, off_c, total = packed_layout(b, k)
    rng = np.random.default_rng(0)
    host = np.zeros((w, total), np.uint8)
    for g in range(w):
        items = host[g, : b * k * 8].view(np.int64).reshape(b, k)
        scores = host[g, off_s: off_s + b * k * 4].view(np.float32).reshape(b, k)
        counts = host[g, off_c: off_c + b * 4].view(np.int32)
        s = np.sort(rng.integers(0, 64, (b, k)).astype(np.float32) / 64, axis=1)[:, ::-1]  # many equal scores
        scores[:] = s
        items[:] = g * b * k + np.arange(b * k).reshape(b, k)
        counts[:] = k
    buf = torch.from_numpy(host).to(dev)
    out_i = torch.empty((b, k), dtype=torch.int64, device=dev)
    out_s = torch.empty((b, k), dtype=torch.float32, device=dev)
    out_c = torch.empty((b,), dtype=torch.int32, device=dev)
    base = buf.data_ptr()
    args = (C.c_void_p(base), C.c_void_p(base + off_s), C.c_void_p(base + off_c), total // 8, total // 4, total // 4)
    outs = (C.c_void_p(out_i.data_ptr()), C.c_void_p(out_s.data_ptr()), C.c_void_p(out_c.data_ptr()))
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    runs = {"tav_merge_topk": lambda: lib.tav_merge_topk(0, w, b, k, *args, *outs, stream)}
    for order in range(4):
        runs[f"ordered_{order}"] = lambda o=order: lib.tav_merge_topk_ordered(0, w, b, k, *args, o, *outs, stream)
    res = {}
    for name, fn in runs.items():
        for _ in range(10):
            _capi.check(fn())
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        res[name] = round(e0.elapsed_time(e1) / reps * 1e3, 2)
    print(json.dumps({"probe": "merge", "W": w, "B": b, "k": k, "us_per_merge": res}), flush=True)


def subset_probe(v_dev, d):
    lib = _capi.load()
    vb = tab.VectorBase.from_device_tensor(tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel()), v_dev)
    lib_, ix = vb._ensure_device()
    n = v_dev.shape[0]
    rng = np.random.default_rng(1)
    for b, m, k in ((1, 4096, 10), (16, 200_000, 100)):
        q = np.ascontiguousarray(rng.standard_normal((b, d)).astype(np.float32) / np.sqrt(d))
        sub = np.ascontiguousarray(rng.integers(0, n, m).astype(np.int64))
        items, scores, counts = np.empty((b, k), np.int64), np.empty((b, k), np.float32), np.empty(b, np.int32)
        res = {}
        for name, flags in (("ordinals", 0), ("positions", _capi.TAV_ITEMS_AS_POSITIONS)):
            def call(flags=flags):
                _capi.check(lib.tav_search(ix, q.ctypes.data_as(C.c_void_p), b, k, C.c_float(0.0), flags,
                                           sub.ctypes.data_as(C.c_void_p), m, 0, items.ctypes.data_as(C.c_void_p),
                                           scores.ctypes.data_as(C.c_void_p), counts.ctypes.data_as(C.c_void_p), None))
            res[name] = round(median_ms(call, reps=50) * 1e3, 1)
        print(json.dumps({"probe": "subset_search", "B": b, "subset": m, "k": k, "launches": vb.last_timing()["launches"],
                          "us": res}), flush=True)


def one_rank_probe(v, d):
    import torch.distributed as dist

    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    dist.init_process_group("gloo", rank=0, world_size=1, init_method=f"tcp://127.0.0.1:{port}")
    try:
        settings = tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel())
        n = len(v)
        one = tab.VectorBase(settings, storage_dtype="bfloat16")
        one.add_embeddings(None, v)
        sh = ShardedVectorBase(settings, device=0, storage_dtype="bfloat16")
        sh.deserialize(v)
        rng = np.random.default_rng(2)
        q = rng.standard_normal((16, d)).astype(np.float32) / np.sqrt(d)
        allowed = rng.random(n) < 0.5
        pred = lambda i: bool(allowed[i])  # noqa: E731
        sub = rng.integers(0, n, 4096).tolist()
        cases = {
            "predicate_k10_cached": lambda x: x.fuzzy_lookup_embedding(q[0], 10, 0.0, predicate=pred),
            "in_subset_4096_k10": lambda x: x.fuzzy_lookup_embedding_in_subset(q[0], sub, 10, 0.0),
            "search_arrays_mask_B16_k100": lambda x: x.search_arrays(q, 100, 0.0, allowed=allowed),
            "search_arrays_subset_B16_k100": lambda x: x.search_arrays(q, 100, 0.0, subset=sub),
        }
        for name, fn in cases.items():
            res = {"VectorBase": round(median_ms(lambda: fn(one), reps=20), 3),
                   "ShardedVectorBase_1rank": round(median_ms(lambda: fn(sh), reps=20), 3)}
            print(json.dumps({"probe": "one_rank", "case": name, "rows": n, "ms": res}), flush=True)
    finally:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=2_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--host-rows", type=int, default=200_000, help="rows of the one-rank comparison (host corpus)")
    a = ap.parse_args()
    print(json.dumps({"gpu": torch.cuda.get_device_name(0)}), flush=True)
    merge_probe()
    v_dev = (torch.randn(a.rows, a.dim, device="cuda") / a.dim ** 0.5).to(torch.bfloat16)
    subset_probe(v_dev, a.dim)
    del v_dev
    torch.cuda.empty_cache()
    rng = np.random.default_rng(3)
    one_rank_probe((rng.standard_normal((a.host_rows, a.dim)) / np.sqrt(a.dim)).astype(np.float32), a.dim)


if __name__ == "__main__":
    main()
