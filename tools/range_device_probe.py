"""Probe of the threshold search into caller tensors (``search_range_device`` / ``tav_range_search_into``): its
device time next to ``tav_range_search`` at the shapes of DESIGN.md section 3.4's table, and the host time of one
deferred call.

    python tools/range_device_probe.py [--rows 1000000] [--big-rows 10000000] [--reps 5] [--json OUT]

Shapes: rows x 768 float32, one query, min_score 0.85 / 0.5 / 0.0 (the row scan); big-rows x 768 bfloat16, 64
queries, min_score 0.6, and 0.55 where every query overflows the default region (the tensor cores).  Rows are unit-norm Gaussian, seeded (tools/range_probe.py).  Device
time: CUDA events around one call, the median of ``--reps`` after a warm-up; ``tav_range_search`` writes its
offsets to the device and leaves its hits in the library (no fetch), the new call writes everything into caller
tensors sized to the total.  Host time: the wall clock of one deferred call (``defer_check=True``), which queues
its work and returns.  The card's name and power limit are read in the same run.  Writes nothing unless
``--json`` is given.
"""

from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def device_ms(fn, reps):
    import torch

    fn()
    times = []
    for _ in range(reps):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        fn()
        end.record()
        end.synchronize()
        times.append(start.elapsed_time(end))
    return statistics.median(times)


def probe(base, q, ms, reps):
    import torch

    from typeagent_py_b200 import _capi

    lib, ix = base._ensure_device()
    b = q.shape[0]
    offsets = torch.empty(b + 1, dtype=torch.int64, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    flags = _capi.TAV_QUERIES_ON_DEVICE | _capi.TAV_OUTPUTS_ON_DEVICE

    def old():
        _capi.check(lib.tav_range_search(ix, C.c_void_p(q.data_ptr()), b, C.c_float(ms), flags, None, 0, 0, 0,
                                         C.c_void_p(offsets.data_ptr()), C.c_void_p(stream)))

    old()
    torch.cuda.synchronize()
    total = int(offsets[-1])
    out = (torch.empty(b + 1, dtype=torch.int64, device="cuda"), torch.empty(max(total, 1), dtype=torch.int64, device="cuda"),
           torch.empty(max(total, 1), dtype=torch.float32, device="cuda"))

    def new(defer=False):
        base.search_range_device(q, ms, total, out=out, defer_check=defer, expected_hits=0)

    t_old = device_ms(old, reps)
    t_new = device_ms(new, reps)
    # one deferred call: what the host spends before it can queue more work
    new(True)
    base.finish_search()
    torch.cuda.synchronize()
    host = []
    for _ in range(reps):
        t0 = time.perf_counter()
        new(True)
        host.append((time.perf_counter() - t0) * 1e3)
        base.finish_search()
        torch.cuda.synchronize()
    assert torch.equal(out[0], offsets), "the two searches disagree on the offsets"
    return {"queries": b, "min_score": ms, "hits": total, "range_search_device_ms": round(t_old, 3),
            "range_search_into_device_ms": round(t_new, 3), "deferred_call_host_ms": round(statistics.median(host), 3),
            "path": base.last_timing()["path"]}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--big-rows", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json")
    args = ap.parse_args(argv)
    import torch

    import typeagent_py_b200 as tab
    from oracle import vectorbase_oracle as O
    from range_probe import card, unit_rows

    settings = tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel())
    report = {**card(), "results": []}
    t = unit_rows(args.rows, 768, torch.float32, seed=1)
    base = tab.VectorBase.from_device_tensor(settings, t)
    base.enable_timing()
    q = unit_rows(1, 768, torch.float32, seed=2)
    for ms in (0.85, 0.5, 0.0):
        report["results"].append({"shape": f"{args.rows} x 768 float32", **probe(base, q, ms, args.reps)})
    del base, t
    torch.cuda.empty_cache()
    t = unit_rows(args.big_rows, 768, torch.bfloat16, seed=3)
    base = tab.VectorBase.from_device_tensor(settings, t)
    base.enable_timing()
    q = unit_rows(64, 768, torch.float32, seed=4)
    for ms in (0.6, 0.55):  # 0.55: ~28k hits per query, past the default region: every query is re-passed
        report["results"].append({"shape": f"{args.big_rows} x 768 bfloat16", **probe(base, q, ms, args.reps)})
    print(json.dumps(report, indent=1))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
