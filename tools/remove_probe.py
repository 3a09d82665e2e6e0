"""Row-removal probe: what ``tav_remove_rows`` and ``tav_write_rows`` cost on the GPU, next to the
clear-and-re-append route they replace.

    python tools/remove_probe.py [--rows 10000000] [--dim 768] [--reps 3] [--json OUT]

On a rows x dim bfloat16 index built by device appends (capacity = rows), times with CUDA events on the call's
stream, each case from a freshly refilled index:
  * removal of 1 row near the start (row 10: every later row moves), in place (the default: 256 MB windows)
    and forced out of place (a second allocation of the rows);
  * removal of 1% and of 50% of the rows, at random;
  * removal of rows [10, 20) and [1000, rows / 2): a long run of removed rows that begins inside a warp's
    destinations (the compaction gallops over its equal keys);
  * an overwrite of 1M rows from device bfloat16 rows (a plain copy) and from host float32 rows (PCIe, then
    the conversion kernel);
  * the route a removal needed before: tav_clear, then the surviving rows appended again from host float32
    memory (what ``VectorBase`` re-uploads after a ``deserialize``), timed for the 1% removal.
Reports the card's name and power limit, the milliseconds (median over reps), the bytes the device moves and
those bytes over the time against the 3.35 TB/s data-sheet HBM3 bandwidth.  Writes nothing unless ``--json`` is
given.
"""

from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_TBPS = 3.35  # H100 SXM data sheet
NOT_MEASURED = "not measured"


def card():
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20)
        power = out.stdout.strip() or NOT_MEASURED
    except (OSError, subprocess.SubprocessError):
        power = NOT_MEASURED
    return {"card": name, "power_limit": power}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch

    from typeagent_py_b200 import _capi

    lib = _capi.load()
    policy = lib.tav_internal_compact_policy
    policy.argtypes, policy.restype = [C.c_void_p, C.c_int, C.c_int64], C.c_int
    stats = lib.tav_internal_compact_stats
    stats.argtypes, stats.restype = [C.c_void_p, C.c_void_p, C.c_void_p], C.c_int

    n, d = args.rows, args.dim
    row = 2 * d
    stream = torch.cuda.Stream()
    sp = C.c_void_p(stream.cuda_stream)
    g = torch.Generator(device="cuda").manual_seed(0)
    source = torch.empty((n, d), dtype=torch.bfloat16, device="cuda")
    for lo in range(0, n, 1 << 20):
        source[lo:lo + (1 << 20)] = torch.randn((min(1 << 20, n - lo), d), generator=g, device="cuda").to(torch.bfloat16)
    h = C.c_void_p()
    _capi.check(lib.tav_create(0, d, _capi.TAV_BF16, 0, n, C.byref(h)))

    def refill():
        _capi.check(lib.tav_clear(h))
        _capi.check(lib.tav_append(h, C.c_void_p(source.data_ptr()), n, d, _capi.TAV_BF16, 1, sp))
        stream.synchronize()

    def timed(prepare, call):
        """Median ms over reps (after one warm-up) of `call`, events recorded on the call's stream."""
        times = []
        for _ in range(args.reps + 1):
            prepare()
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record(stream)
            call()
            end.record(stream)
            end.synchronize()
            times.append(start.elapsed_time(end))
        return statistics.median(times[1:])

    rng = np.random.default_rng(1)
    cases = []

    def removal(name, ordinals, mode=0):
        ordinals = np.ascontiguousarray(np.sort(ordinals), np.int64)
        _capi.check(policy(h, mode, 0))
        ms = timed(refill, lambda: _capi.check(lib.tav_remove_rows(h, ordinals.ctypes.data_as(C.c_void_p),
                                                                      len(ordinals), sp)))
        path, windows = C.c_int(0), C.c_int64(0)
        _capi.check(stats(h, C.byref(path), C.byref(windows)))
        first, m = int(ordinals[0]), len(ordinals)
        moving = n - m - first
        rows_moved = moving if path.value == 2 else first + moving  # out of place also copies the prefix
        trips = 4 if path.value == 2 else 2  # in place: read, scratch write, scratch read, write
        moved = trips * rows_moved * row + 8 * m
        cases.append({"case": name, "path": {0: "none", 1: "out of place", 2: "in place"}[path.value],
                      "windows": windows.value, "ms": ms, "bytes_moved": moved,
                      "tb_per_s": moved / ms / 1e9, "of_hbm_peak": moved / ms / 1e9 / HBM_TBPS})

    removal("remove 1 row at 10 (in place, 256 MB windows)", np.array([10]))
    removal("remove 1 row at 10 (out of place)", np.array([10]), mode=1)
    removal("remove 1% at random, out of place", rng.choice(n, n // 100, replace=False), mode=1)
    removal("remove 1% at random", rng.choice(n, n // 100, replace=False))
    removal("remove 50% at random", rng.choice(n, n // 2, replace=False))
    removal("remove [10, 20) and [1000, rows / 2)", np.concatenate([np.arange(10, 20), np.arange(1000, n // 2)]))

    # overwrite of 1M rows
    m = min(1_000_000, n)
    first = n // 3
    refill()
    dev_rows = source[:m].clone()
    ms = timed(lambda: None, lambda: _capi.check(lib.tav_write_rows(h, first, C.c_void_p(dev_rows.data_ptr()), m, d,
                                                                    _capi.TAV_BF16, 1, sp)))
    moved = 2 * m * row
    cases.append({"case": "overwrite 1M rows from device bf16", "ms": ms, "bytes_moved": moved,
                  "tb_per_s": moved / ms / 1e9, "of_hbm_peak": moved / ms / 1e9 / HBM_TBPS})
    host_rows = np.ascontiguousarray(source[:m].float().cpu().numpy())
    ms = timed(lambda: None, lambda: _capi.check(lib.tav_write_rows(h, first, host_rows.ctypes.data_as(C.c_void_p), m, d,
                                                                    _capi.TAV_F32, 0, sp)))
    cases.append({"case": "overwrite 1M rows from host float32", "ms": ms, "host_bytes": host_rows.nbytes,
                  "host_gb_per_s": host_rows.nbytes / ms / 1e6})

    # the route it replaces: clear, then the surviving rows again from host float32 memory.  The host holds one
    # block of 1M rows, appended as often as the survivors need: the same bytes cross PCIe.
    survivors = n - n // 100

    def reupload():
        _capi.check(lib.tav_clear(h))
        for lo in range(0, survivors, m):
            k = min(m, survivors - lo)
            _capi.check(lib.tav_append(h, host_rows.ctypes.data_as(C.c_void_p), k, d, _capi.TAV_F32, 0, sp))

    ms = timed(lambda: None, reupload)
    cases.append({"case": "clear and re-append the survivors of a 1% removal from host float32", "ms": ms,
                  "host_bytes": survivors * d * 4, "host_gb_per_s": survivors * d * 4 / ms / 1e6})

    lib.tav_destroy(h)
    result = {**card(), "rows": n, "dim": d, "storage": "bfloat16", "reps": args.reps, "cases": cases}
    for c in cases:
        print(json.dumps(c))
    print(json.dumps({k: v for k, v in result.items() if k != "cases"}))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
