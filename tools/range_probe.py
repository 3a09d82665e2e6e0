"""Threshold-search probe: what ``max_hits=0`` lookups and ``search_range`` cost on the GPU, next to the
paged top-k form they replace and the reference's numpy lookup.

    python tools/range_probe.py [--rows 1000000] [--big-rows 10000000] [--reps 5] [--json OUT]

Reports, in one run: the card's name and power limit; device time of ``fuzzy_lookup_embedding(max_hits=0)``
at rows x 768 float32 with min_score 0.85 / 0.5 / 0.0; ``search_range`` with 64 queries at big-rows x 768
bfloat16, min_score 0.6; hits per second; the scoring scans' bytes over their time against the 3.35 TB/s
data-sheet HBM3 bandwidth; the unmodified reference's CPU time for the float32 case (when its modules are
importable: ``oracle/_ref`` made by ``build()``); and the old cost as one paged pass (scan + select, k = 2048)
times the number of passes the paged form needs.  Rows are unit-norm Gaussian, seeded.  Writes nothing
unless ``--json`` is given.  Anything not measured is reported as "not measured".
"""

from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_TBPS = 3.35     # H100 SXM data sheet
PASS_K = 2048       # hits per paged pass (TAV_PASS_K)
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


def unit_rows(n, d, dtype, seed):
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    out = torch.empty((n, d), dtype=dtype, device="cuda")
    step = 1 << 20
    for lo in range(0, n, step):  # float32 work buffer a block at a time
        x = torch.randn((min(step, n - lo), d), generator=g, device="cuda")
        out[lo:lo + len(x)] = (x / x.norm(dim=1, keepdim=True)).to(dtype)
    return out


def timed(base, fn, reps):
    """Median over reps of (device first-launch-to-last-byte ms, main kernels ms, main kernels run), after a warm-up."""
    fn()
    rows = []
    for _ in range(reps):
        fn()
        t = base.last_timing()
        mains = [ms for name, ms in t["kernels"] if name == "main"]
        rows.append((t["total_ms"], t["scan_ms"], len(mains)))
    rows.sort()
    return rows[len(rows) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--big-rows", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    ap.add_argument("--no-reference", action="store_true")
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("range_probe needs a CUDA device (no CPU fallback)")
    import typeagent_py_b200 as tab
    from oracle import vectorbase_oracle as O

    report = card()
    settings = tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel())
    n, d = args.rows, args.dim

    # ---- fuzzy_lookup_embedding(max_hits=0), n x d float32
    rows = unit_rows(n, d, torch.float32, seed=1)
    q = unit_rows(1, d, torch.float32, seed=2)
    q = (0.5 * q + 0.5 * rows[12345:12346]).float()  # a query with neighbours
    q = (q / q.norm()).cpu().numpy()[0]
    base = tab.VectorBase.from_device_tensor(settings, rows)
    base.enable_timing()
    single = []
    for ms in (0.85, 0.5, 0.0):
        hits = len(base.fuzzy_lookup_embedding(q, max_hits=0, min_score=ms))
        total, scan, mains = timed(base, lambda: base.fuzzy_lookup_embedding(q, max_hits=0, min_score=ms), args.reps)
        t0 = time.perf_counter()
        base.fuzzy_lookup_embedding(q, max_hits=0, min_score=ms)
        wall = (time.perf_counter() - t0) * 1e3
        scan_bytes = mains * n * d * 4
        single.append({"min_score": ms, "hits": hits, "device_ms": total, "wall_ms": wall, "scans": mains,
                       "scan_ms": scan, "scan_TBps": scan_bytes / (scan * 1e-3) / 1e12,
                       "scan_share_of_3.35TBps": scan_bytes / (scan * 1e-3) / 1e12 / HBM_TBPS,
                       "hits_per_s": hits / (total * 1e-3)})
    # old cost: one paged pass (scan + select at k = 2048) times the passes of k = n
    base.force_path = "scan"
    total, scan, _ = timed(base, lambda: base.search_arrays(q[None], PASS_K, 0.0), args.reps)
    passes = math.ceil(n / PASS_K)
    paged = {"one_pass_device_ms": total, "passes": passes, "estimated_ms": total * passes}
    report["lookup_max_hits_0_f32"] = {"rows": n, "dim": d, "results": single, "paged_form": paged}

    # the unmodified reference on the same rows (numpy on this host's CPU)
    ref = {"cpu_ms": NOT_MEASURED}
    if not args.no_reference:
        try:
            from oracle.ref_loader import make_reference_vectorbase, reference_available

            if reference_available():
                host = rows.cpu().numpy()
                rv = make_reference_vectorbase(host)
                per = {}
                for ms in (0.85, 0.5, 0.0):
                    rv.fuzzy_lookup_embedding(q, max_hits=0, min_score=ms)
                    t0 = time.perf_counter()
                    got = rv.fuzzy_lookup_embedding(q, max_hits=0, min_score=ms)
                    per[str(ms)] = {"cpu_ms": (time.perf_counter() - t0) * 1e3, "hits": len(got)}
                ref = {"per_min_score": per, "cpus": os.cpu_count()}
                del host, rv
        except Exception as e:  # a missing reference is reported, not hidden
            ref = {"cpu_ms": NOT_MEASURED, "why": repr(e)}
    report["reference_cpu"] = ref
    del base, rows
    torch.cuda.empty_cache()

    # ---- search_range, 64 queries, big x d bfloat16
    nb = args.big_rows
    try:
        big = unit_rows(nb, d, torch.bfloat16, seed=3)
        qb = unit_rows(64, d, torch.float32, seed=4)
        qb = 0.6 * qb + 0.4 * big[:64 * 997:997].float()  # queries with neighbours above 0.6
        qb = (qb / qb.norm(dim=1, keepdim=True)).cpu().numpy()
        vb = tab.VectorBase.from_device_tensor(settings, big)
        vb.enable_timing()
        offsets = vb.search_range(qb, 0.6)[0]
        total, scan, mains = timed(vb, lambda: vb.search_range(qb, 0.6), args.reps)
        hits = int(offsets[-1])
        scan_bytes = mains * nb * d * 2
        vb.force_path = "scan"  # the paged form of k = rows runs on the row scan
        one_pass, _, _ = timed(vb, lambda: vb.search_arrays(qb, PASS_K, 0.6), args.reps)
        passes = math.ceil(nb / PASS_K)
        report["search_range_bf16_B64"] = {
            "rows": nb, "dim": d, "queries": 64, "min_score": 0.6, "hits": hits, "device_ms": total,
            "scans": mains, "scan_ms": scan, "scan_TBps": scan_bytes / (scan * 1e-3) / 1e12,
            "scan_share_of_3.35TBps": scan_bytes / (scan * 1e-3) / 1e12 / HBM_TBPS,
            "hits_per_s": hits / (total * 1e-3),
            "paged_form": {"one_pass_device_ms": one_pass, "passes": passes, "estimated_ms": one_pass * passes}}
        del vb, big
    except torch.cuda.OutOfMemoryError as e:
        report["search_range_bf16_B64"] = {"device_ms": NOT_MEASURED, "why": repr(e)}
    line = json.dumps(report)
    print(line)
    if args.json:
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
