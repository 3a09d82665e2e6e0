#!/usr/bin/env python3
"""The reference's own micro-benchmark (tools/benchmark_vectorbase.py), pointed at the GPU class.

Same cases, same seeds, same statistic set: 1k x 384 (seed 42), 10k x 384 (seed 43),
fuzzy_lookup_embedding_in_subset over 1 000 of the 10k rows (subset rng seed 99); max_hits=10,
min_score=0.0; 20 warm-up + 200 timed rounds with time.perf_counter_ns; min / mean / median /
max in microseconds.  Each case is run on the GPU VectorBase and — as the CPU comparator, in the
same process on the same box — on the numpy restatement of the reference (oracle/, test
infrastructure).  This is BASELINE.json configs[0]; the L2 stays warm between rounds exactly as
the CPU caches do in the reference's harness.

Usage: python tools/benchmark_vectorbase_gpu.py [--rounds 200] [--warmup-rounds 20] [--dim 384]
"""

from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time
from types import SimpleNamespace

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import typeagent_py_b200 as tab  # noqa: E402
from oracle import vectorbase_oracle as O  # noqa: E402


class NullModel:
    model_name = "benchmark-local"

    def add_embedding(self, key, embedding):
        return None


def make_pair(count: int, dim: int, seed: int):
    vectors, queries = O.make_corpus(count, dim, seed)  # same construction as the reference's make_vectorbase
    gpu = tab.VectorBase(tab.TextEmbeddingIndexSettings(embedding_model=NullModel()))
    gpu.add_embeddings(None, vectors)
    cpu = O.OracleVectorBase(SimpleNamespace(embedding_model=NullModel(), min_score=0.85, max_matches=None))
    cpu.add_embeddings(None, vectors)
    return gpu, cpu, queries[0]


def run(target, rounds: int, warmup: int) -> list[float]:
    for _ in range(warmup):
        target()
    out = []
    for _ in range(rounds):
        t0 = time.perf_counter_ns()
        target()
        out.append((time.perf_counter_ns() - t0) / 1_000)
    return out


def report(label: str, samples: list[float]) -> dict:
    stats = {"min": min(samples), "mean": statistics.fmean(samples), "median": statistics.median(samples),
             "max": max(samples)}
    print(f"{label}\n" + "".join(f"  {k + ':':8s}{v:9.3f} us\n" for k, v in stats.items()), end="")
    return stats


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=200)
    ap.add_argument("--warmup-rounds", type=int, default=20)
    ap.add_argument("--dim", type=int, default=384)
    ap.add_argument("--subset-size", type=int, default=1_000)
    ap.add_argument("--json", default=None, help="also write the statistics to this file")
    args = ap.parse_args()

    gpu_1k, cpu_1k, q_1k = make_pair(1_000, args.dim, 42)
    gpu_10k, cpu_10k, q_10k = make_pair(10_000, args.dim, 43)
    subset = np.random.default_rng(99).choice(10_000, size=args.subset_size, replace=False).tolist()
    cases = [
        ("fuzzy_lookup_embedding (1k vectors)",
         lambda b, q=q_1k: b.fuzzy_lookup_embedding(q, max_hits=10, min_score=0.0), gpu_1k, cpu_1k),
        ("fuzzy_lookup_embedding (10k vectors)",
         lambda b, q=q_10k: b.fuzzy_lookup_embedding(q, max_hits=10, min_score=0.0), gpu_10k, cpu_10k),
        (f"fuzzy_lookup_embedding_in_subset ({args.subset_size} of 10k)",
         lambda b, q=q_10k: b.fuzzy_lookup_embedding_in_subset(q, subset, max_hits=10, min_score=0.0),
         gpu_10k, cpu_10k),
    ]
    results = {}
    for label, call, gpu, cpu in cases:
        got, want = call(gpu), call(cpu)
        if len(got) != 10 or [h.item for h in got] != [h.item for h in want]:
            raise SystemExit(f"{label}: GPU and CPU disagree: {got} vs {want}")
        results[label] = {
            "gpu": report(f"[GPU] {label}", run(lambda: call(gpu), args.rounds, args.warmup_rounds)),
            "cpu": report(f"[CPU numpy, {os.cpu_count()} cores] {label}",
                          run(lambda: call(cpu), args.rounds, args.warmup_rounds)),
        }
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"rounds": args.rounds, "warmup": args.warmup_rounds, "dim": args.dim,
                       "cpu_count": os.cpu_count(), "numpy": np.__version__, "cases": results}, f, indent=1)


if __name__ == "__main__":
    main()
