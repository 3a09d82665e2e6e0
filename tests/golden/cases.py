"""Golden-case catalogue shared by ``make_golden.py`` (which runs the unmodified
reference over each case, in the build container) and by the tests (which re-create the
identical inputs from seeds and compare the oracle / the CUDA path with the recorded
reference outputs).

Inputs are never stored except the real-data Episode-53 excerpt; everything else is
regenerated from ``numpy.random.default_rng(seed)`` exactly as the reference's own
benchmark does (tools/benchmark_vectorbase.py:80-94).
"""

from __future__ import annotations

import json
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
EPISODE53_FILE = os.path.join(HERE, "episode53_excerpt.npy")
GOLDEN_FILE = os.path.join(HERE, "golden_cases.json")
EPISODE53_GOLDEN_FILE = os.path.join(HERE, "golden_episode53.json")

# rows of tests/testdata/Episode_53_AdrianTchaikovsky_index_embeddings.bin kept in the
# excerpt (kept under 1 MB): the first 100 related-term rows and the first 50 message-chunk rows
# (1188..1237)
EPISODE53_ROWS = list(range(100)) + list(range(1188, 1238))


def load_golden() -> dict:
    """The recorded reference outputs: ``golden_cases.json``, with the Episode-53 case taken from its
    own file, recorded over the excerpt as stored now."""
    with open(GOLDEN_FILE) as f:
        golden = json.load(f)
    with open(EPISODE53_GOLDEN_FILE) as f:
        golden["cases"]["episode53"] = json.load(f)
    return golden


def unit_rows(rng, n, d):
    v = rng.standard_normal((n, d)).astype(np.float32)
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    return v


def _bf16(x):
    bits = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    r = ((bits + 0x7FFF + ((bits >> 16) & 1)) >> 16) << 16
    return (r & 0xFFFFFFFF).astype(np.uint32).view(np.float32).reshape(x.shape)


def synthetic(n, d, seed, nq=1, storage="float32"):
    rng = np.random.default_rng(seed)
    v = unit_rows(rng, n, d)
    q = unit_rows(rng, nq, d)
    if storage == "bfloat16":
        v, q = _bf16(v), _bf16(q)
    elif storage == "float16":
        v = v.astype(np.float16).astype(np.float32)
        q = q.astype(np.float16).astype(np.float32)
    return v, q


def episode53():
    v = np.load(EPISODE53_FILE)
    # queries: a few term rows and a few message rows, slightly perturbed so that the
    # best hit is not a trivial exact duplicate with score 1.0 only
    rng = np.random.default_rng(53)
    picks = [0, 7, 63, 99, 100, 125, 149]
    q = v[picks] + 0.05 * unit_rows(rng, len(picks), v.shape[1])
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    return v, q.astype(np.float32)


def _mod3(i: int) -> bool:
    return i % 3 == 0


PREDICATES = {"mod3": _mod3}


# Each case: name, how to build (vectors, queries), and the lookups to record.
# A lookup is (kind, kwargs): kind in {"lookup", "subset", "predicate"}.
CASES: list[dict] = [
    dict(name="bench_1k", make=("synthetic", dict(n=1000, d=384, seed=42)),
         lookups=[("lookup", dict(max_hits=10, min_score=0.0))]),
    dict(name="bench_10k", make=("synthetic", dict(n=10000, d=384, seed=43)),
         lookups=[("lookup", dict(max_hits=10, min_score=0.0)),
                  ("lookup", dict(max_hits=None, min_score=None)),
                  ("lookup", dict(max_hits=50, min_score=0.55)),
                  ("lookup", dict(max_hits=10, min_score=0.58)),
                  ("lookup", dict(max_hits=100, min_score=0.0)),
                  ("lookup", dict(max_hits=10, min_score=0.99)),
                  ("subset", dict(subset=("choice", 99, 10000, 1000), max_hits=10, min_score=0.0)),
                  ("subset", dict(subset=("choice", 7, 10000, 37), max_hits=50, min_score=0.5)),
                  ("predicate", dict(predicate="mod3", max_hits=10, min_score=0.5)),
                  # max_hits=0 on the predicate path slices [:0]: nothing (the argpartition path returns everything)
                  ("predicate", dict(predicate="mod3", max_hits=0, min_score=0.5))]),
    dict(name="tiny_k_exceeds_n", make=("synthetic", dict(n=7, d=5, seed=5)),
         lookups=[("lookup", dict(max_hits=10, min_score=0.0)),
                  ("lookup", dict(max_hits=3, min_score=0.0)),
                  ("lookup", dict(max_hits=1, min_score=0.0))]),
    dict(name="quirk_k0_returns_all_passing", make=("synthetic", dict(n=50, d=8, seed=8)),
         lookups=[("lookup", dict(max_hits=0, min_score=0.5))]),
    dict(name="odd_dims", make=("synthetic", dict(n=333, d=17, seed=17, nq=3)),
         lookups=[("lookup", dict(max_hits=5, min_score=0.0)),
                  ("subset", dict(subset=("list", [5, 5, 9, 332, 0, 5]), max_hits=4, min_score=0.0))]),
    dict(name="dim_1536_batch", make=("synthetic", dict(n=2000, d=1536, seed=1536, nq=4)),
         lookups=[("lookup", dict(max_hits=32, min_score=0.0))]),
    dict(name="dim_100_unaligned", make=("synthetic", dict(n=4100, d=100, seed=100, nq=2)),
         lookups=[("lookup", dict(max_hits=20, min_score=0.45))]),
    dict(name="bf16_768", make=("synthetic", dict(n=4096, d=768, seed=768, nq=8, storage="bfloat16")),
         lookups=[("lookup", dict(max_hits=32, min_score=0.0))]),
    dict(name="f16_384_terms", make=("synthetic", dict(n=5000, d=384, seed=384, nq=8, storage="float16")),
         lookups=[("lookup", dict(max_hits=5, min_score=0.0)),
                  ("lookup", dict(max_hits=5, min_score=0.56))]),
    dict(name="episode53", make=("episode53", dict()),
         lookups=[("lookup", dict(max_hits=50, min_score=0.85)),
                  ("lookup", dict(max_hits=10, min_score=0.7)),
                  ("lookup", dict(max_hits=25, min_score=0.0)),
                  ("subset", dict(subset=("range", 100, 150), max_hits=25, min_score=0.7))]),
]


def build_inputs(case: dict):
    kind, kw = case["make"]
    if kind == "synthetic":
        return synthetic(**kw)
    if kind == "episode53":
        return episode53()
    raise ValueError(kind)


def build_subset(spec) -> list[int]:
    tag = spec[0]
    if tag == "choice":
        _, seed, n, size = spec
        return np.random.default_rng(seed).choice(n, size=size, replace=False).tolist()
    if tag == "list":
        return list(spec[1])
    if tag == "range":
        return list(range(spec[1], spec[2]))
    raise ValueError(tag)
