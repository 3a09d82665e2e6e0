#!/usr/bin/env python3
"""Generate the committed golden vectors by running the UNMODIFIED reference.

Run in the build container only (needs /root/reference):

    python tests/golden/make_golden.py

Writes ``golden_cases.json`` and ``golden_episode53.json`` (reference outputs: items + float32 scores as Python
floats, which round-trip exactly through JSON) and ``episode53_excerpt.npy`` (150 of
the 1294 real embedding rows of the reference's Episode-53 test fixture).  Also records
the reference's own known-answer tests as literal cases.
"""

from __future__ import annotations

import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle.ref_loader import make_reference_vectorbase  # noqa: E402
from tests.golden import cases as C  # noqa: E402

EP53_BIN = "/root/reference/tests/testdata/Episode_53_AdrianTchaikovsky_index_embeddings.bin"


def main() -> None:
    full = np.fromfile(EP53_BIN, dtype=np.float32).reshape(-1, 1536)
    assert full.shape == (1294, 1536), full.shape
    np.save(C.EPISODE53_FILE, np.ascontiguousarray(full[C.EPISODE53_ROWS]))

    out: dict = {"numpy": np.__version__, "cases": {}}
    for case in C.CASES:
        vectors, queries = C.build_inputs(case)
        base = make_reference_vectorbase(vectors)
        recorded = []
        for kind, kw in case["lookups"]:
            per_query = []
            for q in queries:
                if kind == "lookup":
                    hits = base.fuzzy_lookup_embedding(q, **kw)
                elif kind == "subset":
                    kw2 = dict(kw)
                    subset = C.build_subset(kw2.pop("subset"))
                    hits = base.fuzzy_lookup_embedding_in_subset(q, subset, **kw2)
                elif kind == "predicate":
                    kw2 = dict(kw)
                    pred = C.PREDICATES[kw2.pop("predicate")]
                    hits = base.fuzzy_lookup_embedding(q, predicate=pred, **kw2)
                else:
                    raise ValueError(kind)
                per_query.append({"items": [h.item for h in hits], "scores": [h.score for h in hits]})
            recorded.append(per_query)
        out["cases"][case["name"]] = recorded
        print(f"{case['name']}: {len(recorded)} lookups x {len(queries)} queries")

    # The reference's own known-answer test (tests/test_vectorbase.py:239-252).
    base = make_reference_vectorbase()
    for row in ([1.0, 0.0], [0.0, 1.0], [-1.0, 0.0]):
        base.add_embedding(None, np.array(row, dtype=np.float32))
    hits = base.fuzzy_lookup_embedding(np.array([1.0, 0.0], dtype=np.float32), max_hits=3, min_score=0.0)
    kat = {"items": [h.item for h in hits], "scores": [h.score for h in hits]}
    assert kat == {"items": [0, 1, 2], "scores": [1.0, 0.5, 0.0]}, kat
    out["known_answer_score_scale"] = kat

    with open(C.EPISODE53_GOLDEN_FILE, "w") as f:
        json.dump(out["cases"].pop("episode53"), f)
    with open(C.GOLDEN_FILE, "w") as f:
        json.dump(out, f)
    print("wrote", C.GOLDEN_FILE, os.path.getsize(C.GOLDEN_FILE), "bytes")


if __name__ == "__main__":
    main()
