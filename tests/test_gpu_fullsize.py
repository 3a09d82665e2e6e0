"""Parity at BASELINE.json's full single-GPU sizes (configs 2, 3, one shard of config 4 with its
real batch of 1024, config 5):

  * ORACLE-anchored: the device corpus is read back in 1M-row float32 blocks and the numpy oracle
    (the reference's np.dot / clip / flatnonzero / argpartition, tests/parity.blocked_oracle_lookup)
    ranks a handful of the batch's queries — including a planted one — at the contract tolerances
    (scores 1e-4, ties 2e-6; aitools/vectorbase.py:163-190, tools/benchmark_vectorbase.py:80-94);
  * two independent CUDA paths agree: the tensor-core kernel vs the exact row-scan kernel, on the
    same device-resident corpus, for a handful of the batch's queries (identical index sets up
    to float32 summation-order ties, scores within 2e-6);
  * planted rows: exact copies of some queries overwrite known rows and must come back first
    with score 1.0 (bf16-representable unit vectors: the dot is within 1 ulp-ish of 1);
  * structure: full counts, scores descending, ordinals in range and unique;
  * decomposition: top-k over the whole corpus == merge of top-k over two halves (the sharded
    path's merge kernel), bit for bit.

These checks run on random data, with tolerances, for a handful of queries.  Every query of every batch
at these sizes is compared bit for bit in tests/test_gpu_scale_exact.py, on exact-arithmetic corpora.
"""

from __future__ import annotations

import numpy as np
import pytest

import typeagent_py_b200 as tab
from bench import make_shard_on_device
from tests.parity import assert_hits_match, blocked_oracle_lookup

pytestmark = pytest.mark.gpu


class _Null:
    model_name = "fullsize"

    def add_embedding(self, key, e):
        pass


@pytest.mark.parametrize("rows,dim,storage,batch,k", [
    (1_000_000, 768, "bfloat16", 64, 32),      # BASELINE configs[1]
    (10_000_000, 768, "bfloat16", 256, 100),   # BASELINE configs[2] (the bench workload)
    (1_250_000, 1536, "float16", 1024, 100),   # one shard of configs[3], with its real batch (8 query chunks of 128)
    (50_000, 384, "bfloat16", 1000, 5),        # BASELINE configs[4]
])
def test_full_size_properties(rows, dim, storage, batch, k):
    import torch

    from typeagent_py_b200.sharded import CudaShardEngine, packed_layout

    dev = torch.device("cuda", 0)
    corpus = make_shard_on_device(torch, dev, 0, rows, dim, storage, seed=99)
    gen = torch.Generator(device=dev).manual_seed(5)
    q = torch.randn((batch, dim), generator=gen, device=dev, dtype=torch.float32)
    q /= q.norm(dim=1, keepdim=True)
    q = q.to(corpus.dtype).to(torch.float32)           # storage-representable queries
    q /= 1.0                                            # (kept un-renormalised: reference semantics = plain dot)
    planted = {3: 17, 7: rows - 1, 11: rows // 2}       # query index -> row
    for qi, row in planted.items():
        corpus[row] = q[qi].to(corpus.dtype)
    torch.cuda.synchronize()

    settings = tab.TextEmbeddingIndexSettings(_Null())
    base = tab.VectorBase.from_device_tensor(settings, corpus)
    base.force_path = "mma"
    items, scores, counts = base.search_device(q, k, 0.0)
    torch.cuda.synchronize()
    assert base.last_timing()["path"] == "mma"
    items_h, scores_h, counts_h = items.cpu().numpy(), scores.cpu().numpy(), counts.cpu().numpy()

    # structure
    assert (counts_h == k).all()
    assert (np.diff(scores_h, axis=1) <= 0).all()
    assert items_h.min() >= 0 and items_h.max() < rows
    assert all(len(set(r)) == k for r in items_h)
    assert scores_h.max() <= 1.0 and scores_h.min() >= 0.0

    # planted rows come back first, score ~ clip((|q|^2 + 1) / 2); fp32 accumulation of `dim`
    # positive products in the tensor core is good to a few 1e-6 at dim 1536
    for qi, row in planted.items():
        assert items_h[qi, 0] == row
        want = min(1.0, (float((q[qi].double() * q[qi].double()).sum()) + 1.0) / 2.0)
        assert abs(scores_h[qi, 0] - want) < 1e-5

    # the oracle, blocked over the device corpus: contract tolerances (scores 1e-4, ties 2e-6)
    pick = [0, 3, 7, batch // 2, batch - 1]
    q_np = q[pick].cpu().numpy()
    for j, want in enumerate(blocked_oracle_lookup(corpus, q_np, k, 0.0)):
        qi = pick[j]
        assert_hits_match({"items": items_h[qi].tolist(), "scores": scores_h[qi].tolist()}, want,
                          score_tol=1e-4, tie_tol=2e-6, what=f"mma vs blocked oracle q{qi}")

    # independent path: exact row scan for a few queries
    base.force_path = "scan"
    s_items, s_scores, s_counts = base.search_device(q[pick].contiguous(), k, 0.0)
    torch.cuda.synchronize()
    assert base.last_timing()["path"] == "scan"
    for j, qi in enumerate(pick):
        assert_hits_match({"items": items_h[qi].tolist(), "scores": scores_h[qi].tolist()},
                          {"items": s_items[j].tolist(), "scores": s_scores[j].tolist()},
                          score_tol=1e-5, tie_tol=2e-6, what=f"mma vs scan q{qi}")

    # decomposition: merge of two halves == whole, bit for bit
    half = rows // 2
    parts = []
    for lo, hi in ((0, half), (half, rows)):
        eng = CudaShardEngine(settings, 0, storage)
        eng.adopt_tensor(corpus[lo:hi])
        eng.base.force_path = "mma"
        parts.append(eng.search_packed(q, k, 0.0, lo))
    gathered = torch.stack(parts)
    assert gathered.shape[1] == packed_layout(batch, k)[2]
    m_items, m_scores, m_counts = eng.merge(gathered, 2, batch, k)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(m_counts.cpu().numpy(), counts_h)
    np.testing.assert_array_equal(m_items.cpu().numpy(), items_h)
    np.testing.assert_array_equal(m_scores.cpu().numpy(), scores_h)
    del corpus
    torch.cuda.empty_cache()
