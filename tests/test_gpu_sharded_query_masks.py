"""Per-query masks across row blocks, on one GPU, bit for bit against one ``VectorBase`` over the whole corpus:
W = 1, 2, 3 and 8 blocks driven through ``CudaShardEngine``'s per-rank steps (each block's columns of every
query's mask, cut by ``block_mask``, then the ordered merge or ``tav_merge_range``), and one rank of
``ShardedVectorBase``.  The corpus has identical rows in different blocks (tests/test_gpu_sharded_filter.py)."""

from __future__ import annotations

import numpy as np
import pytest

from tests.test_gpu_sharded_filter import (N, assert_same, blocks, corpus, engines_for, masked_topk,  # noqa: F401
                                           one_rank_group, settings, whole)

pytestmark = pytest.mark.gpu


def query_masks(b, seed):
    rng = np.random.default_rng(seed)
    dens = [0.45, 0.05, 1.0, 0.002, 0.3]
    m = np.stack([rng.random(N) < dens[i % len(dens)] for i in range(b)])
    m[::2, :600] = True          # rows whose copies sit in later blocks: equal scores across blocks
    m[::2, 1500:2100] = True
    return m


def masked_range(engines, n, q, ms, masks, ties_low):
    import torch

    from typeagent_py_b200.sharded import block_mask, offsets_with_status, pack_range_payload, range_pad

    locals_ = [eng.range_local(q, ms, lo, ties_low, mask=block_mask(masks, n, lo, hi, len(q)))
               for eng, (lo, hi) in zip(engines, blocks(n, len(engines)))]
    dev = engines[0].comm_device()
    offsets_all = torch.from_numpy(np.stack([offsets_with_status(loc.offsets, False) for loc in locals_])).to(dev)
    totals = [int(loc.offsets[-1]) for loc in locals_]
    t_pad = max(range_pad(totals), 2)
    payload = torch.stack([pack_range_payload(loc, t_pad, dev) for loc in locals_])
    o, i, s = engines[0].merge_range(offsets_all, payload, len(engines), len(q), t_pad, sum(totals), ties_low)
    return o.cpu().numpy(), i.cpu().numpy(), s.cpu().numpy()


@pytest.mark.parametrize("w,storage,b,k", [(1, "float32", 4, 50), (2, "bfloat16", 20, 100), (3, "float16", 5, 64),
                                           (8, "float32", 6, 300), (3, "bfloat16", 17, 10), (2, "float32", 1, 20)])
@pytest.mark.parametrize("ties_low", [False, True], ids=["ties_high", "ties_low"])
def test_per_query_masks_across_blocks_equal_whole_corpus(w, storage, b, k, ties_low):
    v, q = corpus(b, seed=5 * w + b)
    masks = query_masks(b, seed=w + k)
    one = whole(v, storage)
    engines = engines_for(v, w, storage)
    for ms in (0.0, 0.6):
        want = one.search_arrays(q, k, ms, allowed=masks, ties_low_first=ties_low)
        assert_same(masked_topk(engines, N, q, k, ms, masks, ties_low), want, f"W={w} {storage} ms={ms}")
        assert_same(masked_range(engines, N, q, ms, masks, ties_low),
                    one.search_range(q, ms, allowed=masks, ties_low_first=ties_low), f"W={w} {storage} range ms={ms}")


def test_one_rank_of_sharded_vectorbase_equals_vectorbase(one_rank_group):
    from typeagent_py_b200 import VectorBase
    from typeagent_py_b200.sharded import ShardedVectorBase

    v, q = corpus(12, seed=3)
    masks = query_masks(len(q), seed=4)
    words = VectorBase.pack_query_masks(masks)
    sh = ShardedVectorBase(settings(), device=0, storage_dtype="bfloat16")
    sh.deserialize(v)
    one = whole(v, "bfloat16")
    for mask in (masks, words):
        for tl in (False, True):
            assert_same(sh.search_arrays(q, 40, 0.0, allowed=mask, ties_low_first=tl),
                        one.search_arrays(q, 40, 0.0, allowed=masks, ties_low_first=tl), f"rank 0 {mask.dtype} {tl}")
            assert_same(sh.search_range(q, 0.55, allowed=mask, ties_low_first=tl),
                        one.search_range(q, 0.55, allowed=masks, ties_low_first=tl), f"rank 0 range {mask.dtype} {tl}")
    with pytest.raises(ValueError, match="rows for 12 queries"):
        sh.search_arrays(q, 5, 0.0, allowed=masks[:3])
