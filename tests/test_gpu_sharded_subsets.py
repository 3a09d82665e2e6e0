"""Sharded per-query subsets on the GPU, bit for bit on dyadic corpora with identical rows in different row blocks:

(a) W in {1, 2, 3, 8} row blocks of one corpus on one GPU, each a ``CudaShardEngine`` driven through its own
    per-rank steps (``search_subsets_packed``, ``range_local(subsets=)``), the packed buffers stacked as the
    all-gather produces them, merged by flat position (``merge_ordered`` orders 2 / 3, ``merge_range``) and decoded
    through the caller's ordinals (``map_items``): equal to one ``VectorBase`` with ``subsets=`` over the whole corpus;
(b) ``ShardedVectorBase`` with one rank equal to ``VectorBase`` for ``subsets=`` and
    ``fuzzy_lookup_embeddings_in_subsets``, and its argument errors.
"""

from __future__ import annotations

import numpy as np
import pytest

from tests.test_gpu_sharded_filter import (  # noqa: F401  (one_rank_group: a fixture)
    N, assert_same, blocks, corpus, engines_for, one_rank_group, settings, subset_of, whole)

pytestmark = pytest.mark.gpu


def batch_subsets(b, seed):
    """Per query: the filter tests' subset (duplicates across blocks, negatives), cut to different lengths, one
    query inside one block only, and an empty one."""
    out = []
    for i in range(b):
        sub = subset_of(seed + i)
        if i % 4 == 1:
            sub = sub[: 1 + 37 * i]
        elif i % 4 == 2:
            sub = np.arange(N - 700, N, 3)[::-1]
        elif i % 4 == 3 and i > 8:
            sub = np.empty(0, np.int64)
        out.append(sub)
    return out


def csr(subs):
    from typeagent_py_b200.vectorbase import VectorBase

    return VectorBase._subsets_csr(subs, len(subs))


def subsets_topk(engines, n, q, k, ms, subs, ties_low):
    import torch

    from typeagent_py_b200.sharded import subsets_share

    offsets, ordinals = csr(subs)
    parts = []
    for eng, (lo, hi) in zip(engines, blocks(n, len(engines))):
        pos, loff, lord = subsets_share(offsets, ordinals, n, lo, hi)
        parts.append(eng.search_subsets_packed(q, k, ms, loff, lord, pos, ties_low))
    items, scores, counts = engines[0].merge_ordered(torch.stack(parts), len(engines), len(q), k, 3 if ties_low else 2)
    engines[0].map_items(items, ordinals)
    return items.cpu().numpy(), scores.cpu().numpy(), counts.cpu().numpy()


def subsets_range(engines, n, q, ms, subs, ties_low):
    import torch

    from typeagent_py_b200.sharded import offsets_with_status, pack_range_payload, range_pad, subsets_share

    offsets, ordinals = csr(subs)
    locals_ = []
    for eng, (lo, hi) in zip(engines, blocks(n, len(engines))):
        pos, loff, lord = subsets_share(offsets, ordinals, n, lo, hi)
        locals_.append(eng.range_local(q, ms, lo, ties_low, subsets=(loff, lord), positions=pos))
    dev = engines[0].comm_device()
    offsets_all = torch.from_numpy(np.stack([offsets_with_status(loc.offsets, False) for loc in locals_])).to(dev)
    totals = [int(loc.offsets[-1]) for loc in locals_]
    t_pad = max(range_pad(totals), 2)
    payload = torch.stack([pack_range_payload(loc, t_pad, dev) for loc in locals_])
    o, i, s = engines[0].merge_range(offsets_all, payload, len(engines), len(q), t_pad, sum(totals), ties_low)
    engines[0].map_items(i, ordinals)
    return o.cpu().numpy(), i.cpu().numpy(), s.cpu().numpy()


# ---------------------------------------------------------------- (a) per-rank steps, W blocks on one GPU
@pytest.mark.parametrize("w", [1, 2, 3, 8])
@pytest.mark.parametrize("storage", ["float32", "bfloat16"])
def test_subsets_equal_whole_corpus(w, storage):
    v, q = corpus(12, seed=31)
    subs = batch_subsets(len(q), seed=5)
    one = whole(v, storage)
    engines = engines_for(v, w, storage)
    longest = max(len(s) for s in subs)
    for ms in (0.0, 0.6):
        for tl in (False, True):
            for k in (1, 10, 100):
                want = one.search_arrays(q, k, ms, subsets=subs, ties_low_first=tl)
                got = subsets_topk(engines, N, q, min(k, longest), ms, subs, tl)
                assert_same(got, want, f"W={w} {storage} top-k ms={ms} tl={tl} k={k}")
            assert_same(subsets_range(engines, N, q, ms, subs, tl), one.search_range(q, ms, subsets=subs,
                                                                                    ties_low_first=tl),
                        f"W={w} {storage} range ms={ms} tl={tl}")


# ---------------------------------------------------------------- (b) one rank of ShardedVectorBase
@pytest.mark.parametrize("storage", ["float32", "bfloat16"])
def test_sharded_one_rank_equals_vectorbase(one_rank_group, storage):
    from typeagent_py_b200.sharded import ShardedVectorBase

    v, q = corpus(12, seed=43)
    subs = batch_subsets(len(q), seed=9)
    one = whole(v, storage)
    sh = ShardedVectorBase(settings(), device=0, storage_dtype=storage)
    sh.deserialize(v)
    longest = max(len(s) for s in subs)
    for ms in (0.0, 0.6, float("nan")):
        for tl in (False, True):
            for k in (10, 100, 2049, longest):  # above 2048: the threshold exchange, cut to k
                assert_same(sh.search_arrays(q, k, ms, subsets=subs, ties_low_first=tl),
                            one.search_arrays(q, k, ms, subsets=subs, ties_low_first=tl), f"top-k {ms} {tl} {k}")
            assert_same(sh.search_range(q, ms, ties_low_first=tl, subsets=subs),
                        one.search_range(q, ms, subsets=subs, ties_low_first=tl), f"range {ms} {tl}")
    lists = [s.tolist() for s in subs]
    for mh in (None, 5, 0):
        got = sh.fuzzy_lookup_embeddings_in_subsets(q, lists, mh, 0.6)
        want = one.fuzzy_lookup_embeddings_in_subsets(q, lists, mh, 0.6)
        assert [[(h.item, h.score) for h in r] for r in got] == [[(h.item, h.score) for h in r] for r in want], mh
    for call, exc in [(lambda: sh.search_arrays(q, 5, subsets=subs[:3]), ValueError),
                      (lambda: sh.search_range(q, 0.0, subsets=subs, subset=[1]), ValueError),
                      (lambda: sh.search_arrays(q, 5, subsets=[[N]] + lists[1:]), IndexError),
                      (lambda: sh.search_range(q, 0.0, subsets=[[0.5]] + lists[1:]), IndexError)]:
        with pytest.raises(exc):
            call()
