#!/usr/bin/env python3
"""Multi-GPU parity check, launched one rank per GPU:

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
        --master-port 29517 tools/multi_gpu_check.py

Every rank builds the same seeded corpus on the host, keeps its own row block on its GPU
(ShardedVectorBase), and checks that the sharded lookup — local search, candidate exchange (libtavec's
peer-memory publish/merge over NVLink, and the NCCL all-gather form), merge kernel — is BIT-IDENTICAL to
the single-GPU lookup over the whole corpus on that rank's GPU, for the float32 row-scan path, the
float32 split form and the bf16 / fp16 tensor-core paths, and agrees with the CPU oracle.  The sharded
threshold search (``search_range``, merged by ``tav_merge_range``) must equal the
single-GPU ``search_range`` bit for bit on every rank: float32 row scan, bf16 tensor cores, float32 split form.
Filtered and subset lookups (row masks, predicates, subsets; top-k and threshold) must equal the single-GPU
``VectorBase`` bit for bit on every rank.  The same filtered, per-query-mask and per-query-subset top-k lookups go
through the peer exchange (``tav_sharded_search`` / ``tav_sharded_search_subset``) with ``exchange="peer"``, also
deferred on the device (``search_tensors(..., defer_check=True)`` and one ``finish()``), and through the NCCL
exchange with ``exchange="nccl"``: both must equal the single-GPU lookup.  Threshold searches (plain, every row,
row and per-query masks, subsets, per-query subsets) through the peer exchange's range inbox and through the process
group must equal the single-GPU ``search_range``.  These peer-exchange cases, top-k and threshold, have not been run
on two or more GPUs.
"""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import typeagent_py_b200 as tab  # noqa: E402
from oracle import vectorbase_oracle as O  # noqa: E402
from tests.parity import assert_hits_match  # noqa: E402
from typeagent_py_b200.sharded import ShardedVectorBase  # noqa: E402


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    settings = tab.TextEmbeddingIndexSettings(O.FakeEmbeddingModel())
    cases = (("float32", 30011, 96, 7, 25, 0.45), ("bfloat16", 200003, 256, 200, 100, 0.0),
             ("float16", 70001, 128, 33, 10, 0.5), ("float32", 90001, 128, 40, 20, 0.0),
             ("bfloat16", 120000, 64, 300, 5, 0.0), ("float16", 150000, 128, 1024 + 5, 100, 0.0))
    for ci, (storage, n, d, b, k, ms) in enumerate(cases):
        exchange = "nccl" if ci == 2 else "peer"
        v, q = O.make_corpus(n, d, seed=n, n_queries=b)
        vr, qr = O.round_to_storage(v, storage), O.round_to_storage(q, storage)
        sh = ShardedVectorBase(settings, device=local, storage_dtype=storage, exchange=exchange)
        sh.deserialize(v)
        whole = tab.VectorBase(settings, device=local, storage_dtype=storage)
        whole.add_embeddings(None, v)
        got = sh.search_arrays(qr, k, ms)
        want = whole.search_arrays(qr, k, ms)
        assert sh._engine.base.last_timing()["path"] == whole.last_timing()["path"]
        np.testing.assert_array_equal(got[2], want[2])
        for i in range(b):
            c = want[2][i]
            np.testing.assert_array_equal(got[0][i, :c], want[0][i, :c])
            np.testing.assert_array_equal(got[1][i, :c], want[1][i, :c])
        for i in range(min(b, 5)):
            assert_hits_match({"items": got[0][i, : got[2][i]].tolist(), "scores": got[1][i, : got[2][i]].tolist()},
                              O.lookup(vr, qr[i], k, ms), min_score=ms)
        # pipelined: several deferred searches (different queries each), one finish
        qd = [torch.from_numpy(np.ascontiguousarray(np.roll(qr, j, axis=0))).cuda() for j in range(3)]
        outs = [sh.search_tensors(x, k, ms, defer_check=True) for x in qd]
        assert sh.finish() == 0
        torch.cuda.synchronize()
        for j, (it, sc, ct) in enumerate(outs):
            np.testing.assert_array_equal(np.roll(ct.cpu().numpy(), -j, axis=0), want[2])
            np.testing.assert_array_equal(np.roll(it.cpu().numpy(), -j, axis=0)[:, :1], want[0][:, :1])
        # append goes to the last rank and is found globally
        sh.add_embeddings(None, qr[:3])
        hit = sh.fuzzy_lookup_embedding(qr[1], 1, 0.0)[0]
        assert hit.item == n + 1, hit
        dist.barrier()
        if rank == 0:
            print(f"multi-gpu ok: world={world} {storage} n={n} d={d} b={b} k={k} path={whole.last_timing()['path']} "
                  f"exchange={exchange}", flush=True)
    # pathological scores (all rows identical): every rank's tensor-core search flags its queries,
    # finish() redoes them exactly and repeats the exchange
    row = O.round_to_bfloat16(O.make_corpus(1, 64, seed=9)[0])
    same = np.repeat(row, 20000 * world, axis=0)
    for exchange in ("peer", "nccl"):
        sh = ShardedVectorBase(settings, device=local, storage_dtype="bfloat16", exchange=exchange)
        sh.deserialize(same)
        nq = 16   # enough queries for the tensor-core path (fewer go to the exact row scan directly)
        items, scores, counts = sh.search_arrays(np.repeat(row, nq, axis=0), 6, 0.0)
        n = len(same)
        assert sh._engine.base.last_timing()["path"] == "mma"
        assert items.tolist() == [list(range(n - 1, n - 7, -1))] * nq, items
        # three deferred searches of the same pathological corpus, ONE finish: every one of them is repaired
        qd = torch.from_numpy(np.repeat(row, nq, axis=0)).cuda()
        ks = (6, 4, 9)
        outs = [sh.search_tensors(qd, kk, 0.0, defer_check=True) for kk in ks]
        assert sh.finish() > 0
        torch.cuda.synchronize()
        for kk, (it, sc, ct) in zip(ks, outs):
            assert ct.cpu().tolist() == [kk] * nq, ct
            assert it.cpu().tolist() == [list(range(n - 1, n - 1 - kk, -1))] * nq, (kk, it)
        if rank == 0:
            print(f"multi-gpu ok: world={world} exact fallback through finish(), one and three outstanding, "
                  f"exchange={exchange}", flush=True)
    # threshold search (search_range, merged by tav_merge_range): bit-identical to the single-GPU
    # search_range over the whole corpus, at sizes where every rank takes the same path as the whole-corpus search
    for storage, n, d, b, ms, path in (("float32", 70001, 96, 5, 0.55, "scan"),
                                       ("bfloat16", 160001, 128, 32, 0.6, "mma"),
                                       ("float32", 90001, 64, 20, 0.58, "mma_split")):
        v, q = O.make_corpus(n, d, seed=n + 1, n_queries=b)
        sh = ShardedVectorBase(settings, device=local, storage_dtype=storage)
        sh.deserialize(v)
        whole = tab.VectorBase(settings, device=local, storage_dtype=storage)
        whole.add_embeddings(None, v)
        got = sh.search_range(q, ms)
        want = whole.search_range(q, ms)
        assert whole.last_timing()["path"] == path and sh._engine.base.last_timing()["path"] == path
        np.testing.assert_array_equal(got[0], want[0])
        np.testing.assert_array_equal(got[1], want[1])
        np.testing.assert_array_equal(got[2].view(np.uint32), want[2].view(np.uint32))
        dist.barrier()
        if rank == 0:
            print(f"multi-gpu ok: world={world} search_range {storage} n={n} d={d} b={b} min_score={ms} path={path} "
                  f"hits={int(want[0][-1])}", flush=True)
    # filtered and subset lookups (row masks, predicates, subsets with duplicates and negative ordinals): equal to
    # the single-GPU VectorBase bit for bit on every rank (top-k through the peer exchange, the default; threshold
    # searches over the process group)
    for storage, n, d, b in (("float32", 50001, 96, 6), ("bfloat16", 120001, 128, 24)):
        v, q = O.make_corpus(n, d, seed=n + 2, n_queries=b)
        v[n // 2: n // 2 + 500] = v[:500]  # equal scores on different ranks
        sh = ShardedVectorBase(settings, device=local, storage_dtype=storage)
        sh.deserialize(v)
        whole = tab.VectorBase(settings, device=local, storage_dtype=storage)
        whole.add_embeddings(None, v)
        rng = np.random.default_rng(n)
        sub = np.concatenate([rng.permutation(n)[:3000], np.arange(500), n // 2 + np.arange(500), [-1, -n, 0]])
        allowed = rng.random(n) < 0.3
        pred = lambda i, a=allowed: bool(a[i])  # noqa: E731
        for tl in (False, True):
            for got, want in ((sh.search_arrays(q, 50, 0.4, subset=sub, ties_low_first=tl),
                               whole.search_arrays(q, 50, 0.4, subset=sub, ties_low_first=tl)),
                              (sh.search_arrays(q, 100, 0.4, allowed=allowed, ties_low_first=tl),
                               whole.search_arrays(q, 100, 0.4, allowed=allowed, ties_low_first=tl)),
                              (sh.search_range(q, 0.6, ties_low_first=tl, subset=sub),
                               whole.search_range(q, 0.6, subset=sub, ties_low_first=tl)),
                              (sh.search_range(q, 0.6, ties_low_first=tl, allowed=allowed),
                               whole.search_range(q, 0.6, allowed=allowed, ties_low_first=tl))):
                for g, w in zip(got, want):
                    np.testing.assert_array_equal(g.view(np.uint32) if g.dtype == np.float32 else g,
                                                  w.view(np.uint32) if w.dtype == np.float32 else w)
        for i in range(min(b, 4)):
            assert sh.fuzzy_lookup_embedding(q[i], 10, 0.3, predicate=pred) == \
                whole.fuzzy_lookup_embedding(q[i], 10, 0.3, predicate=pred)
            assert sh.fuzzy_lookup_embedding_in_subset(q[i], sub.tolist(), 20, 0.3) == \
                whole.fuzzy_lookup_embedding_in_subset(q[i], sub.tolist(), 20, 0.3)
        # per-query masks (2-D allowed=): each rank cuts its block's columns out of every query's mask
        qmasks = rng.random((b, n)) < np.array([0.3, 0.01, 1.0, 0.001] * b)[:b, None]
        qmasks[::2, :500] = True
        for tl in (False, True):
            for got, want in ((sh.search_arrays(q, 100, 0.4, allowed=qmasks, ties_low_first=tl),
                               whole.search_arrays(q, 100, 0.4, allowed=qmasks, ties_low_first=tl)),
                              (sh.search_range(q, 0.6, ties_low_first=tl, allowed=qmasks),
                               whole.search_range(q, 0.6, allowed=qmasks, ties_low_first=tl))):
                for g, w in zip(got, want):
                    np.testing.assert_array_equal(g.view(np.uint32) if g.dtype == np.float32 else g,
                                                  w.view(np.uint32) if w.dtype == np.float32 else w)
        # the same top-k lookups through either exchange, synchronous and deferred on the device
        subsets = [rng.permutation(n)[: 200 + 50 * i].astype(np.int64) - (n if i % 3 == 1 else 0) for i in range(b)]
        lookups = [dict(allowed=allowed), dict(allowed=allowed, ties_low_first=True), dict(allowed=qmasks),
                   dict(subset=sub), dict(subset=sub, ties_low_first=True), dict(subsets=subsets),
                   dict(subsets=subsets, ties_low_first=True)]
        wants = [whole.search_arrays(q, 40, 0.4, **kw) for kw in lookups]
        for exchange in ("peer", "nccl"):
            shx = sh if exchange == "peer" else ShardedVectorBase(settings, device=local, storage_dtype=storage,
                                                                  exchange="nccl")
            if exchange == "nccl":
                shx.deserialize(v)
            outs = [shx.search_tensors(q, 40, 0.4, defer_check=True, **kw) for kw in lookups]
            shx.finish()
            torch.cuda.synchronize()
            for kw, out, want in zip(lookups, outs, wants):
                got = [t.cpu().numpy() for t in out]
                for g, w in zip(got, want):
                    np.testing.assert_array_equal(g.view(np.uint32) if g.dtype == np.float32 else g,
                                                  w.view(np.uint32) if w.dtype == np.float32 else w)
                for g, w in zip(shx.search_arrays(q, 40, 0.4, **kw), want):
                    np.testing.assert_array_equal(g.view(np.uint32) if g.dtype == np.float32 else g,
                                                  w.view(np.uint32) if w.dtype == np.float32 else w)
        dist.barrier()
        if rank == 0:
            print(f"multi-gpu ok: world={world} filtered, subset and per-query-mask lookups {storage} n={n} d={d} "
                  f"b={b}, synchronous and deferred, peer and nccl exchanges", flush=True)
    # threshold searches through either exchange (exchange="peer": the range inbox over NVLink, with a grow when
    # min_score 0 returns every row): equal to the single-GPU search_range bit for bit on every rank
    n, d, b = 120001, 128, 24
    v, q = O.make_corpus(n, d, seed=n + 3, n_queries=b)
    whole = tab.VectorBase(settings, device=local, storage_dtype="bfloat16")
    whole.add_embeddings(None, v)
    rng = np.random.default_rng(n)
    sub = np.concatenate([rng.permutation(n)[:3000], np.arange(500), [-1, -n, 0]])
    subsets = [rng.permutation(n)[: 200 + 50 * i].astype(np.int64) for i in range(b)]
    searches = [(q, 0.6, {}), (q[:2], 0.0, {}), (q, 0.6, dict(allowed=rng.random(n) < 0.3, ties_low_first=True)),
                (q, 0.5, dict(allowed=rng.random((b, n)) < 0.3)), (q, 0.4, dict(subset=sub)),
                (q, 0.4, dict(subsets=subsets, ties_low_first=True))]
    for exchange in ("peer", "nccl"):
        shx = ShardedVectorBase(settings, device=local, storage_dtype="bfloat16", exchange=exchange)
        shx.deserialize(v)
        for qq, ms, kw in searches:
            for g, w in zip(shx.search_range(qq, ms, **kw), whole.search_range(qq, ms, **kw)):
                np.testing.assert_array_equal(g.view(np.uint32) if g.dtype == np.float32 else g,
                                              w.view(np.uint32) if w.dtype == np.float32 else w)
        shx.close()
    dist.barrier()
    if rank == 0:
        print(f"multi-gpu ok: world={world} threshold searches bfloat16 n={n} d={d} b={b}, peer and nccl exchanges",
              flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
