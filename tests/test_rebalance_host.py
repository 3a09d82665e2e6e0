"""Host logic of ``ShardedVectorBase.rebalance`` that needs no process group and no GPU: the plan of which rows move
(``rebalance_plan``), the target blocks and their argument checks (``rebalance_starts``), and the replacement of a
``VectorBase`` host mirror after its device rows were swapped, which must keep the row generation (the device
already holds the rows) and stay bit-exact with ``serialize()``."""

from __future__ import annotations

import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from typeagent_py_b200.sharded import rebalance_plan, rebalance_starts, shard_bounds  # noqa: E402


def starts_of(sizes):
    return [0] + np.cumsum(sizes, dtype=np.int64).tolist()


def laid_out(old_starts, new_starts):
    """Every destination rank's new block as the global rows its pieces name, in order."""
    world = len(old_starts) - 1
    blocks = {dst: [] for dst in range(world)}
    for dst, src, first, n in rebalance_plan(old_starts, new_starts):
        assert n > 0
        assert 0 <= first and first + n <= old_starts[src + 1] - old_starts[src]
        blocks[dst].extend(range(old_starts[src] + first, old_starts[src] + first + n))
    return blocks


CASES = [
    ("skewed by appends", [10, 10, 80], None),
    ("an emptied middle block", [50, 0, 50], None),
    ("every row on the first rank", [100, 0, 0, 0], None),
    ("fewer rows than ranks", [0, 0, 3], None),
    ("one row", [0, 1], None),
    ("custom sizes", [30, 30, 40], [0, 70, 30]),
    ("custom sizes with empty blocks", [5, 90, 5], [50, 0, 50]),
    ("eight ranks", [1, 2, 3, 4, 5, 6, 7, 972], None),
    ("one rank", [17], None),
]


@pytest.mark.parametrize("what,old,sizes", CASES, ids=[c[0].replace(" ", "_") for c in CASES])
def test_every_row_lands_once_in_destination_order(what, old, sizes):
    n, world = sum(old), len(old)
    old_starts = starts_of(old)
    new_starts = rebalance_starts(n, world, sizes)
    want = shard_bounds(n, world) if sizes is None else list(zip(new_starts[:-1], new_starts[1:]))
    assert list(zip(new_starts[:-1], new_starts[1:])) == want
    blocks = laid_out(old_starts, new_starts)
    for dst, (lo, hi) in enumerate(want):
        assert blocks[dst] == list(range(lo, hi)), (what, dst)
    plan = rebalance_plan(old_starts, new_starts)
    # destination by destination, each in global row order; at most one piece per (source, destination)
    assert [p[0] for p in plan] == sorted(p[0] for p in plan)
    assert len({(p[0], p[1]) for p in plan}) == len(plan)
    moved = sum(p[3] for p in plan if p[0] != p[1])
    rank_of = lambda starts, r: int(np.searchsorted(starts, r, side="right")) - 1  # noqa: E731
    assert moved == sum(rank_of(old_starts, r) != rank_of(new_starts, r) for r in range(n))


def test_no_op_plan_keeps_every_row_in_place():
    s = starts_of([4, 4, 3])
    plan = rebalance_plan(s, s)
    assert plan == [(0, 0, 0, 4), (1, 1, 0, 4), (2, 2, 0, 3)]
    assert rebalance_starts(11, 3) == s
    assert rebalance_plan([0, 0, 0], [0, 0, 0]) == []


@pytest.mark.parametrize("sizes,message", [
    ([1, 2], "entries"), ([5, 4, 4], "sum"), ([7, -1, 6], "negative"), ([4.0, 4, 4], "integers"),
    (["4", 4, 4], "integers"), ([4, 4, 4, 0], "entries")])
def test_invalid_sizes(sizes, message):
    with pytest.raises(ValueError, match=message):
        rebalance_starts(12, 3, sizes)


def test_sizes_take_numpy_integers():
    assert rebalance_starts(12, 3, np.array([0, 12, 0])) == [0, 0, 12, 12]


def test_plan_rejects_different_totals():
    with pytest.raises(ValueError):
        rebalance_plan([0, 5, 10], [0, 5, 11])


def test_mirror_replacement_keeps_the_generation_and_matches_serialize():
    from types import SimpleNamespace

    from oracle import vectorbase_oracle as O
    from typeagent_py_b200.vectorbase import VectorBase

    settings = SimpleNamespace(embedding_model=O.FakeEmbeddingModel(), min_score=0.85, max_matches=None)
    vb = VectorBase(settings)
    v, _ = O.make_corpus(40, 8, seed=3)
    vb.add_embeddings(None, v[:25])
    gen = vb._generation
    vb._mask_key, vb._qmask_key = ("k",), ("q",)
    vb._predicate_masks[("p", gen, 25)] = np.zeros(1, np.uint32)
    new = v[10:40].copy()
    new[3, 2] = np.float32(2.0 ** 17)   # beyond the fp16 range
    new[4, 0] = np.float32(np.nan)
    vb._replace_rebalanced(new)
    assert vb._generation == gen
    assert len(vb) == 30 and vb._ix_rows == 30
    np.testing.assert_array_equal(vb.serialize().view(np.uint32), new.view(np.uint32))
    assert vb._mask_key is None and vb._qmask_key is None and not vb._predicate_masks
    for i in (0, 3, 29):
        np.testing.assert_array_equal(vb.get_embedding_at(i).view(np.uint32), new[i].view(np.uint32))
    # appends after the replacement continue the new rows, still without a new generation
    vb.add_embeddings(None, v[:2])
    assert len(vb) == 32 and vb._generation == gen
    np.testing.assert_array_equal(vb.serialize()[30:], v[:2])

    # a base that never held a row learns the width from its new rows
    empty = VectorBase(settings)
    empty._replace_rebalanced(v[:5])
    assert empty._embedding_size == 8 and len(empty) == 5
    np.testing.assert_array_equal(empty.serialize(), v[:5])
