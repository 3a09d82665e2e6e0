"""One process, several GPUs: the device side of ``VectorBase(settings, devices=[...])``.

The float32 host mirror of ``VectorBase`` stays the authoritative copy of the rows.  The device side is W shard
indexes (``tav_index``), shard g holding the contiguous block of rows [starts[g], starts[g + 1]) on ``devices[g]``
(a device may repeat), and one ``tav_multi`` that fans a lookup out to every shard and merges on the first device
(``tav_multi_search`` / ``tav_multi_range_search``, csrc/tav_multi.cu).  The blocks follow the mirror lazily, at the
next lookup (``MultiDevice.sync``):

  * appended rows join the last block;
  * when the largest block then holds more than twice the even share (rows / W), the rows are split again as
    ``shard_bounds(rows, W)``; a shard whose block only loses a prefix and gains a suffix is updated in place
    (``tav_remove_rows`` + ``tav_append``), any other shard is reloaded from the mirror;
  * removals and overwrites go straight to the owning shards (``tav_remove_rows``, ``tav_write_rows``), and the block
    starts are recomputed as ``ShardedVectorBase.remove_embeddings`` recomputes them; a block may empty.

The layout rules are pure functions (``layout_plan``, ``removal_plan``, ``write_plan``) so that they are testable
without a GPU.
"""

from __future__ import annotations

import ctypes as C
import operator

import numpy as np

from . import _capi
from .sharded import as_topk_arrays, block_mask, shard_bounds

MAX_DEVICES = 32            # tav_multi_create's limit (tav_merge_range merges at most 32 lists)
MERGE_MAX_K = 8192          # tav_multi_search's limit; a larger k is served by the threshold search, cut to k
RESPLIT_SHARE = 2           # re-split when the largest block holds more than this many even shares
MULTI_FLAGS = _capi.TAV_FORCE_SCAN | _capi.TAV_FORCE_MMA | _capi.TAV_USE_ROW_MASK | _capi.TAV_TIES_LOW_FIRST


def check_devices(devices) -> list[int]:
    """``devices=`` as a list of CUDA ordinals: 1 to 32 non-negative integers, repeats allowed; TypeError or
    ValueError otherwise."""
    if isinstance(devices, (str, bytes)) or not hasattr(devices, "__len__"):
        raise TypeError(f"devices must be a sequence of CUDA device ordinals, not {type(devices).__name__}")
    out = []
    for d in devices:
        if isinstance(d, bool):
            raise TypeError("devices must hold integers, not bool")
        try:
            d = operator.index(d)
        except TypeError:
            raise TypeError(f"devices must hold integers, not {type(d).__name__}") from None
        if d < 0:
            raise ValueError(f"device ordinals must not be negative: {d}")
        out.append(d)
    if not 1 <= len(out) <= MAX_DEVICES:
        raise ValueError(f"devices must name 1 to {MAX_DEVICES} devices, not {len(out)}")
    return out


def even_starts(n_rows: int, world: int) -> list[int]:
    """Block starts [W + 1] of ``shard_bounds(n_rows, world)``."""
    return [lo for lo, _ in shard_bounds(n_rows, world)] + [n_rows]


def layout_plan(starts, n_rows: int, world: int) -> tuple[list[int], list[tuple[int, int, int, bool]]]:
    """The blocks after the device catches up with a mirror of ``n_rows`` rows, and what each shard is told.

    ``starts``: the blocks the shards hold now ([W + 1]; rows past starts[-1] are appended), or None when nothing on the
    devices can be kept (first use, or the rows were replaced).  Returns (new starts, steps); step g is
    (drop, lo, hi, reload): remove the first ``drop`` rows of shard g, or clear it when ``reload``, then append mirror
    rows [lo, hi)."""
    if starts is None:
        new = even_starts(n_rows, world)
        return new, [(0, new[g], new[g + 1], True) for g in range(world)]
    new = list(starts[:-1]) + [n_rows]
    if max(new[g + 1] - new[g] for g in range(world)) * world > RESPLIT_SHARE * n_rows:
        new = even_starts(n_rows, world)
    steps = []
    for g in range(world):
        a, b, c, d = starts[g], starts[g + 1], new[g], new[g + 1]
        if a <= c <= b <= d:
            steps.append((c - a, b, d, False))
        else:
            steps.append((0, c, d, True))
    return new, steps


def removal_plan(starts, removed: np.ndarray) -> tuple[list[np.ndarray], list[int]]:
    """Removal of the sorted, distinct mirror rows ``removed`` from blocks ``starts``: each shard's block-local ordinals
    (int64, ascending; rows at or past starts[-1] are not on the devices yet) and the new block starts."""
    per = [np.ascontiguousarray(removed[(removed >= lo) & (removed < hi)] - lo, dtype=np.int64)
           for lo, hi in zip(starts[:-1], starts[1:])]
    s = np.asarray(starts, np.int64)
    return per, (s - np.searchsorted(removed, s, side="left")).tolist()


def write_plan(starts, first: int, n: int) -> list[tuple[int, int, int, int]]:
    """Overwrite of mirror rows [first, first + n) on blocks ``starts``: (shard, its first row, source rows [lo, hi)
    relative to ``first``) for every block the rows touch; rows at or past starts[-1] are not on the devices yet."""
    out = []
    end = min(first + n, starts[-1])
    for g, (lo, hi) in enumerate(zip(starts[:-1], starts[1:])):
        a, b = max(lo, first), min(hi, end)
        if b > a:
            out.append((g, a - lo, a - first, b - first))
    return out


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


class MultiDevice:
    """The shard indexes and the ``tav_multi`` of one multi-device ``VectorBase``."""

    def __init__(self, devices: list[int], storage_dtype: str, normalize: bool):
        self.devices = list(devices)
        self.world = len(self.devices)
        self._dtype = _capi.DTYPE_CODES[storage_dtype]
        self._index_flags = _capi.TAV_NORMALIZE if normalize else 0
        self.shards: list | None = None  # tav_index handles
        self.handle = None               # tav_multi
        self.starts: list[int] | None = None
        self.generation = -1             # the mirror generation the shards hold
        self.dim = 0

    # ---- lifecycle ---------------------------------------------------------------------------
    def close(self, lib) -> None:
        if self.handle is not None:
            lib.tav_multi_destroy(self.handle)
            self.handle = None
        for ix in self.shards or ():
            lib.tav_destroy(ix)
        self.shards = None
        self.starts = None
        self.generation = -1

    def _open(self, lib) -> None:
        shards = []
        try:
            for dev in self.devices:
                h = C.c_void_p()
                _capi.check(lib.tav_create(dev, 0, self._dtype, self._index_flags, 0, C.byref(h)))
                shards.append(h)
            arr = (C.c_void_p * self.world)(*[h.value for h in shards])
            handle = C.c_void_p()
            _capi.check(lib.tav_multi_create(self.devices[0], self.world, arr, C.byref(handle)))
        except BaseException:
            for h in shards:
                lib.tav_destroy(h)
            raise
        self.shards, self.handle = shards, handle

    def in_sync(self, generation: int) -> bool:
        return self.starts is not None and self.generation == generation

    def sync(self, lib, rows: np.ndarray, generation: int, dim: int) -> bool:
        """Bring the shards up to date with the mirror ``rows`` (float32 [N, dim]) of ``generation``; True when the
        rows some shard holds changed (its row mask is then stale)."""
        if self.shards is not None and not self.in_sync(generation) and self.dim not in (0, dim):
            self.close(lib)  # the rows were replaced by rows of another width
        if self.shards is None:
            self._open(lib)
        self.dim = dim
        starts = self.starts if self.in_sync(generation) else None
        new, steps = layout_plan(starts, len(rows), self.world)
        if new == starts:
            return False
        self.starts, self.generation = None, -1  # a failure part way leaves nothing to keep
        for ix, (drop, lo, hi, reload) in zip(self.shards, steps):
            if reload:
                _capi.check(lib.tav_clear(ix))
            elif drop:
                gone = np.arange(drop, dtype=np.int64)
                _capi.check(lib.tav_remove_rows(ix, _ptr(gone), drop, None))
            if hi > lo:
                block = np.ascontiguousarray(rows[lo:hi], dtype=np.float32)
                _capi.check(lib.tav_append(ix, _ptr(block), hi - lo, dim, _capi.TAV_F32, 0, None))
        self.starts, self.generation = new, generation
        return True

    # ---- row changes -------------------------------------------------------------------------------
    def remove(self, lib, removed: np.ndarray) -> None:
        """Removal of the sorted, distinct mirror rows ``removed`` (call before the mirror changes)."""
        per, new = removal_plan(self.starts, removed)
        self.starts, self.generation, generation = None, -1, self.generation
        for ix, local in zip(self.shards, per):
            if len(local):
                _capi.check(lib.tav_remove_rows(ix, _ptr(local), len(local), None))
        self.starts, self.generation = new, generation

    def write(self, lib, first: int, rows: np.ndarray) -> None:
        """Overwrite of mirror rows [first, first + len(rows)) with ``rows`` (float32 [n, dim], C-contiguous)."""
        for g, local_first, lo, hi in write_plan(self.starts, first, len(rows)):
            part = rows[lo:hi]
            _capi.check(lib.tav_write_rows(self.shards[g], local_first, _ptr(part), hi - lo, self.dim, _capi.TAV_F32,
                                           0, None))

    def set_row_mask(self, lib, words: np.ndarray, n_rows: int) -> None:
        """A row mask over every row (packed uint32 words): each shard gets its block's bits."""
        for ix, lo, hi in zip(self.shards, self.starts[:-1], self.starts[1:]):
            if hi > lo:
                part = block_mask(words, n_rows, lo, hi)
                _capi.check(lib.tav_set_row_mask(ix, _ptr(part), hi - lo, 0, None))

    # ---- lookups -------------------------------------------------------------------------------------
    def topk(self, lib, q: np.ndarray, k: int, floor, flags: int, sub, items, scores, counts) -> None:
        """``tav_search`` over every block: results into the host arrays items / scores [B, k], counts [B]."""
        flags &= MULTI_FLAGS
        b = len(q)
        if k > MERGE_MAX_K:
            offsets, hits, hit_scores = self.range(lib, q, floor, flags, sub, b * k)
            items[:], scores[:], counts[:] = as_topk_arrays(offsets, hits, hit_scores, b, k)
            return
        starts = np.asarray(self.starts, np.int64)
        _capi.check(lib.tav_multi_search(
            self.handle, _ptr(starts), _ptr(q), b, k, C.c_float(float(floor)), flags,
            _ptr(sub) if sub is not None else None, len(sub) if sub is not None else 0,
            _ptr(items), _ptr(scores), _ptr(counts)))

    def range(self, lib, q: np.ndarray, floor, flags: int, sub, hint: int, offsets=None):
        """``tav_range_search`` over every block: (offsets int64 [B + 1], items int64 [T], scores float32 [T])."""
        flags &= MULTI_FLAGS
        b = len(q)
        if offsets is None:
            offsets = np.zeros(b + 1, dtype=np.int64)
        starts = np.asarray(self.starts, np.int64)
        _capi.check(lib.tav_multi_range_search(
            self.handle, _ptr(starts), _ptr(q), b, C.c_float(float(floor)), flags,
            _ptr(sub) if sub is not None else None, len(sub) if sub is not None else 0, int(hint), _ptr(offsets)))
        total = int(offsets[-1])
        items = np.empty(total, dtype=np.int64)
        scores = np.empty(total, dtype=np.float32)
        if total:
            _capi.check(lib.tav_multi_range_fetch(self.handle, 0, total, _ptr(items), _ptr(scores)))
        return offsets, items, scores
