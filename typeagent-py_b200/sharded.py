"""Row-sharded ``VectorBase`` across the GPUs of one box: one process per GPU
(``torch.distributed``), contiguous row blocks, one candidate all-gather per lookup.

Reference behaviour being scaled out: ``VectorBase.fuzzy_lookup_embedding`` (/root/reference/
src/typeagent/aitools/vectorbase.py:163-201) over the *whole* corpus.  Top-k is a decomposable
reduction, so every rank runs the single-GPU search on its rows (ordinals shifted to global
rows by ``item_offset``) and the per-rank ``[B, k]`` candidate lists — packed into one buffer —
are exchanged and merged on every rank.  Result: identical to the unsharded search, including
tie order.

Two exchanges:
  * ``exchange="peer"`` (default on CUDA): libtavec's own (``tav_sharded_search``, csrc/tav_group.cu) —
    every rank's publish kernel stores its list straight into every peer's HBM over NVLink (CUDA IPC
    mapped exchange regions, system-scope release flags), the merge waits on the flags; no NCCL call,
    no host synchronisation, two tiny launches after the local search.  ``torch.distributed`` only
    carries the 64-byte IPC handles once;
  * ``exchange="nccl"``: ONE ``all_gather_into_tensor`` + ``tav_merge_topk`` (also what the CPU tests
    drive over ``gloo`` with an injected engine).

Threshold searches (``search_range``; ``max_hits=0`` lookups and ``search_arrays`` with k >= rows > 8192) have
results whose size is known only after the local searches.  With ``exchange="peer"`` they go through the group's
range inbox (``tav_sharded_range_*``: every rank's offsets and hits stored into its peers' inboxes, the inboxes
grown collectively when a rank's hits do not fit); otherwise they exchange over the process group (offsets, then
the hits padded to the largest rank's total).  Either way ``tav_merge_range`` merges them.

Filtered and subset lookups (``predicate=``, ``fuzzy_lookup_embedding_in_subset``, ``subset=`` / ``allowed=`` /
``ties_low_first=``) return what ``VectorBase`` returns for the whole corpus, tie order included.  With
``exchange="peer"`` they take the peer exchange as well (``tav_sharded_search`` with the mask and tie flags,
``tav_sharded_search_subset``), can stay on the device and be deferred (``search_tensors``); otherwise they exchange
the packed layout over the process group and merge with ``tav_merge_topk_ordered``.  Either way: a row mask (a predicate is
evaluated by each rank over its own rows only) merges low row first where the reference's predicate path does;
a subset is searched per rank with ``TAV_ITEMS_AS_POSITIONS``, its hits mapped to positions in the caller's
subset (``tav_map_items``), merged by position and decoded through the caller's list at the end.  Per-query
subsets (``subsets=``, ``fuzzy_lookup_embeddings_in_subsets``) do the same with ``tav_search_subsets`` and the
entries' flat positions in the caller's concatenated ordinals.

``torch`` is plumbing here (process group, device buffers); the search, exchange and merge are
libtavec kernels.  The engine is injectable so that the host logic (partitioning, packing, gather,
offsets) is testable on CPU with the ``gloo`` backend.
"""

from __future__ import annotations

import ctypes as C
import operator
from array import array as _array

import numpy as np

from . import _capi
from .vectorbase import (_DEFAULT_MAX_HITS, ScoredInt, TextEmbeddingIndexSettings, VectorBase, _as_f32_scalar,
                         removal_ordinals)

RANGE_ROUTE_MIN_ROWS = 4 * 2048  # search_arrays with k >= rows above this (4 * TAV_PASS_K) -> search_range
# per-query subsets with a larger k are served by the threshold exchange and cut to k: the top-k merge keeps k keys
# per query in shared memory
SUBSETS_MERGE_MAX_K = 2048


def shard_bounds(n_rows: int, world: int) -> list[tuple[int, int]]:
    """Rank g owns rows [g*ceil(N/G), (g+1)*ceil(N/G)) clipped to N."""
    per = -(-n_rows // world) if world > 0 else 0
    return [(min(g * per, n_rows), min((g + 1) * per, n_rows)) for g in range(world)]


def rebalance_starts(n_rows: int, world: int, sizes=None) -> list[int]:
    """Block starts [world + 1] of a rebalance to ``shard_bounds(n_rows, world)``, or to blocks of ``sizes`` rows
    (``world`` non-negative integers summing to ``n_rows``; ValueError otherwise)."""
    if sizes is None:
        bounds = shard_bounds(n_rows, world)
        return [lo for lo, _ in bounds] + [n_rows]
    try:
        counts = [operator.index(s) for s in sizes]
    except TypeError:
        raise ValueError("sizes must be integers") from None
    if len(counts) != world:
        raise ValueError(f"sizes has {len(counts)} entries for {world} ranks")
    if any(c < 0 for c in counts):
        raise ValueError(f"sizes must not be negative: {counts}")
    if sum(counts) != n_rows:
        raise ValueError(f"sizes sum to {sum(counts)}, not to the {n_rows} rows")
    return [0] + np.cumsum(counts, dtype=np.int64).tolist()


def rebalance_plan(old_starts, new_starts) -> list[tuple[int, int, int, int]]:
    """Which rows a rebalance moves: pieces (destination rank, source rank, first row within the source's block,
    rows), destination by destination and, within one, in global row order, so that each rank's pieces laid out
    one after another are its new block.  Blocks are contiguous and ordered, so a (source, destination) pair
    has at most one piece."""
    world = len(old_starts) - 1
    if len(new_starts) != world + 1 or old_starts[-1] != new_starts[-1]:
        raise ValueError("old and new blocks must cover the same rows with the same number of ranks")
    plan = []
    for dst in range(world):
        lo, hi = new_starts[dst], new_starts[dst + 1]
        for src in range(world):
            a, b = max(lo, old_starts[src]), min(hi, old_starts[src + 1])
            if b > a:
                plan.append((dst, src, a - old_starts[src], b - a))
    return plan


# rows of one (source, destination) pair per round of the float32 mirror exchange of a rebalance: bounds the
# exchange's buffers on the communication device
MIRROR_ROUND_BYTES = 256 << 20


RANGE_MIN_HITS = 1 << 12       # the smallest range inbox: hits per rank
RANGE_RETAIN_BYTES = 64 << 20  # the most hit capacity a group keeps in its range inbox between threshold searches


def pow2_at_least(n: int, floor: int) -> int:
    """The smallest power of two that is at least ``n`` and ``floor``."""
    return 1 << (max(int(n), int(floor), 1) - 1).bit_length()


def range_retain_hits(world: int, retain_bytes: int = RANGE_RETAIN_BYTES) -> int:
    """Hits per rank the range inbox keeps between threshold searches: the largest power of two whose hits from
    every rank (12 bytes each) fit in ``retain_bytes``, and at least ``RANGE_MIN_HITS``."""
    per = max(int(retain_bytes) // (12 * max(world, 1)), 1)
    return max(1 << (per.bit_length() - 1), RANGE_MIN_HITS)


def range_capacity_plan(totals, capacity: int, retain: int) -> tuple[int | None, int | None]:
    """(grow, keep) of one threshold search through the range inbox, from every rank's total (replicated, so
    every rank plans alike) and the inbox's capacity in hits per rank: ``grow`` is the capacity to reserve before
    round 2 (the next power of two of the largest total), None when round 1 held every rank's hits; ``keep`` the
    capacity to give the excess back to at the end of the call, None when the inbox is within ``retain``."""
    t_max = int(np.max(totals)) if len(totals) else 0
    grow = pow2_at_least(t_max, RANGE_MIN_HITS) if t_max > capacity else None
    after = capacity if grow is None else grow
    return grow, (retain if after > retain else None)


def reserve_everywhere(dist, process_group, world: int, reserve, release) -> list[bytes]:
    """Collective: ``reserve()`` on every rank (an allocation; returns its handle), then every rank's (status,
    handle) through ``all_gather_object``.  If any rank failed, every rank runs ``release()`` and raises: its own
    error, else MemoryError when some rank ran out of memory, else RuntimeError.  Returns the handles in rank
    order."""
    status, handle, error = 0, b"", None
    try:
        handle = reserve()
    except Exception as e:  # noqa: BLE001
        status, error = (2 if isinstance(e, MemoryError) else 1), e
    got = [(status, handle)]
    if world > 1:
        got = [None] * world
        dist.all_gather_object(got, (status, handle), group=process_group)
    worst = max(st for st, _ in got)
    if worst:
        release()
        if error is not None:
            raise error
        raise (MemoryError if worst == 2 else RuntimeError)("search_range: another rank failed to reserve its "
                                                            "range inbox")
    return [h for _, h in got]


def packed_layout(n_queries: int, k: int) -> tuple[int, int, int]:
    """Byte offsets (scores, counts) and total size of one rank's packed candidate buffer:
    [items int64 B*k | scores float32 B*k | counts int32 B], each section 8-byte aligned."""
    a8 = lambda v: (v + 7) & ~7  # noqa: E731
    off_scores = a8(n_queries * k * 8)
    off_counts = off_scores + a8(n_queries * k * 4)
    total = off_counts + a8(n_queries * 4)
    return off_scores, off_counts, total


class CudaShardEngine:
    """The product engine: a GPU VectorBase for the local rows + libtavec's merge kernel."""

    def __init__(self, settings, device: int, storage_dtype: str = "float32"):
        import torch

        self.torch = torch
        self.device = torch.device("cuda", device)
        self.base = VectorBase(settings, device=device, storage_dtype=storage_dtype)
        self._group = None        # tav_group handle (peer exchange)
        self._group_keep = []     # outputs of deferred group searches, alive until finish
        self._range_cap_hint = RANGE_MIN_HITS  # range inbox capacity the last threshold search needed
        self.last_range_rounds = 0  # rounds (1, or 2 after a grow) of the last threshold search through the inbox

    # ---- peer exchange (tav_group) --------------------------------------------------------
    GROUP_DEPTH = 8

    def _ensure_group(self, dist, process_group, rank: int, world: int, n_queries: int, k: int):
        """(Re)create this rank's exchange region when the batch shape outgrows it — collectively:
        every rank calls with the same shape, the IPC handles travel through all_gather_object."""
        lib = _capi.load()
        if self._group is not None:
            mq, mk = C.c_int(0), C.c_int(0)
            _capi.check(lib.tav_group_capacity(self._group, C.byref(mq), C.byref(mk), None))
            if n_queries <= mq.value and k <= mk.value:
                return self._group
            self.group_finish()
            self.torch.cuda.synchronize(self.device)
            dist.barrier(group=process_group)       # nobody still publishes into a region about to die
            _capi.check(lib.tav_group_destroy(self._group))
            self._group = None
        handle = C.c_void_p()
        cap_q = max(256, 1 << (max(n_queries, 1) - 1).bit_length())
        cap_k = max(16, 1 << (max(k, 1) - 1).bit_length())
        _capi.check(lib.tav_group_create(self.device.index, rank, world, cap_q, cap_k, self.GROUP_DEPTH,
                                         C.byref(handle)))
        nbytes = lib.tav_group_handle_bytes()
        mine = C.create_string_buffer(nbytes)
        _capi.check(lib.tav_group_local_handle(handle, mine))
        gathered = [None] * world
        dist.all_gather_object(gathered, bytes(mine.raw), group=process_group)
        _capi.check(lib.tav_group_connect(handle, b"".join(gathered)))
        dist.barrier(group=process_group)
        self._group = handle
        return handle

    def group_search(self, dist, process_group, rank, world, queries, k, min_score, item_offset, defer_check,
                     ties_low_first=False, mask=None, subset=None):
        """One search through the peer exchange.  ``mask``: this block's packed words, key and owner (as
        ``search_rows_packed`` takes them), uploaded unless already on the device; ``subset``: this rank's share
        (block-local ordinals, their CSR offsets per query or None for one shared subset, their positions in the
        caller's list), searched by ``tav_sharded_search_subset``, whose merged items are those positions.  A local
        failure (the mask upload here, or the local search) is still published, so that every peer raises too."""
        torch = self.torch
        if isinstance(queries, np.ndarray):
            queries = torch.from_numpy(np.ascontiguousarray(queries, dtype=np.float32)).to(self.device, non_blocking=True)
        b = queries.shape[0]
        group = self._ensure_group(dist, process_group, rank, world, b, k)
        lib, ix = self.base._ensure_device()
        items = torch.empty((b, k), dtype=torch.int64, device=self.device)
        scores = torch.empty((b, k), dtype=torch.float32, device=self.device)
        counts = torch.empty((b,), dtype=torch.int32, device=self.device)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        flags = self.base._flags() | (_capi.TAV_DEFER_RETRY if defer_check else 0)
        flags |= _capi.TAV_TIES_LOW_FIRST if ties_low_first else 0
        error = None
        if mask is not None:
            flags |= _capi.TAV_USE_QUERY_MASKS if np.ndim(mask[0]) == 2 else _capi.TAV_USE_ROW_MASK
            try:
                self.upload_mask(mask, b)
            except Exception as e:  # noqa: BLE001
                error = e
                self._drop_masks(lib, ix)  # the local search then fails and publishes this rank's failure
        keep = (queries, items, scores, counts, stream)
        if subset is None:
            rc = lib.tav_sharded_search(ix, group, C.c_void_p(queries.data_ptr()), b, k, C.c_float(min_score), flags,
                                        item_offset, C.c_void_p(items.data_ptr()), C.c_void_p(scores.data_ptr()),
                                        C.c_void_p(counts.data_ptr()), C.c_void_p(stream))
        else:
            local, offsets, positions = subset
            sub = np.ascontiguousarray(local, np.int64)
            offs = None if offsets is None else np.ascontiguousarray(offsets, np.int64)
            pos = torch.from_numpy(np.ascontiguousarray(positions, np.int64)).to(self.device)
            keep += (pos,)
            rc = lib.tav_sharded_search_subset(
                ix, group, C.c_void_p(queries.data_ptr()), b, k, C.c_float(min_score), flags,
                sub.ctypes.data_as(C.c_void_p), len(sub), None if offs is None else offs.ctypes.data_as(C.c_void_p),
                C.c_void_p(pos.data_ptr()), C.c_void_p(items.data_ptr()), C.c_void_p(scores.data_ptr()),
                C.c_void_p(counts.data_ptr()), C.c_void_p(stream))
        if defer_check:  # a search that failed after its publish is open too: its buffers live until finish
            self._group_keep.append(keep)
        if error is not None:
            raise error
        _capi.check(rc)
        return items, scores, counts

    # ---- threshold search through the peer exchange (the group's range inbox) ---------------------------------
    RANGE_RETAIN_BYTES = RANGE_RETAIN_BYTES

    def range_capacity(self) -> tuple[int, int]:
        """(queries, hits per rank) the group's connected range inbox holds; (0, 0) without one."""
        if self._group is None:
            return 0, 0
        mq, cap = C.c_int(0), C.c_int64(0)
        _capi.check(_capi.load().tav_group_range_capacity(self._group, C.byref(mq), C.byref(cap)))
        return mq.value, cap.value

    def _range_reserve(self, dist, process_group, world: int, n_queries: int, capacity: int) -> None:
        """Collective: every rank's range inbox replaced by one for ``n_queries`` queries and ``capacity`` hits per
        rank, as ``_ensure_group`` makes a region: quiesce and wait for every rank, reserve, exchange (status,
        handle), connect.  If any rank fails (MemoryError for an allocation), every rank frees its inbox and raises,
        so that all ranks hold none and the next search reserves again; so does a failed connect."""
        lib = _capi.load()
        self.torch.cuda.synchronize(self.device)
        dist.barrier(group=process_group)       # nobody still reads or publishes into an inbox about to die

        def reserve() -> bytes:
            _capi.check(lib.tav_group_range_reserve(self._group, n_queries, capacity))
            buf = C.create_string_buffer(lib.tav_group_handle_bytes())
            _capi.check(lib.tav_group_range_handle(self._group, buf))
            return bytes(buf.raw)

        release = lambda: lib.tav_group_range_reserve(self._group, 0, 0)  # noqa: E731
        handles = reserve_everywhere(dist, process_group, world, reserve, release)
        # the connect is agreed too (its gather is the barrier after it): every rank holds a connected inbox, or none
        reserve_everywhere(dist, process_group, world,
                           lambda: _capi.check(lib.tav_group_range_connect(self._group, b"".join(handles))) or b"",
                           release)

    def group_range(self, dist, process_group, rank: int, world: int, queries: np.ndarray, min_score: float,
                    item_offset: int, ties_low_first: bool, mask=None, mask_key=None, mask_owner=None, subset=None,
                    positions=None, subsets=None):
        """One threshold search through the peer exchange (``tav_sharded_range_*``), collective.  Local arguments as
        ``range_local`` takes them; returns device tensors (offsets int64 [B + 1], items int64 [T], scores float32
        [T]), items being positions in the caller's subset(s) for the subset forms.  Round 1 publishes every rank's
        header, and its hits when they fit in the inbox; if some rank's did not, every rank reserves an inbox for
        the largest total and publishes again (``range_capacity_plan``).  A local failure (a mask upload here, or the
        local search) is still published, so that every peer raises too.  A failure after round 1 (the output
        allocation, say) closes the round on this rank (``tav_sharded_range_abort``: its peers' next publish does
        not wait for it) and raises on this rank only, after the give-back every rank runs; the peers' results are
        complete.  A failed grow raises on every rank."""
        torch = self.torch
        b = len(queries)
        group = self._ensure_group(dist, process_group, rank, world, 1, 1)
        retain = range_retain_hits(world, self.RANGE_RETAIN_BYTES)
        mq, cap = self.range_capacity()
        if b > mq:
            mq, cap = pow2_at_least(b, 64), min(max(cap, self._range_cap_hint), retain)
            self._range_reserve(dist, process_group, world, mq, cap)
        base = self.base
        lib, ix = base._ensure_device()
        q = np.ascontiguousarray(queries, np.float32)
        flags = (base._flags() & ~_capi.TAV_NO_FUSED_SCAN) | (_capi.TAV_TIES_LOW_FIRST if ties_low_first else 0)
        error, sub, offs, pos = None, None, None, None
        if mask is not None:
            flags |= _capi.TAV_USE_QUERY_MASKS if np.ndim(mask) == 2 else _capi.TAV_USE_ROW_MASK
        if subset is not None or subsets is not None:
            flags |= _capi.TAV_ITEMS_AS_POSITIONS
            sub = np.ascontiguousarray(subset if subsets is None else subsets[1], np.int64)
            offs = None if subsets is None else np.ascontiguousarray(subsets[0], np.int64)
            pos = np.ascontiguousarray(positions, np.int64)  # the library copies them (a failure there is published)
        headers = np.zeros((world, b + 2), np.int64)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        keep, totals, out = None, None, None
        base._single_lock.acquire()  # the index holds the hits until the last round has published them
        try:
            if mask is not None:
                try:
                    self.upload_mask((mask, mask_key, mask_owner), b)
                except Exception as e:  # noqa: BLE001
                    error = e
                    self._drop_masks(lib, ix)  # the local search then fails and publishes this rank's failure
            rc = lib.tav_sharded_range_search(
                ix, group, q.ctypes.data_as(C.c_void_p), b, C.c_float(min_score), flags,
                None if sub is None else sub.ctypes.data_as(C.c_void_p), 0 if sub is None else len(sub),
                None if offs is None else offs.ctypes.data_as(C.c_void_p),
                None if pos is None else pos.ctypes.data_as(C.c_void_p), item_offset, base._range_hint,
                headers.ctypes.data_as(C.c_void_p), C.c_void_p(stream))
            if error is not None:
                raise error
            _capi.check(rc)  # a failure of any rank's local search: raised on every rank, the round closed
            totals = headers[:, b]
            base._range_hint = int(totals[rank])
            grow, keep = range_capacity_plan(totals, cap, retain)
            self.last_range_rounds = 1
            if grow is not None:
                try:
                    self._range_reserve(dist, process_group, world, mq, grow)
                except Exception:
                    keep = None  # every rank raised and holds no inbox: nothing to give back
                    raise
                _capi.check(lib.tav_sharded_range_republish(group, C.c_void_p(stream)))
                self.last_range_rounds = 2
            total = int(totals.sum())
            out_offsets = torch.empty(b + 1, dtype=torch.int64, device=self.device)
            items = torch.empty(max(total, 1), dtype=torch.int64, device=self.device)
            scores = torch.empty(max(total, 1), dtype=torch.float32, device=self.device)
            _capi.check(lib.tav_sharded_range_merge(group, int(ties_low_first), C.c_void_p(out_offsets.data_ptr()),
                                                    C.c_void_p(items.data_ptr()), C.c_void_p(scores.data_ptr()),
                                                    C.c_void_p(stream)))
            out = out_offsets, items[:total], scores[:total]
        except Exception as e:  # noqa: BLE001
            error = e
            # a round still open on this rank is acknowledged, so that no peer's next publish waits for it
            lib.tav_sharded_range_abort(group, C.c_void_p(stream))
        finally:
            base._single_lock.release()
        if totals is not None:
            self._range_cap_hint = min(pow2_at_least(int(totals.max()), RANGE_MIN_HITS), retain)
        if keep is not None:  # give the excess back, on every rank alike (the totals are replicated)
            self._range_reserve(dist, process_group, world, mq, keep)
        if error is not None:
            raise error
        return out

    def upload_mask(self, mask, n_queries: int) -> None:
        """Put this block's mask (words, key, owner) on the device unless it is there already."""
        if self.n_local() == 0:
            return
        words, key, owner = mask
        lib, ix = self.base._ensure_device()
        if np.ndim(words) == 2:
            self.base._use_query_masks(lib, ix, words, n_queries)
        else:
            self.base._use_row_mask(lib, ix, words, key, owner)

    def _drop_masks(self, lib, ix) -> None:
        lib.tav_set_row_mask(ix, None, 0, 0, None)
        lib.tav_set_query_masks(ix, None, 0, 0, 0, 0, None)
        self.base._mask_key = self.base._qmask_key = None

    def group_finish(self) -> int:
        if self._group is None or not self._group_keep:
            return 0
        stream = self._group_keep[-1][4]
        redone = C.c_int(0)
        try:
            _capi.check(_capi.load().tav_sharded_finish(self.base._ix, self._group, C.c_void_p(stream), C.byref(redone)))
        finally:
            self._group_keep.clear()
        return redone.value

    def close(self, dist, process_group) -> None:
        """Collective: free this rank's exchange region and its rows, in the order that keeps every peer safe —
        synchronise the device, wait for every rank, destroy the region and the index, wait again — so that no
        rank frees a region a peer may still publish into.  Every rank passes both barriers even when its device
        failed; that error is raised afterwards."""
        error = None
        try:
            self.torch.cuda.synchronize(self.device)
        except Exception as e:  # noqa: BLE001
            error = e
        dist.barrier(group=process_group)
        group, self._group = self._group, None
        self._group_keep.clear()
        if group is not None:
            _capi.load().tav_group_destroy(group)
        self.base.clear()
        dist.barrier(group=process_group)
        if error is not None:
            raise error

    def __del__(self):
        try:
            if self._group is not None:
                _capi.load().tav_group_destroy(self._group)
                self._group = None
        except Exception:
            pass

    def comm_device(self):
        return self.device

    def n_local(self) -> int:
        return len(self.base)

    def load_rows(self, rows: np.ndarray | None) -> None:
        self.base.clear()
        if rows is not None and len(rows):
            self.base.add_embeddings(None, np.ascontiguousarray(rows, dtype=np.float32))

    def adopt_tensor(self, tensor) -> None:
        self.base = VectorBase.from_device_tensor(self.base.settings, tensor)

    def append_rows(self, rows: np.ndarray) -> None:
        self.base.add_embeddings(None, rows)

    def remove_rows(self, local_ordinals: np.ndarray) -> None:
        self.base.remove_embeddings(local_ordinals)

    # ---- rebalance (per-rank steps; ShardedVectorBase.rebalance runs the protocol) ------------------------
    def rows_adopted(self) -> bool:
        """The rows are caller-owned device memory (``adopt_tensor``): they cannot be handed out or replaced."""
        return self.base._adopted_tensor is not None

    def rows_export(self) -> bytes:
        """This rank's record for the peers (``tav_rows_export``), after the device rows caught up with the mirror."""
        lib, ix = self.base._ensure_device()
        rec = C.create_string_buffer(lib.tav_rows_handle_bytes())
        _capi.check(lib.tav_rows_export(ix, rec, None))
        return bytes(rec.raw)

    def mirror_from_rows(self) -> bool:
        """The device rows equal the float32 mirror bit for bit (float32 storage, not normalised): the new
        mirror is read back from the staged rows instead of being exchanged."""
        return self.base._storage_dtype == "float32" and not self.base._normalize

    def local_rows(self) -> np.ndarray:
        return self.base.serialize()

    def rows_stage(self, records: list[bytes], pieces: list[tuple[int, int, int]], rank: int, dim: int):
        """``tav_rows_stage`` of this rank's new block from ``pieces`` [(source rank, first row of its block, rows)]
        in order; returns the staged rows read back as the new mirror (``mirror_from_rows``) or None."""
        lib, ix = self.base._ensure_device()
        if lib.tav_dim(ix) == 0:  # a rank that never held a row learns the width (an empty append)
            _capi.check(lib.tav_append(ix, None, 0, dim, _capi.TAV_F32, 0, None))
        src = np.array([p[0] for p in pieces], np.int32)
        first = np.array([p[1] for p in pieces], np.int64)
        rows = np.array([p[2] for p in pieces], np.int64)
        mirror = np.empty((int(rows.sum()), dim), np.float32) if self.mirror_from_rows() else None
        stream = self.torch.cuda.current_stream(self.device).cuda_stream
        _capi.check(lib.tav_rows_stage(ix, len(records), rank, b"".join(records), len(pieces),
                                       src.ctypes.data_as(C.c_void_p), first.ctypes.data_as(C.c_void_p),
                                       rows.ctypes.data_as(C.c_void_p),
                                       None if mirror is None else mirror.ctypes.data_as(C.c_void_p),
                                       C.c_void_p(stream)))
        return mirror

    def rows_commit(self, commit: bool, mirror: np.ndarray | None = None) -> None:
        """Swap in the staged rows and ``mirror`` as the host mirror (``commit``), or drop them."""
        lib, ix = _capi.load(), self.base._ix
        if ix is None:
            return
        _capi.check(lib.tav_rows_commit(ix, int(commit)))
        if commit:
            self.base._replace_rebalanced(mirror)

    def finish(self) -> int:
        return self.base.finish_search()

    def search_packed(self, queries, k: int, min_score: float, item_offset: int, defer_check: bool = False):
        torch = self.torch
        if isinstance(queries, np.ndarray):
            queries = torch.from_numpy(np.ascontiguousarray(queries, dtype=np.float32)).to(
                self.device, non_blocking=True)
        b = queries.shape[0]
        off_s, off_c, total = packed_layout(b, k)
        buf = torch.empty(total, dtype=torch.uint8, device=self.device)
        items = buf[: b * k * 8].view(torch.int64).view(b, k)
        scores = buf[off_s : off_s + b * k * 4].view(torch.float32).view(b, k)
        counts = buf[off_c : off_c + b * 4].view(torch.int32)
        if self.n_local() == 0:
            counts.zero_()
        else:
            self.base.search_device(queries, k, min_score, item_offset=item_offset,
                                    out=(items, scores, counts), defer_check=defer_check)
        return buf

    def merge(self, gathered, world: int, n_queries: int, k: int):
        """gathered: uint8 [world, total] on the device -> (items, scores, counts) tensors."""
        torch = self.torch
        off_s, off_c, total = packed_layout(n_queries, k)
        items = torch.empty((n_queries, k), dtype=torch.int64, device=self.device)
        scores = torch.empty((n_queries, k), dtype=torch.float32, device=self.device)
        counts = torch.empty((n_queries,), dtype=torch.int32, device=self.device)
        base = gathered.data_ptr()
        stream = torch.cuda.current_stream(self.device).cuda_stream
        lib = _capi.load()
        _capi.check(
            lib.tav_merge_topk(self.device.index, world, n_queries, k, C.c_void_p(base),
                               C.c_void_p(base + off_s), C.c_void_p(base + off_c),
                               total // 8, total // 4, total // 4,
                               C.c_void_p(items.data_ptr()), C.c_void_p(scores.data_ptr()),
                               C.c_void_p(counts.data_ptr()), C.c_void_p(stream))
        )
        return items, scores, counts

    # ---- filtered and subset lookups (per-rank steps) --------------------------------------
    def _packed_views(self, buf, b: int, k: int):
        off_s, off_c, _ = packed_layout(b, k)
        return (buf[: b * k * 8].view(self.torch.int64).view(b, k),
                buf[off_s: off_s + b * k * 4].view(self.torch.float32).view(b, k),
                buf[off_c: off_c + b * 4].view(self.torch.int32))

    def search_rows_packed(self, queries: np.ndarray, k: int, min_score: float, item_offset: int,
                           ties_low_first: bool, mask=None, mask_key=None, mask_owner=None):
        """``tav_search`` of host queries over this rank's rows into a packed buffer on the device (items shifted
        by ``item_offset``): only rows whose bit is set in ``mask`` (this block's packed words; ``mask_key`` names
        it, so an unchanged mask is not uploaded again), equal scores lower row first with ``ties_low_first``."""
        torch = self.torch
        b = len(queries)
        buf = torch.empty(packed_layout(b, k)[2], dtype=torch.uint8, device=self.device)
        items, scores, counts = self._packed_views(buf, b, k)
        if self.n_local() == 0:
            counts.zero_()
            return buf
        base = self.base
        q = base._check_queries(queries)
        lib, ix = base._ensure_device()
        flags = base._flags() | _capi.TAV_OUTPUTS_ON_DEVICE
        if mask is not None and mask.ndim == 2:  # one mask per query (this block's columns)
            base._use_query_masks(lib, ix, mask, b)
            flags |= _capi.TAV_USE_QUERY_MASKS
        elif mask is not None:
            base._use_row_mask(lib, ix, mask, mask_key, mask_owner)
            flags |= _capi.TAV_USE_ROW_MASK
        if ties_low_first:
            flags |= _capi.TAV_TIES_LOW_FIRST
        stream = torch.cuda.current_stream(self.device).cuda_stream
        with base._single_lock:
            _capi.check(lib.tav_search(ix, q.ctypes.data_as(C.c_void_p), b, k, C.c_float(min_score), flags, None, 0,
                                       item_offset, C.c_void_p(items.data_ptr()), C.c_void_p(scores.data_ptr()),
                                       C.c_void_p(counts.data_ptr()), C.c_void_p(stream)))
        return buf

    def search_subset_packed(self, queries: np.ndarray, k: int, min_score: float, local_subset: np.ndarray,
                             positions: np.ndarray, ties_low_first: bool):
        """This rank's share of a subset search: ``tav_search`` over ``local_subset`` (block-local ordinals) with
        TAV_ITEMS_AS_POSITIONS, then those positions mapped through ``positions`` (where the share's entries
        stand in the whole subset, ascending) by ``tav_map_items``.  Returns the packed buffer on the device; its
        items are positions in the caller's subset.  Host outputs, so that one query takes the single-launch
        form as it does on one GPU; a rank without a share hands in empty lists."""
        torch = self.torch
        b = len(queries)
        off_s, off_c, total = packed_layout(b, k)
        host = np.zeros(total, np.uint8)
        if len(local_subset):
            base = self.base
            q = base._check_queries(queries)
            sub = np.ascontiguousarray(local_subset, np.int64)
            lib, ix = base._ensure_device()
            flags = base._flags() | _capi.TAV_ITEMS_AS_POSITIONS
            if ties_low_first:
                flags |= _capi.TAV_TIES_LOW_FIRST
            items = host[: b * k * 8].view(np.int64)
            scores = host[off_s: off_s + b * k * 4].view(np.float32)
            counts = host[off_c: off_c + b * 4].view(np.int32)
            with base._single_lock:
                _capi.check(lib.tav_search(ix, q.ctypes.data_as(C.c_void_p), b, k, C.c_float(min_score), flags,
                                           sub.ctypes.data_as(C.c_void_p), len(sub), 0, items.ctypes.data_as(C.c_void_p),
                                           scores.ctypes.data_as(C.c_void_p), counts.ctypes.data_as(C.c_void_p), None))
        buf = torch.from_numpy(host).to(self.device)
        if len(local_subset):
            self.map_items(buf[: b * k * 8].view(torch.int64), positions)
        return buf

    def search_subsets_packed(self, queries: np.ndarray, k: int, min_score: float, local_offsets: np.ndarray,
                              local_ordinals: np.ndarray, positions: np.ndarray, ties_low_first: bool):
        """This rank's share of a per-query subsets search: ``tav_search_subsets`` over each query's block-local
        entries (CSR ``local_offsets`` / ``local_ordinals``) with TAV_ITEMS_AS_POSITIONS, then those flat positions
        mapped through ``positions`` (where the share's entries stand in the caller's concatenated ordinals,
        ascending) by ``tav_map_items``.  Returns the packed buffer on the device; its items are flat positions in
        the caller's ordinals.  A rank without a share hands in empty lists."""
        torch = self.torch
        b = len(queries)
        off_s, off_c, total = packed_layout(b, k)
        host = np.zeros(total, np.uint8)
        if len(local_ordinals):
            base = self.base
            q = base._check_queries(queries)
            offs = np.ascontiguousarray(local_offsets, np.int64)
            ords = np.ascontiguousarray(local_ordinals, np.int64)
            lib, ix = base._ensure_device()
            flags = _capi.TAV_ITEMS_AS_POSITIONS | (_capi.TAV_TIES_LOW_FIRST if ties_low_first else 0)
            items = host[: b * k * 8].view(np.int64)
            scores = host[off_s: off_s + b * k * 4].view(np.float32)
            counts = host[off_c: off_c + b * 4].view(np.int32)
            with base._single_lock:
                _capi.check(lib.tav_search_subsets(ix, q.ctypes.data_as(C.c_void_p), b, k, C.c_float(min_score), flags,
                                                   offs.ctypes.data_as(C.c_void_p), ords.ctypes.data_as(C.c_void_p),
                                                   items.ctypes.data_as(C.c_void_p), scores.ctypes.data_as(C.c_void_p),
                                                   counts.ctypes.data_as(C.c_void_p), None))
        buf = torch.from_numpy(host).to(self.device)
        if len(local_ordinals):
            self.map_items(buf[: b * k * 8].view(torch.int64), positions)
        return buf

    def map_items(self, items, table: np.ndarray):
        """In place on the device: items[i] = table[items[i]] where 0 <= items[i] < len(table) (``tav_map_items``);
        ``items`` an int64 device tensor, ``table`` host int64."""
        torch = self.torch
        t = torch.from_numpy(np.ascontiguousarray(table, np.int64)).to(self.device)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        _capi.check(_capi.load().tav_map_items(self.device.index, items.numel(), C.c_void_p(t.data_ptr()), t.numel(),
                                               C.c_void_p(items.data_ptr()), C.c_void_p(stream)))
        return items

    def merge_ordered(self, gathered, world: int, n_queries: int, k: int, order: int):
        """``merge`` with ``tav_merge_topk_ordered``'s tie order: 0 as ``merge``, 1 lower row first, 2 / 3 the
        item (a subset position) higher / lower first.  ``gathered``: uint8 [world, row] with one rank's packed
        buffer at the start of each row (a row may be longer, a multiple of 8 bytes)."""
        torch = self.torch
        off_s, off_c, _ = packed_layout(n_queries, k)
        total = gathered.shape[1]
        items = torch.empty((n_queries, k), dtype=torch.int64, device=self.device)
        scores = torch.empty((n_queries, k), dtype=torch.float32, device=self.device)
        counts = torch.empty((n_queries,), dtype=torch.int32, device=self.device)
        base = gathered.data_ptr()
        stream = torch.cuda.current_stream(self.device).cuda_stream
        _capi.check(_capi.load().tav_merge_topk_ordered(
            self.device.index, world, n_queries, k, C.c_void_p(base), C.c_void_p(base + off_s),
            C.c_void_p(base + off_c), total // 8, total // 4, total // 4, int(order), C.c_void_p(items.data_ptr()),
            C.c_void_p(scores.data_ptr()), C.c_void_p(counts.data_ptr()), C.c_void_p(stream)))
        return items, scores, counts

    # ---- threshold search (search_range) ---------------------------------------------------
    def range_local(self, queries: np.ndarray, min_score: float, item_offset: int, ties_low_first: bool,
                    mask=None, mask_key=None, mask_owner=None, subset=None, positions=None, subsets=None):
        """``tav_range_search`` on this rank's rows (items shifted by ``item_offset``).  Returns a
        ``LocalRange``: host offsets [B + 1] now, the hits later straight into the caller's buffers.  The
        hits wait in the index between the two calls, so the base's lookup lock is held until then.
        ``mask`` as in ``search_rows_packed``.  ``subset`` / ``positions`` as in ``search_subset_packed``, or
        ``subsets`` (this block's (offsets, ordinals) CSR) / ``positions`` as in ``search_subsets_packed``: the
        hits' items are then positions in the caller's subset(s), and are fetched into device buffers only."""
        base = self.base
        b = len(queries)
        if (self.n_local() == 0 or (subset is not None and len(subset) == 0)
                or (subsets is not None and len(subsets[1]) == 0)):
            return LocalRange(np.zeros(b + 1, np.int64), None, None)
        q = base._check_queries(queries)
        sub = None if subset is None else np.ascontiguousarray(subset, np.int64)
        csr = None if subsets is None else tuple(np.ascontiguousarray(a, np.int64) for a in subsets)
        base._single_lock.acquire()
        try:
            lib, ix = base._ensure_device()
            flags = base._flags() & ~_capi.TAV_NO_FUSED_SCAN
            if ties_low_first:
                flags |= _capi.TAV_TIES_LOW_FIRST
            if mask is not None and mask.ndim == 2:  # one mask per query (this block's columns)
                base._use_query_masks(lib, ix, mask, b)
                flags |= _capi.TAV_USE_QUERY_MASKS
            elif mask is not None:
                base._use_row_mask(lib, ix, mask, mask_key, mask_owner)
                flags |= _capi.TAV_USE_ROW_MASK
            if sub is not None:
                flags |= _capi.TAV_ITEMS_AS_POSITIONS
                item_offset = 0
            offsets = np.zeros(b + 1, np.int64)
            if csr is not None:
                flags = _capi.TAV_ITEMS_AS_POSITIONS | (_capi.TAV_TIES_LOW_FIRST if ties_low_first else 0)
                _capi.check(lib.tav_range_search_subsets(ix, q.ctypes.data_as(C.c_void_p), b, C.c_float(min_score),
                                                         flags, csr[0].ctypes.data_as(C.c_void_p),
                                                         csr[1].ctypes.data_as(C.c_void_p),
                                                         offsets.ctypes.data_as(C.c_void_p), None))
            else:
                _capi.check(lib.tav_range_search(ix, q.ctypes.data_as(C.c_void_p), b, C.c_float(min_score), flags,
                                                 None if sub is None else sub.ctypes.data_as(C.c_void_p),
                                                 0 if sub is None else len(sub), item_offset, base._range_hint,
                                                 offsets.ctypes.data_as(C.c_void_p), None))
                base._range_hint = int(offsets[-1])
        except BaseException:
            base._single_lock.release()
            raise
        stream = self.torch.cuda.current_stream(self.device).cuda_stream

        def fetch(items, scores):
            n = int(offsets[-1])
            if n == 0:
                return
            on_device = not isinstance(items, np.ndarray)
            if (sub is not None or csr is not None) and not on_device:
                raise ValueError("the hits of a subset threshold search are fetched into device buffers")
            ip = C.c_void_p(items.data_ptr()) if on_device else items.ctypes.data_as(C.c_void_p)
            sp = C.c_void_p(scores.data_ptr()) if on_device else scores.ctypes.data_as(C.c_void_p)
            _capi.check(lib.tav_range_fetch(ix, 0, n, ip, sp, _capi.TAV_OUTPUTS_ON_DEVICE if on_device else 0,
                                            C.c_void_p(stream) if on_device else None))
            if sub is not None or csr is not None:
                self.map_items(items[:n], positions)

        return LocalRange(offsets, fetch, base._single_lock)

    def merge_range(self, offsets_all, payload, world: int, n_queries: int, t_pad: int, total: int,
                    ties_low_first: bool):
        """``tav_merge_range`` over the all-gathered lists: ``offsets_all`` int64 [world, B + 2] (offsets and a
        status word per rank), ``payload`` uint8 [world, 12 * t_pad] (items int64 [t_pad], then scores float32
        [t_pad]) -> (offsets int64 [B + 1], items int64 [total], scores float32 [total]) device tensors."""
        torch = self.torch
        out_offsets = torch.empty(n_queries + 1, dtype=torch.int64, device=self.device)
        items = torch.empty(max(total, 1), dtype=torch.int64, device=self.device)
        scores = torch.empty(max(total, 1), dtype=torch.float32, device=self.device)
        base = payload.data_ptr()
        stream = self.torch.cuda.current_stream(self.device).cuda_stream
        _capi.check(_capi.load().tav_merge_range(
            self.device.index, world, n_queries, C.c_void_p(offsets_all.data_ptr()), offsets_all.shape[1],
            C.c_void_p(base), 12 * t_pad // 8, C.c_void_p(base + 8 * t_pad), 12 * t_pad // 4, int(ties_low_first),
            C.c_void_p(out_offsets.data_ptr()), C.c_void_p(items.data_ptr()), C.c_void_p(scores.data_ptr()),
            C.c_void_p(stream)))
        return out_offsets, items[:total], scores[:total]


MAX_RANGE_RANKS = 32  # lists tav_merge_range merges in one call


def offsets_with_status(offsets: np.ndarray, failed: bool) -> np.ndarray:
    """One rank's first exchange of a threshold search: its offsets [B + 1], then a status word (1 = failed)."""
    return np.concatenate([np.asarray(offsets, np.int64), [int(failed)]]).astype(np.int64)


def range_pad(totals) -> int:
    """Hits per rank in the payload exchange: the largest rank's total, rounded up to even so that every rank's
    scores section stays 8-byte aligned."""
    t = int(np.max(totals))
    return t + (t & 1)


def pack_range_payload(local, t_pad: int, device):
    """One rank's payload of the second exchange, uint8 [12 * t_pad]: items int64 [t_pad], then scores float32
    [t_pad], the hits first; ``local.fetch`` writes them straight into it."""
    import torch

    send = torch.empty(12 * t_pad, dtype=torch.uint8, device=device)
    n = int(local.offsets[-1])
    local.fetch(send[: 8 * n].view(torch.int64), send[8 * t_pad: 8 * t_pad + 4 * n].view(torch.float32))
    return send


def subset_ordinals(subset, from_list: bool = False) -> np.ndarray:
    """A caller's subset as int64 [m], read as ``VectorBase`` reads it: IndexError for a non-integer array
    (``from_list``: a Python list goes through ``array('q')`` first, as ``fuzzy_lookup_embedding_in_subset``
    takes it)."""
    if from_list and type(subset) is list:
        try:
            return np.frombuffer(_array("q", subset), dtype=np.int64)
        except (TypeError, OverflowError):
            pass
    sub = np.ascontiguousarray(subset)
    if sub.size and not np.issubdtype(sub.dtype, np.integer):
        raise IndexError("arrays used as indices must be of integer (or boolean) type")
    return sub.astype(np.int64, copy=False).reshape(-1)


def check_subset(sub: np.ndarray, n_rows: int) -> None:
    """IndexError, with the library's message, for an ordinal outside [-n_rows, n_rows)."""
    bad = (sub < -n_rows) | (sub >= n_rows)
    if bad.any():
        raise IndexError(f"index {int(sub[bad][0])} is out of bounds for axis 0 with size {n_rows}")


def subset_share(sub: np.ndarray, n_rows: int, lo: int, hi: int) -> tuple[np.ndarray, np.ndarray]:
    """The entries of a subset that fall in rows [lo, hi): their positions in the subset (ascending) and their
    block-local ordinals.  Negative ordinals wrap with the global row count; a repeated ordinal is one entry
    per occurrence."""
    rows = np.where(sub < 0, sub + n_rows, sub)
    pos = np.flatnonzero((rows >= lo) & (rows < hi)).astype(np.int64)
    return pos, rows[pos] - lo


def check_subsets_total(total: int) -> None:
    """ValueError when a per-query subsets lookup has 2^32 ordinals or more: their flat positions are 32-bit keys."""
    if total >= 1 << 32:
        raise ValueError(f"{total} ordinals in one per-query subsets lookup; at most 2^32 - 1")


def subsets_share(offsets: np.ndarray, ordinals: np.ndarray, n_rows: int, lo: int,
                  hi: int) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """The entries of per-query subsets (CSR ``offsets`` [B + 1], ``ordinals`` [T]) that fall in rows [lo, hi):
    their flat positions in ``ordinals`` (ascending), the share as CSR offsets [B + 1] and block-local ordinals.
    Negative ordinals wrap with the global row count; a repeated ordinal is one entry per occurrence."""
    rows = np.where(ordinals < 0, ordinals + n_rows, ordinals)
    inside = (rows >= lo) & (rows < hi)
    pos = np.flatnonzero(inside).astype(np.int64)
    before = np.concatenate([[0], np.cumsum(inside, dtype=np.int64)])
    return pos, before[offsets], rows[pos] - lo


def block_mask(allowed, n_rows: int, lo: int, hi: int, n_queries: int | None = None) -> np.ndarray:
    """Rows [lo, hi) of a row mask over n_rows rows (bool [n_rows], or packed uint32 words as
    ``VectorBase.pack_row_mask`` makes them), packed again from bit 0: a block need not start on a word.
    A 2-D mask (one per query: bool [B, n_rows] or packed words [B, ceil(n_rows / 32)]) gives each query's
    columns [lo, hi), packed per query as ``VectorBase.pack_query_masks`` does.  ValueError, with
    ``VectorBase``'s message, for a mask of the wrong length, or (``n_queries``) the wrong number of masks."""
    if np.ndim(allowed) == 2:
        shape = np.shape(allowed)
        if n_queries is not None and shape[0] != n_queries:
            raise ValueError(f"query masks have {shape[0]} rows for {n_queries} queries")
        if getattr(allowed, "dtype", None) == np.uint32:
            if shape[1] != (n_rows + 31) // 32:
                raise ValueError(f"query masks have {shape[1] * 32} bits for {n_rows} rows")
            words = np.ascontiguousarray(allowed)
            bits = np.unpackbits(words.view(np.uint8), axis=1, bitorder="little")[:, lo:hi].astype(bool)
        else:
            if shape[1] != n_rows:
                raise ValueError(f"query masks have {shape[1]} entries for {n_rows} rows")
            bits = np.asarray(allowed, dtype=bool)[:, lo:hi]
        return VectorBase.pack_query_masks(bits)
    if np.ndim(allowed) != 1:
        raise ValueError(f"allowed= must be one row mask (1-D) or one mask per query (2-D), not {np.ndim(allowed)}-D")
    if getattr(allowed, "dtype", None) == np.uint32:
        words = np.ascontiguousarray(allowed)
        if len(words) != (n_rows + 31) // 32:
            raise ValueError(f"row mask has {len(words) * 32} bits for {n_rows} rows")
        bits = np.unpackbits(words.view(np.uint8), bitorder="little")[lo:hi].astype(bool)
    else:
        if len(allowed) != n_rows:
            raise ValueError(f"row mask has {len(allowed)} entries for {n_rows} rows")
        bits = np.asarray(allowed, dtype=bool)[lo:hi]
    return VectorBase.pack_row_mask(bits)


def as_topk_arrays(offsets, hits, hit_scores, b: int, k: int):
    """CSR threshold-search results laid out as [B, k] top-k arrays (-1 / 0 padding), as ``tav_search`` lays
    out a search it routes to the threshold engine: the first k hits of each query."""
    per = np.diff(offsets)
    items = np.full((b, k), -1, np.int64)
    scores = np.zeros((b, k), np.float32)
    cols = np.arange(len(hits)) - np.repeat(offsets[:-1], per)
    rows = np.repeat(np.arange(b), per)
    keep = cols < k
    items[rows[keep], cols[keep]] = hits[keep]
    scores[rows[keep], cols[keep]] = hit_scores[keep]
    return items, scores, np.minimum(per, k).astype(np.int32)


class LocalRange:
    """One rank's threshold-search result between the search and the fetch of its hits: ``offsets`` (host
    int64 [B + 1]); ``fetch(items, scores)`` writes the hits into the given buffers (device tensors or host
    arrays) and releases ``lock``; ``release()`` releases it without fetching.  Exactly one of them is called."""

    def __init__(self, offsets: np.ndarray, fetch, lock=None):
        self.offsets = offsets
        self._fetch = fetch
        self._lock = lock

    def fetch(self, items, scores) -> None:
        try:
            if self._fetch is not None:
                self._fetch(items, scores)
        finally:
            self.release()

    def release(self) -> None:
        lock, self._lock = self._lock, None
        if lock is not None:
            lock.release()


class ShardedVectorBase:
    """Global corpus [N, D] partitioned by contiguous row blocks over the ranks of a
    process group.  Every rank calls every method with the same arguments (SPMD)."""

    def __init__(self, settings: TextEmbeddingIndexSettings, *, process_group=None,
                 device: int | None = None, storage_dtype: str = "float32", engine=None,
                 exchange: str = "peer", rebalance_at: float | None = None):
        """``rebalance_at``: when set (at least 1), ``add_embeddings`` and ``remove_embeddings`` call ``rebalance()``
        whenever the largest block holds more than ``rebalance_at`` times the even share (rows / ranks).  A rebalance
        holds each rank's new block beside its old one until it commits, so the bound must fire while the fullest
        GPU still has room for an even share more."""
        import torch.distributed as dist

        if exchange not in ("peer", "nccl"):
            raise ValueError("exchange must be 'peer' or 'nccl'")
        if rebalance_at is not None and not rebalance_at >= 1.0:
            raise ValueError(f"rebalance_at must be at least 1, not {rebalance_at}")
        self.exchange = exchange
        self.rebalance_at = rebalance_at
        self.settings = settings
        self._dist = dist
        self._group = process_group
        self.rank = dist.get_rank(process_group)
        self.world = dist.get_world_size(process_group)
        if engine is None:
            import os

            if device is None:
                device = int(os.environ.get("LOCAL_RANK", self.rank))
            engine = CudaShardEngine(settings, device, storage_dtype)
        self._engine = engine
        self._starts = [0] * (self.world + 1)  # global row where each rank's block starts
        self._embedding_size = 0
        self._pending: list = []  # deferred searches since the last finish(): ["group"] or (local, b, k, out) tuples
        self._generation = 0      # bumped whenever rows are replaced or removed (part of the mask cache keys)
        self._masks: dict = {}    # (kind, id(mask or predicate), generation, rows) -> (this block's words, owner)
        self._peer_masks: dict = {}  # "row" / "query" -> key of the mask every rank uploaded for the peer exchange
        self._decode: list = []   # (items, list) of deferred subset lookups: positions decoded at finish()

    # ---- corpus ------------------------------------------------------------------------
    def __len__(self) -> int:
        return self._starts[-1]

    def __bool__(self) -> bool:
        return True

    @property
    def local_range(self) -> tuple[int, int]:
        return self._starts[self.rank], self._starts[self.rank + 1]

    @property
    def blocks(self) -> list[tuple[int, int]]:
        """Every rank's block of global rows, [(lo, hi)] in rank order (the same on every rank)."""
        return [(self._starts[r], self._starts[r + 1]) for r in range(self.world)]

    def _set_bounds(self, bounds) -> None:
        self._starts = [lo for lo, _ in bounds] + [bounds[-1][1]]

    def deserialize(self, data: np.ndarray | None) -> None:
        """Bulk load: every rank passes the same global float32 [N, D] array (or a
        memory-map of it) and keeps only its own block."""
        self._generation += 1
        if data is None or data.ndim < 2 or len(data) == 0:
            self._engine.load_rows(None)
            self._starts = [0] * (self.world + 1)
            return
        self._embedding_size = data.shape[1]
        bounds = shard_bounds(len(data), self.world)
        self._set_bounds(bounds)
        lo, hi = bounds[self.rank]
        self._engine.load_rows(data[lo:hi])

    def load_local_shard(self, rows, global_rows: int) -> None:
        """Each rank supplies only its own block (numpy rows or a CUDA tensor) of a global
        corpus of ``global_rows`` rows partitioned by ``shard_bounds``."""
        bounds = shard_bounds(global_rows, self.world)
        lo, hi = bounds[self.rank]
        if len(rows) != hi - lo:
            raise ValueError(f"rank {self.rank} must hold rows [{lo}, {hi}), got {len(rows)} rows")
        self._set_bounds(bounds)
        self._generation += 1
        self._embedding_size = rows.shape[1]
        if isinstance(rows, np.ndarray):
            self._engine.load_rows(rows)
        else:
            self._engine.adopt_tensor(rows)

    def add_embeddings(self, keys, embeddings: np.ndarray) -> None:
        """Append rows (global ordinals continue at len(self)); they join the LAST rank's block so that blocks stay
        contiguous and ordered.  ``rebalance()`` moves rows between ranks so that every block is its even share
        again; with ``rebalance_at`` set, this call does so when the last block grew past that bound.  If that
        rebalance fails (MemoryError when a rank cannot hold its new block beside its old one, for one), this call
        raises on every rank AFTER the rows were appended: they are in the index, with their ordinals, and the
        blocks stay as they were; do not append them again.  The next append or removal tries the rebalance
        again."""
        if embeddings.ndim != 2:
            raise ValueError(f"Expected 2D embeddings array, got {embeddings.ndim}D")
        if self._embedding_size == 0:
            self._embedding_size = embeddings.shape[1]
        if embeddings.shape[1] != self._embedding_size:
            raise ValueError(
                f"Embedding size mismatch: expected {self._embedding_size}, got {embeddings.shape[1]}")
        if self.rank == self.world - 1:
            self._engine.append_rows(np.ascontiguousarray(embeddings, dtype=np.float32))
        self._starts[-1] += len(embeddings)
        if keys is not None:
            for key, row in zip(keys, embeddings):
                self.settings.embedding_model.add_embedding(key, row)
        self._rebalance_if_skewed()

    def remove_embeddings(self, ordinals) -> None:
        """Remove rows by global ordinal, as ``VectorBase.remove_embeddings`` does on one GPU (``np.delete``
        semantics: integer ordinals or a boolean mask over every row; IndexError, with nothing removed, for an
        ordinal out of range).  SPMD: every rank passes the same ordinals.  Deferred lookups are finished first
        (``finish()``, collective): the local removal redoes their flagged queries on the old rows, and only
        ``finish()`` exchanges and merges the corrected candidates again.  Each rank then removes its own block's
        share and recomputes the block starts from the replicated list, without a collective; blocks may become
        uneven (a block may empty) until ``rebalance()``, which this call runs when ``rebalance_at`` says so.  If
        that rebalance fails, this call raises on every rank AFTER the rows were removed; the blocks stay as they
        were, and the next append or removal tries again."""
        removed = removal_ordinals(ordinals, len(self))
        if removed.size == 0:
            return
        self.finish()
        lo, hi = self.local_range
        mine = removed[(removed >= lo) & (removed < hi)] - lo
        if len(mine):
            self._engine.remove_rows(mine)
        starts = np.asarray(self._starts, np.int64)
        self._starts = (starts - np.searchsorted(removed, starts, side="left")).tolist()
        self._generation += 1
        self._rebalance_if_skewed()

    # ---- rebalance -----------------------------------------------------------------------
    def _rebalance_if_skewed(self) -> None:
        if self.rebalance_at is None or len(self) == 0:
            return
        largest = max(hi - lo for lo, hi in self.blocks)
        if largest * self.world > self.rebalance_at * len(self):
            self.rebalance()

    def rebalance(self, sizes=None) -> int:
        """Move rows between ranks so that rank r holds ``shard_bounds(len(self), world)[r]``, or, with ``sizes``
        (one non-negative integer per rank, summing to ``len(self)``), that many rows, blocks contiguous and in
        rank order.  Returns the number of rows that changed rank, the same on every rank.  Collective and SPMD.

        Global ordinals do not change, so every lookup returns what it returned before.  Nothing happens, and no
        collective runs, when the blocks already are the target.  Invalid ``sizes`` raise ValueError on every rank
        before any collective.  Deferred lookups are finished first (``finish()``).  Each rank then copies its new
        block, in the storage dtype and byte for byte, from its own rows and its peers' (CUDA IPC, the copy
        engines); the float32 host mirrors follow, read back from the new rows or exchanged over the process
        group.  If any rank fails (an allocation, a copy, rows that are adopted device memory), every rank raises
        (MemoryError for a failed allocation) and nothing changes anywhere.  Until it commits, each rank holds its
        new block (device memory for its new row count) beside its old one."""
        target = rebalance_starts(len(self), self.world, sizes)
        if target == list(self._starts):
            return 0
        plan = rebalance_plan(self._starts, target)
        moved = sum(n for dst, src, _, n in plan if dst != src)
        self.finish()
        engine = self._engine
        # every rank's record of its rows, with a status: 0 fine, 1 adopted rows, 2 failed
        status, record, error = 0, b"", None
        try:
            if engine.rows_adopted():
                status = 1
            else:
                record = engine.rows_export()
        except Exception as e:  # noqa: BLE001
            status, error = 2, e
        got = [(status, record)]
        if self.world > 1:
            got = [None] * self.world
            self._dist.all_gather_object(got, (status, record), group=self._group)
        adopted = [r for r, (st, _) in enumerate(got) if st == 1]
        if adopted:
            raise RuntimeError(f"rebalance: the rows of rank(s) {adopted} are adopted device memory "
                               "(from_device_tensor / load_local_shard with a tensor) and cannot move")
        if any(st for st, _ in got):
            raise error if error is not None else RuntimeError("rebalance: another rank failed to export its rows")
        error, mirror = None, None
        try:
            mirror = engine.rows_stage([rec for _, rec in got], [(src, first, n) for dst, src, first, n in plan
                                                                 if dst == self.rank],
                                       self.rank, self._embedding_size)
        except Exception as e:  # noqa: BLE001
            error = e
        code = 0
        if not engine.mirror_from_rows():
            # the mirror exchange is a collective: the ranks agree first that every one of them can enter it
            code = self._worst_status(error)
            if code == 0:
                try:
                    mirror = self._exchange_mirror(plan)
                except Exception as e:  # noqa: BLE001
                    error = e
        if code == 0:
            code = self._worst_status(error)
        if code:
            engine.rows_commit(False)
            if error is not None:
                raise error
            raise (MemoryError if code == 2 else RuntimeError)("rebalance: another rank failed; nothing was moved")
        engine.rows_commit(True, mirror)
        self._starts = list(target)
        self._generation += 1
        return moved

    def _worst_status(self, error) -> int:
        """Every rank's status, agreed by one all-reduce (max): 0 fine, 1 failed, 2 out of memory."""
        code = 0 if error is None else 2 if isinstance(error, MemoryError) else 1
        if self.world == 1:
            return code
        import torch
        from torch.distributed import ReduceOp

        dev = self._engine.comm_device() if hasattr(self._engine, "comm_device") else torch.device("cpu")
        word = torch.tensor([code], dtype=torch.int64, device=dev)
        self._dist.all_reduce(word, op=ReduceOp.MAX, group=self._group)
        return int(word.item())

    def _exchange_mirror(self, plan) -> np.ndarray:
        """This rank's new float32 host mirror: its kept rows, and the moving pieces from their ranks' mirrors
        through ``all_to_all_single`` on the communication device, in rounds of at most ``MIRROR_ROUND_BYTES``
        per pair of ranks."""
        import torch

        d = self._embedding_size
        mine = self._engine.local_rows()
        dev = torch.device("cpu")  # gloo moves device tensors through host memory anyway
        if hasattr(self._engine, "comm_device") and self._dist.get_backend(self._group) != "gloo":
            dev = self._engine.comm_device()
        send = {dst: (first, n) for dst, src, first, n in plan if src == self.rank and dst != self.rank}
        recv = {src: n for dst, src, _, n in plan if dst == self.rank and src != self.rank}
        parts = {src: [] for src in recv}
        per_round = max(1, MIRROR_ROUND_BYTES // (4 * max(d, 1)))
        rounds = -(-max([n for dst, src, _, n in plan if dst != src], default=0) // per_round)
        for r in range(rounds):
            a = r * per_round
            out_sizes = [max(0, min(recv.get(src, 0) - a, per_round)) for src in range(self.world)]
            in_sizes = [max(0, min(send.get(dst, (0, 0))[1] - a, per_round)) for dst in range(self.world)]
            chunks = [mine[send[dst][0] + a: send[dst][0] + a + in_sizes[dst]] for dst in range(self.world)
                      if in_sizes[dst]]
            data = np.concatenate(chunks) if chunks else np.zeros((0, d), np.float32)
            inp = torch.from_numpy(np.ascontiguousarray(data, np.float32)).to(dev)
            out = torch.empty((sum(out_sizes), d), dtype=torch.float32, device=dev)
            self._dist.all_to_all_single(out, inp, out_sizes, in_sizes, group=self._group)
            host = out.cpu().numpy()
            at = 0
            for src in range(self.world):
                if out_sizes[src]:
                    parts[src].append(host[at: at + out_sizes[src]])
                    at += out_sizes[src]
        rows = []
        for dst, src, first, n in plan:
            if dst == self.rank:
                rows.append(mine[first: first + n] if src == self.rank else np.concatenate(parts[src]))
        return np.concatenate(rows) if rows else np.zeros((0, d), np.float32)

    # ---- lookups -----------------------------------------------------------------------
    def _gather_and_merge(self, local, b: int, k: int):
        import torch

        if self.world == 1:
            gathered = local.view(1, -1)
        else:
            gathered = torch.empty((self.world, local.numel()), dtype=torch.uint8, device=local.device)
            self._dist.all_gather_into_tensor(gathered.view(-1), local, group=self._group)
        return self._engine.merge(gathered, self.world, b, k)

    def search_tensors(self, queries, k: int, min_score: float = 0.0, defer_check: bool = False, *, allowed=None,
                       subset=None, subsets=None, ties_low_first: bool = False):
        """SPMD lookup; returns engine tensors (items, scores, counts), replicated on every
        rank.  ``queries``: float32 [B, D] numpy array or engine-device tensor.

        The local search, the candidate all-gather and the merge are enqueued back to back
        without a host synchronisation; the (rare) "redo this query exactly" check runs at the
        end — immediately, or in ``finish()`` when ``defer_check`` is set — and repeats the
        exchange only if some rank actually had to redo a query.

        ``allowed``, ``subset``, ``subsets`` and ``ties_low_first`` as ``search_arrays`` takes them, with its
        results and errors (the queries are read on the host for their checks).  With ``exchange="peer"`` these
        lookups go through the peer exchange too, and with ``defer_check`` they are resolved by ``finish()``
        together with the plain deferred ones; a subset lookup's items are the caller's ordinals only after
        ``finish()`` then.  Otherwise they exchange over the process group and are complete on return."""
        if allowed is not None or subset is not None or subsets is not None or ties_low_first:
            if hasattr(queries, "cpu"):
                queries = queries.cpu().numpy()
            if subsets is not None:
                return self._search_arrays_subsets(queries, k, min_score, subsets, subset, allowed, ties_low_first,
                                                   tensors=True, defer_check=defer_check)
            return self._search_arrays_filtered(queries, k, min_score, subset, allowed, ties_low_first, tensors=True,
                                                defer_check=defer_check)
        n = len(self)
        b = int(queries.shape[0])
        k = max(1, min(int(k), max(n, 1)))
        lo, _ = self.local_range
        if self._peer():
            return self._group_search(queries, k, float(np.float32(min_score)), defer_check)
        deferrable = hasattr(self._engine, "finish")
        local = (self._engine.search_packed(queries, k, float(np.float32(min_score)), lo, defer_check=True)
                 if deferrable else self._engine.search_packed(queries, k, float(np.float32(min_score)), lo))
        out = self._gather_and_merge(local, b, k)
        pending = getattr(self, "_pending", None) or []
        if pending == ["group"]:
            pending = []
        if deferrable:
            pending.append((local, b, k, out))
        self._pending = pending
        if not defer_check:
            self.finish()
        return out

    def close(self) -> None:
        """Release this rank's device state (its rows and, with ``exchange="peer"``, its exchange region).
        Collective: every rank calls it.  Deferred lookups that were not finished are dropped; call ``finish()``
        first to keep them.  An engine without device state has nothing to release."""
        self._pending = []
        self._decode = []
        self._peer_masks = {}
        close = getattr(self._engine, "close", None)
        if close is not None:
            close(self._dist, self._group)

    def finish(self) -> int:
        """Resolve a deferred lookup on every rank; returns the number of queries (summed over
        ranks) that took the exact fallback.  Collective: every rank must call it."""
        import torch

        pending = getattr(self, "_pending", None)
        if not pending:
            return 0
        self._pending = []
        if pending == ["group"]:       # libtavec agrees across ranks inside tav_sharded_finish
            decode, self._decode = self._decode, []
            redone = self._engine.group_finish()
            for items, table in decode:  # merged subset positions -> the caller's ordinals, as given
                self._engine.map_items(items, table)
            return redone
        # a local failure must not leave the other ranks waiting in the collective: reduce an error
        # flag together with the count and raise on every rank
        error = None
        try:
            redone = self._engine.finish()
        except Exception as e:  # noqa: BLE001
            error, redone = e, 0
        total, failed = redone, int(error is not None)
        if self.world > 1:
            t = torch.tensor([redone, failed], dtype=torch.int32, device=pending[-1][0].device)
            self._dist.all_reduce(t, group=self._group)
            total, failed = int(t[0].item()), int(t[1].item())
        if failed:
            raise error if error is not None else RuntimeError("finish(): another rank failed its exact fallback")
        if total > 0:  # some shard corrected its candidates (in place): exchange and merge every open search again
            for local, b, k, out in pending:
                items, scores, counts = self._gather_and_merge(local, b, k)
                out[0].copy_(items), out[1].copy_(scores), out[2].copy_(counts)
        return total

    def search_arrays(self, queries: np.ndarray, k: int, min_score: float = 0.0, subset=None, allowed=None,
                      ties_low_first: bool = False, subsets=None):
        """SPMD batched lookup, replicated on every rank: items int64 [B, k], scores float32 [B, k], counts int32
        [B].  ``subset``, ``subsets``, ``allowed`` and ``ties_low_first`` as ``VectorBase.search_arrays`` takes
        them over the whole corpus (global ordinals; ``allowed`` a bool [N] mask or its packed words, or one mask
        per query: bool [B, N] or packed words [B, ceil(N / 32)]), with its results and
        errors.  With ``exchange="peer"`` such lookups go through the peer exchange (``tav_sharded_search`` /
        ``tav_sharded_search_subset``), otherwise over the process group; threshold routes (k >= rows > 8192, per-query
        subsets with k > 2048) exchange as ``search_range`` does."""
        if subsets is not None:
            return self._search_arrays_subsets(queries, k, min_score, subsets, subset, allowed, ties_low_first)
        if subset is not None or allowed is not None or ties_low_first:
            return self._search_arrays_filtered(queries, k, min_score, subset, allowed, ties_low_first)
        q = np.ascontiguousarray(queries, dtype=np.float32)
        if q.ndim == 1:
            q = q.reshape(1, -1)
        if q.shape[1] != self._embedding_size and len(self):
            raise ValueError("query width does not match the embedding size")
        if len(self) == 0 or np.isnan(np.float32(min_score)):
            return (np.full((len(q), 1), -1, np.int64), np.zeros((len(q), 1), np.float32),
                    np.zeros(len(q), np.int32))
        n = len(self)
        if k >= n > RANGE_ROUTE_MIN_ROWS and hasattr(self._engine, "range_local"):
            # every passing row, as tav_search routes it on one GPU: one threshold search, laid out [B, n]
            return as_topk_arrays(*self.search_range(q, min_score), len(q), n)
        items, scores, counts = self.search_tensors(q, k, min_score)
        return items.cpu().numpy(), scores.cpu().numpy(), counts.cpu().numpy()

    # ---- filtered and subset lookups ------------------------------------------------------
    def _peer(self) -> bool:
        """Lookups go through the engine's peer exchange (``tav_sharded_search*``)."""
        return self.exchange == "peer" and self.world > 1 and hasattr(self._engine, "group_search")

    def _group_search(self, q, k: int, floor: float, defer_check: bool, ties_low_first: bool = False, mask=None,
                      subset=None, decode=None):
        """One lookup through the peer exchange; ``decode``: the merged items are positions in this list, replaced
        by its entries now, or at ``finish()`` for a deferred lookup.  A mask that is not the one every rank
        uploaded last is uploaded first, and the ranks agree on that upload (one all-reduce) before the publish."""
        if mask is not None:
            self._agree_mask(mask, len(q))
        lo, _ = self.local_range
        try:
            out = self._engine.group_search(self._dist, self._group, self.rank, self.world, q, k, floor, lo,
                                            defer_check, ties_low_first=ties_low_first, mask=mask, subset=subset)
        except Exception:
            if defer_check:  # a deferred search that failed after its publish is open on every rank
                self._pending = ["group"]
            raise
        self._pending = ["group"] if defer_check else []
        if defer_check:
            if decode is not None:
                self._decode.append((out[0], decode))
        else:
            # a synchronous search finished every open one inside the library: decode theirs, then its own
            for items, table in self._decode:
                self._engine.map_items(items, table)
            self._decode = []
            if decode is not None:
                self._engine.map_items(out[0], decode)
        return out

    def _agree_mask(self, mask, n_queries: int) -> None:
        """Upload this block's mask for the peer exchange unless every rank uploaded it last: the upload finishes
        the deferred lookups first, and its failure on any rank raises on every rank, before anything is
        published.  A mask already agreed on adds no collective."""
        kind = "query" if np.ndim(mask[0]) == 2 else "row"
        if self._peer_masks.get(kind) == mask[1]:
            return
        self.finish()
        self._peer_masks.pop(kind, None)
        error = None
        try:
            self._engine.upload_mask(mask, n_queries)
        except Exception as e:  # noqa: BLE001
            error = e
        if self._any_failed(error is not None):
            raise error if error is not None else RuntimeError("a mask upload failed on another rank")
        self._peer_masks[kind] = mask[1]

    def _check_queries(self, queries) -> np.ndarray:
        q = np.ascontiguousarray(queries, dtype=np.float32)
        if q.ndim == 1:
            q = q.reshape(1, -1)
        if q.ndim != 2 or q.shape[1] != self._embedding_size:
            raise ValueError(f"shapes ({len(self)},{self._embedding_size}) and {tuple(np.shape(queries))} not aligned")
        return q

    def _remember(self, key, words, owner) -> None:
        if len(self._masks) > 8:
            self._masks.clear()
        self._masks[key] = (words, owner)  # keeps the owner, and so its id(), alive

    def _block_mask(self, allowed, n_queries: int):
        """(this block's packed words of ``allowed``, its cache key); errors on every rank alike.  A 2-D
        ``allowed`` (one mask per query) must have ``n_queries`` rows; it is checked on every call."""
        if np.ndim(allowed) == 2 and np.shape(allowed)[0] != n_queries:
            raise ValueError(f"query masks have {np.shape(allowed)[0]} rows for {n_queries} queries")
        key = ("allowed", id(allowed), self._generation, len(self))
        hit = self._masks.get(key)
        if hit is None:
            lo, hi = self.local_range
            self._remember(key, block_mask(allowed, len(self), lo, hi), allowed)
            hit = self._masks[key]
        return hit[0], key, allowed

    def _predicate_mask(self, predicate):
        """The predicate over this rank's rows only (global ordinals [lo, hi)), packed, cached per (predicate,
        row generation, rows).  A predicate that raises on one rank raises on every rank (one all-reduce, only
        when the mask is built)."""
        key = ("predicate", id(predicate), self._generation, len(self))
        hit = self._masks.get(key)
        if hit is None:
            lo, hi = self.local_range
            error, words = None, None
            try:
                accepted = np.fromiter((bool(predicate(i)) for i in range(lo, hi)), dtype=bool, count=hi - lo)
                words = VectorBase.pack_row_mask(accepted)
            except Exception as e:  # noqa: BLE001
                error = e
            if self._any_failed(error is not None):
                raise error if error is not None else RuntimeError("the predicate raised on another rank")
            self._remember(key, words, predicate)
            hit = self._masks[key]
        return hit[0], key, predicate

    def _any_failed(self, failed: bool) -> bool:
        if self.world == 1:
            return failed
        import torch

        dev = self._engine.comm_device() if hasattr(self._engine, "comm_device") else torch.device("cpu")
        flag = torch.tensor([int(failed)], dtype=torch.int64, device=dev)
        self._dist.all_reduce(flag, group=self._group)
        return bool(flag.item())

    def _exchange_topk(self, search, b: int, k: int, order: int):
        """The local top-k search ``search()`` (a packed buffer), the packed all-gather over the process group and
        the merge with ``tav_merge_topk_ordered``'s ``order``.  Every rank's buffer travels with a status word
        behind it, so that a local failure raises on every rank instead of leaving the others in the collective."""
        import torch

        error, local = None, None
        try:
            local = search()
        except Exception as e:  # noqa: BLE001
            error = e
        if self.world == 1:
            if error is not None:
                raise error
            return self._engine.merge_ordered(local.view(1, -1), 1, b, k, order)
        total = packed_layout(b, k)[2]
        dev = self._engine.comm_device() if hasattr(self._engine, "comm_device") else torch.device("cpu")
        send = torch.zeros(total + 8, dtype=torch.uint8, device=dev)
        if local is not None:
            send[:total].copy_(local.view(-1))
        else:
            send[total:] = 1
        gathered = torch.empty((self.world, total + 8), dtype=torch.uint8, device=dev)
        self._dist.all_gather_into_tensor(gathered.view(-1), send, group=self._group)
        if gathered[:, total:].any().item():
            raise error if error is not None else RuntimeError("a lookup failed on another rank")
        return self._engine.merge_ordered(gathered, self.world, b, k, order)

    def _as_output(self, arrays, tensors: bool):
        """(items, scores, counts): numpy arrays, or with ``tensors`` tensors on the engine's device."""
        if not tensors:
            return tuple(a.cpu().numpy() if hasattr(a, "cpu") else a for a in arrays)
        import torch

        dev = self._engine.comm_device() if hasattr(self._engine, "comm_device") else torch.device("cpu")
        return tuple(torch.from_numpy(np.ascontiguousarray(a)).to(dev) if isinstance(a, np.ndarray) else a
                     for a in arrays)

    def _search_arrays_filtered(self, queries, k, min_score, subset, allowed, ties_low_first, mask=None,
                                tensors=False, defer_check=False):
        """``VectorBase.search_arrays`` with a subset, a row mask (``allowed``, or ``mask`` = this block's words,
        key, owner as ``_block_mask`` returns them) or ties low-first, checks in its order.  ``tensors``: the
        result as engine tensors; ``defer_check`` as ``search_tensors`` takes it (the peer exchange only)."""
        q = self._check_queries(queries)
        b = len(q)
        if k < 1:
            raise ValueError("k must be >= 1")
        n_rows = len(self)
        sub = None
        if subset is not None:
            sub = subset_ordinals(subset)
            n_rows = len(sub)
        k_eff = max(1, min(k, n_rows))
        items = np.full((b, k_eff), -1, dtype=np.int64)
        scores = np.zeros((b, k_eff), dtype=np.float32)
        counts = np.zeros(b, dtype=np.int32)
        floor = _as_f32_scalar(min_score)
        # early returns and errors on replicated state only: every rank takes them together
        if b == 0 or n_rows == 0 or len(self) == 0 or np.isnan(floor):
            return self._as_output((items, scores, counts), tensors)
        if allowed is not None and sub is not None:
            raise ValueError("allowed= and subset= cannot be combined")
        if allowed is not None:
            mask = self._block_mask(allowed, b)
        if sub is not None:
            check_subset(sub, len(self))
        if k_eff >= n_rows > RANGE_ROUTE_MIN_ROWS:
            # every passing row, as tav_search routes it on one GPU: one threshold search, laid out [B, n_rows]
            csr = self._search_range_filtered(q, floor, ties_low_first, sub, mask)
            return self._as_output(as_topk_arrays(*csr, b, k_eff), tensors)
        lo, hi = self.local_range
        if self._peer():
            if sub is not None:
                positions, local_sub = subset_share(sub, len(self), lo, hi)
                out = self._group_search(q, k_eff, float(floor), defer_check, ties_low_first,
                                         subset=(local_sub, None, positions), decode=sub)
            else:
                out = self._group_search(q, k_eff, float(floor), defer_check, ties_low_first, mask=mask)
            return self._as_output(out, tensors)
        if sub is not None:
            positions, local_sub = subset_share(sub, len(self), lo, hi)
            items_t, scores_t, counts_t = self._exchange_topk(
                lambda: self._engine.search_subset_packed(q, k_eff, float(floor), local_sub, positions, ties_low_first),
                b, k_eff, 3 if ties_low_first else 2)
            self._engine.map_items(items_t, sub)  # subset positions -> the caller's ordinals, as given
        else:
            if mask is not None:
                self.finish()  # the mask upload finishes this rank's deferred searches; their exchange is redone here
            words, key, owner = mask if mask is not None else (None, None, None)
            items_t, scores_t, counts_t = self._exchange_topk(
                lambda: self._engine.search_rows_packed(q, k_eff, float(floor), lo, ties_low_first, words, key, owner),
                b, k_eff, 1 if ties_low_first else 0)
        return self._as_output((items_t, scores_t, counts_t), tensors)

    def _subsets_checked(self, queries, subsets, subset, allowed):
        """(queries, offsets, ordinals) of a per-query subsets lookup; every error is raised from replicated
        arguments, so on every rank alike and before any exchange."""
        q = self._check_queries(queries)
        if subset is not None or allowed is not None:
            raise ValueError("subsets= cannot be combined with subset= or allowed=")
        offsets, ordinals = VectorBase._subsets_csr(subsets, len(q))
        return q, offsets, ordinals

    def _search_arrays_subsets(self, queries, k, min_score, subsets, subset, allowed, ties_low_first, tensors=False,
                               defer_check=False):
        """``VectorBase.search_arrays(subsets=)`` over the whole corpus.  Each rank searches its share of every
        query's subset with flat positions as items, maps them to positions in the caller's ordinals, the ranks'
        lists are merged by position and decoded through the caller's ordinals.  ``tensors`` / ``defer_check`` as
        ``_search_arrays_filtered`` takes them."""
        if k < 1:
            raise ValueError("k must be >= 1")
        q, offsets, ordinals = self._subsets_checked(queries, subsets, subset, allowed)
        b = len(q)
        longest = int(np.diff(offsets).max()) if b else 0
        k_eff = max(1, min(k, longest))
        floor = _as_f32_scalar(min_score)
        if b == 0 or longest == 0 or len(self) == 0 or np.isnan(floor):
            return self._as_output((np.full((b, k_eff), -1, np.int64), np.zeros((b, k_eff), np.float32),
                                    np.zeros(b, np.int32)), tensors)
        check_subset(ordinals, len(self))
        check_subsets_total(len(ordinals))
        if k_eff > SUBSETS_MERGE_MAX_K:
            csr = self._search_range_subsets(q, floor, ties_low_first, offsets, ordinals)
            return self._as_output(as_topk_arrays(*csr, b, k_eff), tensors)
        lo, hi = self.local_range
        positions, local_offsets, local_ordinals = subsets_share(offsets, ordinals, len(self), lo, hi)
        if self._peer():
            out = self._group_search(q, k_eff, float(floor), defer_check, ties_low_first,
                                     subset=(local_ordinals, local_offsets, positions), decode=ordinals)
            return self._as_output(out, tensors)
        items_t, scores_t, counts_t = self._exchange_topk(
            lambda: self._engine.search_subsets_packed(q, k_eff, float(floor), local_offsets, local_ordinals, positions,
                                                       ties_low_first),
            b, k_eff, 3 if ties_low_first else 2)
        self._engine.map_items(items_t, ordinals)  # flat positions -> the caller's ordinals, as given
        return self._as_output((items_t, scores_t, counts_t), tensors)

    def _search_range_subsets(self, q, floor, ties_low_first, offsets, ordinals):
        """The threshold search of validated per-query subsets: flat positions merged, then decoded."""
        lo, hi = self.local_range
        positions, local_offsets, local_ordinals = subsets_share(offsets, ordinals, len(self), lo, hi)
        return self._range_exchange(q, floor, ties_low_first, dict(subsets=(local_offsets, local_ordinals),
                                                                   positions=positions), decode=ordinals)

    def search_range(self, queries, min_score: float = 0.0, ties_low_first: bool = False, subset=None, allowed=None,
                     subsets=None):
        """Threshold search over the whole corpus: EVERY row whose score is >= min_score, per query, as
        ``VectorBase.search_range`` returns it on one GPU — CSR numpy arrays offsets int64 [B + 1], items int64
        [T], scores float32 [T], in the library's order — replicated on every rank.  SPMD.  ``subset`` (global
        ordinals) and ``allowed`` (bool [N] or packed words, or 2-D: one mask per query) as ``VectorBase.search_range``
        takes them, with its
        errors.

        Each rank runs the threshold search on its rows; one all-gather carries every rank's offsets (and a
        status word, so that a rank's failure raises on every rank instead of leaving the others in the next
        collective), a second one every rank's hits, padded to the largest rank's total (after a one-word
        all-reduce that makes a failure to stage them raise on every rank); ``tav_merge_range`` merges them on
        every rank.  A subset search merges positions in the subset and decodes them through the caller's list
        afterwards.  With ``exchange="peer"`` the exchange is the group's range inbox instead (``group_range``:
        no process-group collective unless the inbox must be reserved or grown).  At most
        ``MAX_RANGE_RANKS`` (32) ranks: larger groups get ValueError on every rank before any exchange.
        ``subsets`` (one integer sequence per query) as ``VectorBase.search_range`` takes it."""
        if subsets is not None:
            q, offsets, ordinals = self._subsets_checked(queries, subsets, subset, allowed)
            floor = _as_f32_scalar(min_score)
            if len(q) == 0 or len(ordinals) == 0 or len(self) == 0 or np.isnan(floor):
                return np.zeros(len(q) + 1, np.int64), np.empty(0, np.int64), np.empty(0, np.float32)
            check_subset(ordinals, len(self))
            check_subsets_total(len(ordinals))
            return self._search_range_subsets(q, floor, ties_low_first, offsets, ordinals)
        if subset is not None or allowed is not None:
            q = self._check_queries(queries)
            sub = None if subset is None else subset_ordinals(subset)
            if allowed is not None and sub is not None:
                raise ValueError("allowed= and subset= cannot be combined")
            floor = _as_f32_scalar(min_score)
            n_rows = len(self) if sub is None else len(sub)
            if len(q) == 0 or n_rows == 0 or len(self) == 0 or np.isnan(floor):
                return np.zeros(len(q) + 1, np.int64), np.empty(0, np.int64), np.empty(0, np.float32)
            mask = self._block_mask(allowed, len(q)) if allowed is not None else None
            if sub is not None:
                check_subset(sub, len(self))
            return self._search_range_filtered(q, floor, ties_low_first, sub, mask)
        q = np.ascontiguousarray(queries, dtype=np.float32)
        if q.ndim == 1:
            q = q.reshape(1, -1)
        b = len(q)
        floor = _as_f32_scalar(min_score)
        # early returns on replicated state only: every rank takes them together
        if b == 0 or len(self) == 0 or np.isnan(floor):
            return np.zeros(b + 1, np.int64), np.empty(0, np.int64), np.empty(0, np.float32)
        if q.shape[1] != self._embedding_size:
            raise ValueError("query width does not match the embedding size")
        return self._range_exchange(q, floor, ties_low_first)

    def _search_range_filtered(self, q, floor, ties_low_first, sub, mask):
        """The threshold search of validated arguments with a subset (int64, in range), this block's mask, or
        neither (ties low-first alone)."""
        lo, hi = self.local_range
        if sub is not None:
            positions, local_sub = subset_share(sub, len(self), lo, hi)
            return self._range_exchange(q, floor, ties_low_first, dict(subset=local_sub, positions=positions),
                                        decode=sub)
        if mask is None:
            return self._range_exchange(q, floor, ties_low_first)
        self.finish()  # the mask upload finishes this rank's deferred searches; their exchange is redone here
        words, key, owner = mask
        return self._range_exchange(q, floor, ties_low_first, dict(mask=words, mask_key=key, mask_owner=owner),
                                    mask=mask)

    def _range_exchange(self, q, floor, ties_low_first, local_args=None, decode=None, mask=None):
        """The exchange and the merge of a threshold search whose local part is ``range_local`` with
        ``local_args``; ``decode``: merged items are positions in this list, replaced by its entries on the device;
        ``mask``: this block's mask (words, key, owner) when ``local_args`` carries one.  Through the peer exchange
        (``group_range``) when the lookups use it, otherwise over the process group."""
        import torch

        b = len(q)
        empty = (np.zeros(b + 1, np.int64), np.empty(0, np.int64), np.empty(0, np.float32))
        if self.world > MAX_RANGE_RANKS:
            raise ValueError(f"search_range merges at most {MAX_RANGE_RANKS} ranks (tav_merge_range), not {self.world}")
        local_args = local_args or {}
        lo, _ = self.local_range
        if self._peer() and hasattr(self._engine, "group_range"):
            if mask is not None:
                self._agree_mask(mask, b)
            out = self._engine.group_range(self._dist, self._group, self.rank, self.world, q, float(floor), lo,
                                           bool(ties_low_first), **local_args)
            if decode is not None:
                self._engine.map_items(out[1], decode)  # subset positions -> the caller's ordinals, as given
            return tuple(np.asarray(t.cpu().numpy() if hasattr(t, "cpu") else t) for t in out)
        error, local = None, None
        try:
            local = self._engine.range_local(q, float(floor), lo, bool(ties_low_first), **local_args)
            offsets = np.asarray(local.offsets, np.int64)
        except Exception as e:  # noqa: BLE001
            error, offsets = e, np.zeros(b + 1, np.int64)
        if self.world == 1 and decode is None:
            if error is not None:
                raise error
            total = int(offsets[-1])
            items, scores = np.empty(total, np.int64), np.empty(total, np.float32)
            local.fetch(items, scores)
            return offsets.copy(), items, scores
        try:
            dev = self._engine.comm_device() if hasattr(self._engine, "comm_device") else torch.device("cpu")
            # exchange 1: offsets [B + 1] and a status word per rank
            mine = torch.from_numpy(offsets_with_status(offsets, error is not None)).to(dev)
            flag = torch.zeros(1, dtype=torch.int64, device=dev)
            offsets_all = torch.empty((self.world, b + 2), dtype=torch.int64, device=dev)
            self._all_gather(offsets_all, mine)
            host = offsets_all.cpu().numpy()
            if host[:, -1].any():
                raise error if error is not None else RuntimeError("search_range: another rank's threshold search failed")
            totals = host[:, b]
            total = int(totals.sum())
            if total == 0:
                return empty
            # exchange 2: every rank's hits, padded to the largest total.  Staging them (two allocations and the
            # fetch) can fail on one rank; the ranks agree on that first, so nobody waits in the all-gather alone
            t_pad = range_pad(totals)
            stage_error, send = None, None
            try:
                payload = torch.empty((self.world, 12 * t_pad), dtype=torch.uint8, device=dev)
                send = pack_range_payload(local, t_pad, dev)
            except Exception as e:  # noqa: BLE001
                stage_error = e
            flag.fill_(int(stage_error is not None))
            if self.world > 1:
                self._dist.all_reduce(flag, group=self._group)
            if int(flag.item()):
                raise stage_error if stage_error is not None else RuntimeError(
                    "search_range: another rank failed to stage its hits")
            self._all_gather(payload, send)
            out = self._engine.merge_range(offsets_all, payload, self.world, b, t_pad, total, bool(ties_low_first))
            if decode is not None:
                self._engine.map_items(out[1], decode)  # subset positions -> the caller's ordinals, as given
            return tuple(np.asarray(t.cpu().numpy() if hasattr(t, "cpu") else t) for t in out)
        finally:
            if local is not None:
                local.release()

    def _all_gather(self, out, mine) -> None:
        if self.world == 1:
            out.view(-1).copy_(mine.view(-1))
        else:
            self._dist.all_gather_into_tensor(out.view(-1), mine, group=self._group)

    def fuzzy_lookup_embeddings(self, embeddings, max_hits=None, min_score=None):
        if min_score is None:
            min_score = 0.0
        if len(self) == 0:
            return [[] for _ in range(len(embeddings))]
        if max_hits == 0 and hasattr(self._engine, "range_local"):
            # every passing row (the reference's max_hits=0): CSR lists from the threshold search
            offsets, items, scores = self.search_range(embeddings, min_score)
            il, sl, ol = items.tolist(), scores.tolist(), offsets.tolist()
            return [[ScoredInt(i, s) for i, s in zip(il[ol[b]:ol[b + 1]], sl[ol[b]:ol[b + 1]])]
                    for b in range(len(ol) - 1)]
        k = VectorBase._resolve_k(max_hits, len(self))
        items, scores, counts = self.search_arrays(embeddings, k, min_score)
        il, sl, cl = items.tolist(), scores.tolist(), counts.tolist()
        return [[ScoredInt(i, s) for i, s in zip(il[b][:c], sl[b][:c])] for b, c in enumerate(cl)]

    def fuzzy_lookup_embeddings_in_subsets(self, embeddings, ordinals_of_subsets, max_hits=None, min_score=None):
        """``VectorBase.fuzzy_lookup_embeddings_in_subsets`` over the whole corpus, SPMD: element b equals
        ``fuzzy_lookup_embedding_in_subset(embeddings[b], ordinals_of_subsets[b], max_hits, min_score)``."""
        if min_score is None:
            min_score = 0.0
        q = np.asarray(embeddings, dtype=np.float32)
        if q.ndim != 2:
            raise ValueError(f"Expected 2D embeddings array, got {q.ndim}D")
        if max_hits is not None and max_hits < 0:
            raise ValueError("max_hits must be >= 0")
        if max_hits == 0:
            offsets, items, scores = self.search_range(q, min_score, subsets=ordinals_of_subsets)
            il, sl, ol = items.tolist(), scores.tolist(), offsets.tolist()
            return [[ScoredInt(i, s) for i, s in zip(il[ol[b]:ol[b + 1]], sl[ol[b]:ol[b + 1]])]
                    for b in range(len(q))]
        k = _DEFAULT_MAX_HITS if max_hits is None else max_hits
        items, scores, counts = self.search_arrays(q, k, min_score, subsets=ordinals_of_subsets)
        il, sl, cl = items.tolist(), scores.tolist(), counts.tolist()
        return [[ScoredInt(i, s) for i, s in zip(il[b][:c], sl[b][:c])] for b, c in enumerate(cl)]

    def fuzzy_lookup_embedding(self, embedding, max_hits=None, min_score=None, predicate=None):
        """``VectorBase.fuzzy_lookup_embedding`` over the whole corpus.  With a predicate: every row at or above
        min_score that satisfies it, equal scores lower ordinal first (the reference's stable sort), first
        max_hits; ``max_hits=0`` returns [].  Each rank evaluates the predicate on its own rows only, once per
        (predicate, rows) while the rows stay as they are, and the search runs with that row mask."""
        if predicate is None:
            return self.fuzzy_lookup_embeddings(np.asarray(embedding, np.float32).reshape(1, -1),
                                                max_hits, min_score)[0]
        if min_score is None:
            min_score = 0.0
        n = len(self)
        if n == 0:
            return []
        k = VectorBase._resolve_k(max_hits, n)
        if max_hits == 0:  # the reference's predicate path slices `[:0]` (vectorbase.py:201)
            return []
        mask = self._predicate_mask(predicate)
        items, scores, counts = self._search_arrays_filtered(embedding, k, min_score, None, None, True, mask=mask)
        c = int(counts[0])
        return [ScoredInt(i, s_) for i, s_ in zip(items[0, :c].tolist(), scores[0, :c].tolist())]

    def fuzzy_lookup_embedding_in_subset(self, embedding, ordinals_of_subset, max_hits=None, min_score=None):
        """``VectorBase.fuzzy_lookup_embedding_in_subset`` over the whole corpus: only the given global ordinals
        (negative ones wrap; a repeated ordinal is a separate hit), items as given, equal scores the later
        subset position first.  IndexError on every rank, before any exchange, for an ordinal out of range or a
        non-integer one."""
        if min_score is None:
            min_score = 0.0
        if len(ordinals_of_subset) == 0 or len(self) == 0:
            return []
        k = VectorBase._resolve_k(max_hits, len(ordinals_of_subset))
        q = np.asarray(embedding, dtype=np.float32)
        if q.ndim == 2 and q.shape[0] == 1:
            q = q.reshape(-1)
        if q.ndim != 1 or q.shape[0] != self._embedding_size:
            raise ValueError(f"shapes ({len(self)},{self._embedding_size}) and {tuple(np.shape(embedding))} not aligned")
        if np.isnan(np.float32(min_score)):  # `scores >= nan` is all-false in the reference
            return []
        sub = subset_ordinals(ordinals_of_subset, from_list=True)
        items, scores, counts = self._search_arrays_filtered(q, k, min_score, sub, None, False)
        c = int(counts[0])
        return [ScoredInt(i, s_) for i, s_ in zip(items[0, :c].tolist(), scores[0, :c].tolist())]
