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
results whose size is known only after the local searches: they exchange over the process group (offsets, then
the hits padded to the largest rank's total) and merge with ``tav_merge_range``.

``torch`` is plumbing here (process group, device buffers); the search, exchange and merge are
libtavec kernels.  The engine is injectable so that the host logic (partitioning, packing, gather,
offsets) is testable on CPU with the ``gloo`` backend.
"""

from __future__ import annotations

import ctypes as C

import numpy as np

from . import _capi
from .vectorbase import ScoredInt, TextEmbeddingIndexSettings, VectorBase, _as_f32_scalar, removal_ordinals

RANGE_ROUTE_MIN_ROWS = 4 * 2048  # search_arrays with k >= rows above this (4 * TAV_PASS_K) -> search_range


def shard_bounds(n_rows: int, world: int) -> list[tuple[int, int]]:
    """Rank g owns rows [g*ceil(N/G), (g+1)*ceil(N/G)) clipped to N."""
    per = -(-n_rows // world) if world > 0 else 0
    return [(min(g * per, n_rows), min((g + 1) * per, n_rows)) for g in range(world)]


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

    def group_search(self, dist, process_group, rank, world, queries, k, min_score, item_offset, defer_check):
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
        _capi.check(lib.tav_sharded_search(ix, group, C.c_void_p(queries.data_ptr()), b, k, C.c_float(min_score), flags,
                                           item_offset, C.c_void_p(items.data_ptr()), C.c_void_p(scores.data_ptr()),
                                           C.c_void_p(counts.data_ptr()), C.c_void_p(stream)))
        if defer_check:
            self._group_keep.append((queries, items, scores, counts, stream))
        return items, scores, counts

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

    # ---- threshold search (search_range) ---------------------------------------------------
    def range_local(self, queries: np.ndarray, min_score: float, item_offset: int, ties_low_first: bool):
        """``tav_range_search`` on this rank's rows (items shifted by ``item_offset``).  Returns a
        ``LocalRange``: host offsets [B + 1] now, the hits later straight into the caller's buffers.  The
        hits wait in the index between the two calls, so the base's lookup lock is held until then."""
        base = self.base
        b = len(queries)
        if self.n_local() == 0:
            return LocalRange(np.zeros(b + 1, np.int64), None, None)
        q = base._check_queries(queries)
        base._single_lock.acquire()
        try:
            lib, ix = base._ensure_device()
            flags = base._flags() & ~_capi.TAV_NO_FUSED_SCAN
            if ties_low_first:
                flags |= _capi.TAV_TIES_LOW_FIRST
            offsets = np.zeros(b + 1, np.int64)
            _capi.check(lib.tav_range_search(ix, q.ctypes.data_as(C.c_void_p), b, C.c_float(min_score), flags, None, 0,
                                             item_offset, base._range_hint, offsets.ctypes.data_as(C.c_void_p), None))
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
            ip = C.c_void_p(items.data_ptr()) if on_device else items.ctypes.data_as(C.c_void_p)
            sp = C.c_void_p(scores.data_ptr()) if on_device else scores.ctypes.data_as(C.c_void_p)
            _capi.check(lib.tav_range_fetch(ix, 0, n, ip, sp, _capi.TAV_OUTPUTS_ON_DEVICE if on_device else 0,
                                            C.c_void_p(stream) if on_device else None))

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
                 exchange: str = "peer"):
        import torch.distributed as dist

        if exchange not in ("peer", "nccl"):
            raise ValueError("exchange must be 'peer' or 'nccl'")
        self.exchange = exchange
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

    # ---- corpus ------------------------------------------------------------------------
    def __len__(self) -> int:
        return self._starts[-1]

    def __bool__(self) -> bool:
        return True

    @property
    def local_range(self) -> tuple[int, int]:
        return self._starts[self.rank], self._starts[self.rank + 1]

    def _set_bounds(self, bounds) -> None:
        self._starts = [lo for lo, _ in bounds] + [bounds[-1][1]]

    def deserialize(self, data: np.ndarray | None) -> None:
        """Bulk load: every rank passes the same global float32 [N, D] array (or a
        memory-map of it) and keeps only its own block."""
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
        self._embedding_size = rows.shape[1]
        if isinstance(rows, np.ndarray):
            self._engine.load_rows(rows)
        else:
            self._engine.adopt_tensor(rows)

    def add_embeddings(self, keys, embeddings: np.ndarray) -> None:
        """Append rows (global ordinals continue at len(self)); they join the LAST rank's
        block so that blocks stay contiguous and ordered.  ``rebalance`` evens blocks out."""
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

    def remove_embeddings(self, ordinals) -> None:
        """Remove rows by global ordinal, as ``VectorBase.remove_embeddings`` does on one GPU (``np.delete``
        semantics: integer ordinals or a boolean mask over every row; IndexError, with nothing removed, for an
        ordinal out of range).  SPMD: every rank passes the same ordinals.  Deferred lookups are finished first
        (``finish()``, collective): the local removal redoes their flagged queries on the old rows, and only
        ``finish()`` exchanges and merges the corrected candidates again.  Each rank then removes its own block's
        share and recomputes the block starts from the replicated list, without a collective; blocks may become
        uneven (a block may empty)."""
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

    # ---- lookups -----------------------------------------------------------------------
    def _gather_and_merge(self, local, b: int, k: int):
        import torch

        if self.world == 1:
            gathered = local.view(1, -1)
        else:
            gathered = torch.empty((self.world, local.numel()), dtype=torch.uint8, device=local.device)
            self._dist.all_gather_into_tensor(gathered.view(-1), local, group=self._group)
        return self._engine.merge(gathered, self.world, b, k)

    def search_tensors(self, queries, k: int, min_score: float = 0.0, defer_check: bool = False):
        """SPMD lookup; returns engine tensors (items, scores, counts), replicated on every
        rank.  ``queries``: float32 [B, D] numpy array or engine-device tensor.

        The local search, the candidate all-gather and the merge are enqueued back to back
        without a host synchronisation; the (rare) "redo this query exactly" check runs at the
        end — immediately, or in ``finish()`` when ``defer_check`` is set — and repeats the
        exchange only if some rank actually had to redo a query."""
        n = len(self)
        b = int(queries.shape[0])
        k = max(1, min(int(k), max(n, 1)))
        lo, _ = self.local_range
        if self.exchange == "peer" and self.world > 1 and hasattr(self._engine, "group_search"):
            out = self._engine.group_search(self._dist, self._group, self.rank, self.world, queries, k,
                                            float(np.float32(min_score)), lo, defer_check)
            self._pending = ["group"] if defer_check else []
            return out
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

    def finish(self) -> int:
        """Resolve a deferred lookup on every rank; returns the number of queries (summed over
        ranks) that took the exact fallback.  Collective: every rank must call it."""
        import torch

        pending = getattr(self, "_pending", None)
        if not pending:
            return 0
        self._pending = []
        if pending == ["group"]:       # libtavec agrees across ranks inside tav_sharded_finish
            return self._engine.group_finish()
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

    def search_arrays(self, queries: np.ndarray, k: int, min_score: float = 0.0):
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
            offsets, hits, hit_scores = self.search_range(q, min_score)
            counts = np.diff(offsets).astype(np.int32)
            items = np.full((len(q), n), -1, np.int64)
            scores = np.zeros((len(q), n), np.float32)
            cols = np.arange(len(hits)) - np.repeat(offsets[:-1], counts)
            rows = np.repeat(np.arange(len(q)), counts)
            items[rows, cols] = hits
            scores[rows, cols] = hit_scores
            return items, scores, counts
        items, scores, counts = self.search_tensors(q, k, min_score)
        return items.cpu().numpy(), scores.cpu().numpy(), counts.cpu().numpy()

    def search_range(self, queries, min_score: float = 0.0, ties_low_first: bool = False):
        """Threshold search over the whole corpus: EVERY row whose score is >= min_score, per query, as
        ``VectorBase.search_range`` returns it on one GPU — CSR numpy arrays offsets int64 [B + 1], items int64
        [T], scores float32 [T], in the library's order — replicated on every rank.  SPMD.

        Each rank runs the threshold search on its rows; one all-gather carries every rank's offsets (and a
        status word, so that a rank's failure raises on every rank instead of leaving the others in the next
        collective), a second one every rank's hits, padded to the largest rank's total (after a one-word
        all-reduce that makes a failure to stage them raise on every rank); ``tav_merge_range`` merges them on
        every rank.  The exchanges go through the process group whatever ``exchange`` says.  At most
        ``MAX_RANGE_RANKS`` (32) ranks: larger groups get ValueError on every rank before any exchange."""
        import torch

        q = np.ascontiguousarray(queries, dtype=np.float32)
        if q.ndim == 1:
            q = q.reshape(1, -1)
        b = len(q)
        floor = _as_f32_scalar(min_score)
        empty = (np.zeros(b + 1, np.int64), np.empty(0, np.int64), np.empty(0, np.float32))
        # early returns on replicated state only: every rank takes them together
        if b == 0 or len(self) == 0 or np.isnan(floor):
            return empty
        if q.shape[1] != self._embedding_size:
            raise ValueError("query width does not match the embedding size")
        if self.world > MAX_RANGE_RANKS:
            raise ValueError(f"search_range merges at most {MAX_RANGE_RANKS} ranks (tav_merge_range), not {self.world}")
        lo, _ = self.local_range
        error, local = None, None
        try:
            local = self._engine.range_local(q, float(floor), lo, bool(ties_low_first))
            offsets = np.asarray(local.offsets, np.int64)
        except Exception as e:  # noqa: BLE001
            error, offsets = e, np.zeros(b + 1, np.int64)
        if self.world == 1:
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
            self._dist.all_gather_into_tensor(offsets_all.view(-1), mine, group=self._group)
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
            self._dist.all_reduce(flag, group=self._group)
            if int(flag.item()):
                raise stage_error if stage_error is not None else RuntimeError(
                    "search_range: another rank failed to stage its hits")
            self._dist.all_gather_into_tensor(payload.view(-1), send, group=self._group)
            out = self._engine.merge_range(offsets_all, payload, self.world, b, t_pad, total, bool(ties_low_first))
            return tuple(np.asarray(t.cpu().numpy() if hasattr(t, "cpu") else t) for t in out)
        finally:
            if local is not None:
                local.release()

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

    def fuzzy_lookup_embedding(self, embedding, max_hits=None, min_score=None):
        return self.fuzzy_lookup_embeddings(np.asarray(embedding, np.float32).reshape(1, -1),
                                            max_hits, min_score)[0]
