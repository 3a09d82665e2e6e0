"""GPU ``VectorBase`` — same surface as ``typeagent.aitools.vectorbase.VectorBase``.

Reference: /root/reference/src/typeagent/aitools/vectorbase.py (class :82-287,
``ScoredInt`` :50-55, ``TextEmbeddingIndexSettings`` :58-79, per-model score defaults
:16-41, ``cosine_to_score`` :44-47).  Method names, argument meaning, defaults, return
types and error behaviour follow the reference; the arithmetic of the lookups runs in
libtavec's CUDA kernels (``include/tavec.h``).  A float32 host mirror of the rows is the
authoritative copy for ``serialize`` / ``get_embedding_at`` (bit-exact round trips); the
device copy (float32, or bf16 / fp16 for the tensor-core path) is derived from it lazily,
appending only the rows added since the last lookup.

Additions (not in the reference; all opt-in):
  * ``fuzzy_lookup_embeddings`` / ``search_arrays`` — batched lookups, the replacement for
    the one-query-at-a-time loops in storage/memory/reltermsindex.py:320-332 and
    storage/sqlite/reltermsindex.py:259-271;
  * ``search_range`` — threshold (range) search: every row at or above min_score, CSR results in
    one read of the rows; ``fuzzy_lookup_embeddings(max_hits=0)`` builds its lists from it;
  * ``search_arrays(..., allowed=mask)`` — predicate / post-filter pushdown as a row bitmask
    evaluated inside the kernels (vectorbase.py:191-201, storage/sqlite/messageindex.py:296-326);
  * ``search_arrays`` / ``search_range(..., subsets=)`` and ``fuzzy_lookup_embeddings_in_subsets`` — one
    batched lookup in which every query scores only its own candidate ordinals (the batched form of
    ``fuzzy_lookup_embedding_in_subset``, vectorbase.py:203-230: candidate re-ranking);
  * constructor keywords ``device``, ``storage_dtype``, ``normalize``;
  * ``devices=[...]`` — the rows in contiguous blocks over several GPUs of this process, every lookup fanned out to
    all of them and merged on the first (``multi.py``, ``tav_multi_*``);
  * ``from_device_tensor`` / ``search_device`` / ``search_range_device`` — torch tensors as device-memory
    handles (the threshold search into caller tensors, sized on the device, optionally without a host
    synchronisation).

Documented divergences: negative ``max_hits`` raises ``ValueError`` (the reference returns
an arbitrary slice); among *exactly* equal scores the order is "higher ordinal first" on
every path except the predicate path, which keeps the reference's stable "lower first".
"""

from __future__ import annotations

import ctypes as C
import threading
from array import array as _array
from collections.abc import Callable, Sequence
from dataclasses import dataclass

import numpy as np

from . import _capi

DEFAULT_MIN_SCORE = 0.85

# Repository defaults of the reference for OpenAI's embedding models (vectorbase.py:31-35).
MODEL_DEFAULT_MIN_SCORES: dict[str, float] = {
    "text-embedding-3-large": 0.74,
    "text-embedding-3-small": 0.73,
    "text-embedding-ada-002": 0.93,
}

_DEFAULT_MAX_HITS = 10  # fuzzy_lookup_embedding(max_hits=None) means 10 (vectorbase.py:170-171)


def get_default_min_score(model_name: str) -> float:
    return MODEL_DEFAULT_MIN_SCORES.get(model_name, DEFAULT_MIN_SCORE)


def cosine_to_score(cosine_similarity: np.ndarray) -> np.ndarray:
    """Host-side statement of the score scale the kernels apply: clip((x + 1) / 2, 0, 1)."""
    return np.clip((cosine_similarity + 1.0) / 2.0, 0.0, 1.0)


@dataclass
class ScoredInt:
    item: int
    score: float


class TextEmbeddingIndexSettings:
    """Same fields and defaulting rules as the reference (vectorbase.py:58-79)."""

    def __init__(
        self,
        embedding_model=None,
        min_score: float | None = None,
        max_matches: int | None = None,
        batch_size: int | None = None,
    ):
        if embedding_model is None:
            embedding_model = _create_default_embedding_model()
        self.embedding_model = embedding_model
        model_name = getattr(embedding_model, "model_name", "")
        self.min_score = min_score if min_score is not None else get_default_min_score(model_name)
        self.max_matches = max_matches if max_matches and max_matches >= 1 else None
        self.batch_size = batch_size if batch_size and batch_size >= 1 else 8


def _create_default_embedding_model():
    try:
        from typeagent.aitools.model_adapters import create_embedding_model
    except Exception as e:  # typeagent is optional; this package only replaces its VectorBase
        raise RuntimeError(
            "TextEmbeddingIndexSettings needs an embedding_model (typeagent's "
            "create_embedding_model is not importable here)"
        ) from e
    return create_embedding_model()


def removal_ordinals(ordinals, n: int) -> np.ndarray:
    """The rows ``np.delete(rows, ordinals, axis=0)`` removes from n rows, sorted and distinct (int64): integer
    ordinals (negative ones count from the end, repeats remove one row) or a boolean mask of length n.  The same
    errors as numpy: IndexError for an ordinal out of range or a non-integer array, ValueError for a mask of
    the wrong shape."""
    idx = np.asarray(ordinals)
    if idx.dtype == bool:
        if idx.ndim != 1 or len(idx) != n:
            raise ValueError("boolean array argument obj to delete must be one dimensional and match the axis "
                             f"length of {n}")
        return np.flatnonzero(idx).astype(np.int64)
    if idx.size and not np.issubdtype(idx.dtype, np.integer):
        raise IndexError("arrays used as indices must be of integer (or boolean) type")
    idx = idx.astype(np.int64, copy=False).reshape(-1)
    bad = (idx < -n) | (idx >= n)
    if bad.any():
        raise IndexError(f"index {int(idx[bad][0])} is out of bounds for axis 0 with size {n}")
    return np.unique(np.where(idx < 0, idx + n, idx))


def _as_f32_scalar(value: float) -> np.float32:
    # a Python float is a weak scalar in `scores >= min_score` (NEP 50): compared as float32
    return np.float32(value)


class VectorBase:
    """In-HBM embedding matrix with brute-force top-k lookup on an H100."""

    def __init__(
        self,
        settings: TextEmbeddingIndexSettings,
        *,
        device: int | None = None,
        storage_dtype: str = "float32",
        normalize: bool = False,
        devices: Sequence[int] | None = None,
    ):
        """``device``: the CUDA ordinal of the index (default 0).  ``devices``: CUDA ordinals (1 to 32, repeats
        allowed) to hold the rows in contiguous blocks, one per entry, every lookup searching all of them and merging
        on the first; exclusive with ``device``.  Per-query masks and subsets and the device-tensor forms are not
        available with ``devices`` (NotImplementedError)."""
        if storage_dtype not in _capi.DTYPE_CODES:
            raise ValueError(f"storage_dtype must be one of {sorted(_capi.DTYPE_CODES)}")
        self._multi = None
        if devices is not None:
            if device is not None:
                raise ValueError("device= and devices= cannot be combined")
            from .multi import MultiDevice, check_devices

            devices = check_devices(devices)
            self._multi = MultiDevice(devices, storage_dtype, normalize)
            device = devices[0]
        self.settings = settings
        self._model = settings.embedding_model
        self._embedding_size = 0
        self._device = 0 if device is None else int(device)
        self._storage_dtype = storage_dtype
        self._normalize = bool(normalize)
        # host mirror: growable float32 buffer, `_count` rows valid
        self._buf = np.empty((0, 0), dtype=np.float32)
        self._count = 0
        self._generation = 0  # bumped whenever rows are replaced rather than appended
        self._buf_is_callers = False  # _buf was handed in by deserialize(): rows never change in it
        # device side (created on first lookup)
        self._ix: C.c_void_p | None = None
        self._ix_generation = -1
        self._ix_rows = 0
        self._device_only_rows = 0  # rows living only on the device (from_device_tensor)
        self._adopted_tensor = None
        self._single_out: dict[int, tuple] = {}  # k -> reusable result arrays of fuzzy_lookup_embedding
        self._subset_buf: tuple | None = None  # (reusable int64 buffer for list subsets, its address)
        # guards the two reusable buffers above, and the index's threshold-search hits between a search and
        # their fetch (a lookup with k >= rows may be served by that engine too)
        self._single_lock = threading.Lock()
        self.force_path: str | None = None  # "scan" | "mma" | "scan2" (two-kernel scan) | None (tests / benchmarks)
        self._timing = False
        self._pending: list = []             # tensors of deferred device searches, kept alive until finish_search()
        self._mask_key = None                # identity of the row mask currently on the device
        self._mask_ref = None                # ... and the object(s) that identity belongs to (so id() cannot be recycled)
        self._qmask_key = None               # identity of the per-query masks currently on the device
        self._qmask_ref = None               # ... and the mask object itself (so its id() cannot be recycled)
        self._predicate_masks: dict = {}     # (id(predicate), generation, n) -> packed bitmask
        self._range_hint = 0                 # hits of the last search_range: the next one's capacity hint
        self._groups_key = None              # identity of the group map currently on the device
        self._groups_ref = None              # ... and the map object itself (so its id() cannot be recycled)
        self.last_redone = 0                 # queries the last search_groups redid by the grouped threshold search
        self.clear()

    # ------------------------------------------------------------------ housekeeping
    def __del__(self):
        try:
            self._drop_device()
        except Exception:
            pass

    def __len__(self) -> int:
        return self._count + self._device_only_rows

    def __bool__(self) -> bool:  # an empty index must stay truthy (vectorbase.py:111-113)
        return True

    @property
    def _vectors(self) -> np.ndarray:
        """The rows as a float32 [N, D] view of the host mirror (the reference attribute)."""
        if self._embedding_size == 0:
            return self._buf[:0].reshape(0)
        return self._buf[: self._count]

    @_vectors.setter
    def _vectors(self, value: np.ndarray) -> None:
        value = np.asarray(value, dtype=np.float32)
        if value.ndim == 2:
            self._buf = value
            self._buf_is_callers = True
            self._count = len(value)
            if value.shape[1] > 0:
                self._embedding_size = value.shape[1]
        else:
            self._buf = np.empty((0, max(self._embedding_size, 0)), dtype=np.float32)
            self._count = 0
        self._generation += 1

    # ------------------------------------------------------------------ embedding model
    async def get_embedding(self, key: str, cache: bool = True):
        if cache:
            return await self._model.get_embedding(key)
        return await self._model.get_embedding_nocache(key)

    async def get_embeddings(self, keys: list[str], cache: bool = True):
        if cache:
            return await self._model.get_embeddings(keys)
        return await self._model.get_embeddings_nocache(keys)

    # ------------------------------------------------------------------ append
    def _set_embedding_size(self, size: int) -> None:
        assert size > 0
        self._embedding_size = size
        if self._buf.ndim != 2 or self._buf.shape[1] != size:
            self._buf = np.empty((0, size), dtype=np.float32)
            self._count = 0

    def _check_width(self, width: int) -> None:
        if width != self._embedding_size:
            raise ValueError(
                f"Embedding size mismatch: expected {self._embedding_size}, got {width}"
            )

    def _append_rows(self, rows: np.ndarray) -> None:
        if self._device_only_rows:
            raise RuntimeError("this VectorBase wraps a device tensor; it cannot be appended to")
        n = len(rows)
        need = self._count + n
        if need > len(self._buf) or not self._buf.flags.writeable or not self._buf.flags.owndata:
            # amortised growth (the reference copies the whole matrix on every add, :128/:145);
            # never write into an array adopted from deserialize()
            cap = max(need, 2 * len(self._buf), 16)
            fresh = np.empty((cap, self._embedding_size), dtype=np.float32)
            fresh[: self._count] = self._buf[: self._count]
            self._buf = fresh
            self._buf_is_callers = False
        self._buf[self._count : need] = rows
        self._count = need

    def add_embedding(self, key: str | None, embedding) -> None:
        row = np.asarray(embedding, dtype=np.float32)
        if self._embedding_size == 0:
            self._set_embedding_size(len(row))
        self._check_width(len(row))
        self._append_rows(row.reshape(1, -1))
        if key is not None:
            self._model.add_embedding(key, row)

    def add_embeddings(self, keys: None | list[str], embeddings: np.ndarray) -> None:
        if embeddings.ndim != 2:
            raise ValueError(f"Expected 2D embeddings array, got {embeddings.ndim}D")
        if self._embedding_size == 0:
            self._set_embedding_size(embeddings.shape[1])
        self._check_width(embeddings.shape[1])
        self._append_rows(embeddings)
        if keys is not None:
            for key, row in zip(keys, embeddings):
                self._model.add_embedding(key, row)

    async def add_key(self, key: str, cache: bool = True) -> None:
        embedding = await self.get_embedding(key, cache=cache)
        self.add_embedding(key if cache else None, embedding)

    async def add_keys(self, keys: list[str], cache: bool = True):
        if not keys:
            return None
        embeddings = await self.get_embeddings(keys, cache=cache)
        self.add_embeddings(keys if cache else None, embeddings)
        return embeddings

    # ------------------------------------------------------------------ state
    def clear(self) -> None:
        width = self._embedding_size
        self._buf = np.empty((0, width), dtype=np.float32)
        self._count = 0
        self._generation += 1
        self._device_only_rows = 0
        self._adopted_tensor = None

    def get_embedding_at(self, pos: int):
        if 0 <= pos < self._count:
            return self._buf[pos]
        raise IndexError(f"Index {pos} out of bounds for embedding index of size {len(self)}")

    def serialize_embedding_at(self, pos: int):
        return self._buf[pos] if 0 <= pos < self._count else None

    def serialize(self) -> np.ndarray:
        return self._vectors  # a view, like the reference hands out its internal array

    def deserialize(self, data: np.ndarray | None) -> None:
        if data is None:
            self.clear()
            return
        if self._embedding_size == 0:
            if data.ndim < 2 or data.shape[0] == 0:
                self.clear()
                return
            self._embedding_size = data.shape[1]
        assert data.shape == (len(data), self._embedding_size), [data.shape, self._embedding_size]
        if data.dtype != np.float32:
            data = data.astype(np.float32)
        self._buf = data  # adopted without a copy, as the reference does
        self._buf_is_callers = True
        self._count = len(data)
        self._generation += 1
        self._device_only_rows = 0
        self._adopted_tensor = None

    # ------------------------------------------------------------------ remove / overwrite
    def _device_in_sync(self) -> bool:
        """The device holds the host mirror's rows [0, _ix_rows) (rows after that are appended at the next
        lookup; after a deserialize() the next lookup re-uploads everything)."""
        return self._ix is not None and self._ix_generation == self._generation and self._ix_rows > 0

    def _own_buffer(self) -> None:
        """Rows are about to change in place: never write into an array adopted from deserialize()."""
        if self._buf_is_callers or not self._buf.flags.writeable or not self._buf.flags.owndata:
            self._buf = np.array(self._buf[: self._count], dtype=np.float32)
            self._buf_is_callers = False

    def remove_embeddings(self, ordinals) -> None:
        """Remove rows, as ``np.delete(self.serialize(), ordinals, axis=0)`` would: integer ordinals (negative
        ones count from the end, a repeated ordinal removes one row, order does not matter) or a boolean mask of
        one entry per row; IndexError for an ordinal out of range, with nothing removed.  The surviving rows keep their order (row r becomes row r - #{removed < r}).
        The device copy is compacted on the device (``tav_remove_rows``), not re-uploaded.  Row masks and
        cached predicate masks are dropped: ordinals change meaning."""
        if self._device_only_rows:
            raise RuntimeError("this VectorBase wraps a device tensor; rows cannot be removed from it")
        n = self._count
        removed = removal_ordinals(ordinals, n)
        if removed.size == 0:
            return
        if self._multi is not None:
            if self._multi.in_sync(self._generation):
                self._multi.remove(_capi.load(), removed)
        elif self._device_in_sync():
            on_device = np.ascontiguousarray(removed[removed < self._ix_rows])
            if len(on_device):
                _capi.check(_capi.load().tav_remove_rows(self._ix, on_device.ctypes.data_as(C.c_void_p),
                                                         len(on_device), None))
                self._ix_rows -= len(on_device)
        first = int(removed[0])
        keep = np.ones(n - first, dtype=bool)
        keep[removed - first] = False
        self._own_buffer()
        tail = self._buf[first:n][keep]  # a copy: the rows move down within the same buffer
        self._buf[first : first + len(tail)] = tail
        self._count = n - len(removed)
        self._mask_key = None
        self._mask_ref = None
        self._qmask_key = None
        self._qmask_ref = None
        self._groups_key = None
        self._predicate_masks.clear()

    def _replace_rebalanced(self, rows: np.ndarray) -> None:
        """The host mirror becomes ``rows`` (float32 [n, D]) after the device rows were replaced by the same rows
        (``tav_rows_commit``).  The generation is kept: the device already holds them, and a new generation would
        upload them all again.  Row masks and cached predicate masks are dropped: ordinals changed meaning."""
        rows = np.ascontiguousarray(rows, dtype=np.float32)
        if self._embedding_size == 0 and rows.ndim == 2 and rows.shape[1] > 0:
            self._embedding_size = rows.shape[1]
        self._buf = rows
        self._buf_is_callers = False
        self._count = len(rows)
        self._ix_rows = len(rows)
        self._mask_key = None
        self._mask_ref = None
        self._qmask_key = None
        self._qmask_ref = None
        self._groups_key = None
        self._predicate_masks.clear()

    def remove_embedding_at(self, pos: int) -> None:
        if not 0 <= pos < len(self):
            raise IndexError(f"Index {pos} out of bounds for embedding index of size {len(self)}")
        self.remove_embeddings([pos])

    def set_embeddings_at(self, first: int, embeddings: np.ndarray) -> None:
        """Overwrite rows [first, first + len(embeddings)) in place (float32 [n, D]); the device rows are
        rewritten through ``tav_write_rows`` with the conversion of an append, so every lookup afterwards equals
        one on an index built from the new rows.  IndexError when the rows are not all there."""
        if self._device_only_rows:
            raise RuntimeError("this VectorBase wraps a device tensor; its rows cannot be overwritten")
        rows = np.ascontiguousarray(embeddings, dtype=np.float32)
        if rows.ndim != 2:
            raise ValueError(f"Expected 2D embeddings array, got {rows.ndim}D")
        self._check_width(rows.shape[1])
        n = len(rows)
        if first < 0 or first + n > self._count:
            raise IndexError(
                f"Index {first if first < 0 or n == 0 else first + n - 1} out of bounds for embedding index of "
                f"size {len(self)}"
            )
        if n == 0:
            return
        if self._multi is not None:
            if self._multi.in_sync(self._generation):
                self._multi.write(_capi.load(), first, rows)
        elif self._device_in_sync() and first < self._ix_rows:
            m = min(n, self._ix_rows - first)
            _capi.check(_capi.load().tav_write_rows(self._ix, first, rows.ctypes.data_as(C.c_void_p), m,
                                                    self._embedding_size, _capi.TAV_F32, 0, None))
        self._own_buffer()
        self._buf[first : first + n] = rows

    def set_embedding_at(self, pos: int, embedding) -> None:
        row = np.asarray(embedding, dtype=np.float32)
        if row.ndim != 1:
            raise ValueError(f"Expected 1D embedding, got {row.ndim}D")
        self._check_width(len(row))
        if not 0 <= pos < len(self):
            raise IndexError(f"Index {pos} out of bounds for embedding index of size {len(self)}")
        self.set_embeddings_at(pos, row.reshape(1, -1))

    # ------------------------------------------------------------------ device plumbing
    def _drop_device(self) -> None:
        if self._multi is not None and self._multi.shards is not None:
            self._multi.close(_capi.load())
        if self._ix is not None:
            lib = _capi.load()
            lib.tav_destroy(self._ix)
            self._ix = None
        self._ix_rows = 0

    def _ensure_device(self):
        """Bring the device copy up to date with the host mirror; returns (lib, handle)."""
        lib = _capi.load()
        if self._multi is not None:
            if self._multi.sync(lib, self._buf[: self._count], self._generation, self._embedding_size):
                self._mask_key = None
            return lib, None
        if self._ix is None:
            handle = C.c_void_p()
            flags = _capi.TAV_NORMALIZE if self._normalize else 0
            _capi.check(
                lib.tav_create(self._device, 0, _capi.DTYPE_CODES[self._storage_dtype], flags, 0,
                               C.byref(handle))
            )
            self._ix = handle
            self._ix_generation = -1
            self._ix_rows = 0
            if self._timing:
                _capi.check(lib.tav_set_timing(self._ix, int(self._timing)))
        if self._device_only_rows:
            return lib, self._ix
        if self._ix_generation != self._generation:
            _capi.check(lib.tav_clear(self._ix))
            if lib.tav_dim(self._ix) not in (0, self._embedding_size):
                self._drop_device()
                return self._ensure_device()
            self._ix_rows = 0
            self._ix_generation = self._generation
            self._mask_key = None
            self._qmask_key = None
            self._groups_key = None
        if self._ix_rows < self._count:
            self._mask_key = None
            self._qmask_key = None
            self._groups_key = None
            fresh = np.ascontiguousarray(self._buf[self._ix_rows : self._count])
            _capi.check(
                lib.tav_append(self._ix, fresh.ctypes.data_as(C.c_void_p), len(fresh),
                               self._embedding_size, _capi.TAV_F32, 0, None)
            )
            self._ix_rows = self._count
        return lib, self._ix

    def _flags(self) -> int:
        if self.force_path == "scan":
            return _capi.TAV_FORCE_SCAN
        if self.force_path == "scan2":
            return _capi.TAV_FORCE_SCAN | _capi.TAV_NO_FUSED_SCAN
        if self.force_path == "mma":
            return _capi.TAV_FORCE_MMA
        return 0

    # ------------------------------------------------------------------ row masks
    @staticmethod
    def pack_row_mask(allowed) -> np.ndarray:
        """bool [N] -> little-endian bit-packed uint32 words (bit r of word r // 32 = row r)."""
        bits = np.packbits(np.asarray(allowed, dtype=bool), bitorder="little")
        pad = (-len(bits)) % 4
        if pad:
            bits = np.concatenate([bits, np.zeros(pad, np.uint8)])
        return np.ascontiguousarray(bits).view(np.uint32)

    def _use_row_mask(self, lib, ix, allowed, key=None, owner=None) -> None:
        """Upload ``allowed`` (bool [N], or packed uint32 words) unless it is the mask already
        on the device.  Masks are treated as immutable: identity + row generation is the key
        (``owner``: the object whose id() a caller-made key is built on — kept alive here, as is
        ``allowed``, because the id of a collected object can be handed to a new one)."""
        n = len(self)
        if key is None:
            key = (id(allowed), self._generation, n)
        if self._mask_key == key:
            return
        self._mask_key = None
        if getattr(allowed, "dtype", None) == np.uint32:
            words = allowed
        else:
            if len(allowed) != n:
                raise ValueError(f"row mask has {len(allowed)} entries for {n} rows")
            words = self.pack_row_mask(allowed)
        if len(words) != (n + 31) // 32:
            raise ValueError(f"row mask has {len(words) * 32} bits for {n} rows")
        words = np.ascontiguousarray(words)
        if self._multi is not None:
            self._multi.set_row_mask(lib, words, n)
        else:
            _capi.check(lib.tav_set_row_mask(ix, words.ctypes.data_as(C.c_void_p), n, 0, None))
        self._mask_key = key
        self._mask_ref = (allowed, owner)

    @staticmethod
    def pack_query_masks(allowed) -> np.ndarray:
        """bool [B, N] -> little-endian bit-packed uint32 words [B, ceil(N / 32)] (row b: query b's mask, in the
        bit order of ``pack_row_mask``)."""
        bits = np.packbits(np.asarray(allowed, dtype=bool), axis=1, bitorder="little")
        pad = (-bits.shape[1]) % 4
        if pad:
            bits = np.concatenate([bits, np.zeros((len(bits), pad), np.uint8)], axis=1)
        return np.ascontiguousarray(bits).view(np.uint32)

    @staticmethod
    def _is_query_masks(allowed) -> bool:
        """A 2-D ``allowed=``: one mask per query."""
        return allowed is not None and len(getattr(allowed, "shape", np.shape(allowed))) == 2

    def _use_query_masks(self, lib, ix, allowed, n_queries: int, stream=None) -> None:
        """Upload a 2-D ``allowed`` (bool [B, N], packed uint32 [B, ceil(N / 32)], or an int32 CUDA tensor of
        those words, copied on ``stream``) unless it is the set already on the device.  Like the row mask, the
        masks are treated as immutable: identity + row generation + rows is the key."""
        n = len(self)
        words_per = (n + 31) // 32
        shape = tuple(getattr(allowed, "shape", np.shape(allowed)))
        if shape[0] != n_queries:
            raise ValueError(f"query masks have {shape[0]} rows for {n_queries} queries")
        key = (id(allowed), self._generation, n)
        if self._qmask_key == key:
            return
        self._qmask_key = None
        if getattr(allowed, "is_cuda", False):
            import torch

            if not (allowed.dtype == torch.int32 and allowed.is_contiguous()):
                raise ValueError("device query masks must be a contiguous int32 CUDA tensor of packed words")
            if allowed.device.index != self._device:
                raise ValueError(f"device query masks are on cuda:{allowed.device.index}, the index on cuda:{self._device}")
            if shape[1] != words_per:
                raise ValueError(f"query masks have {shape[1] * 32} bits for {n} rows")
            _capi.check(lib.tav_set_query_masks(ix, C.c_void_p(allowed.data_ptr()), n_queries, n, words_per, 1,
                                                C.c_void_p(stream)))
        else:
            if getattr(allowed, "dtype", None) == np.uint32:
                if shape[1] != words_per:
                    raise ValueError(f"query masks have {shape[1] * 32} bits for {n} rows")
                words = np.ascontiguousarray(allowed)
            else:
                if shape[1] != n:
                    raise ValueError(f"query masks have {shape[1]} entries for {n} rows")
                words = self.pack_query_masks(allowed)
            _capi.check(lib.tav_set_query_masks(ix, words.ctypes.data_as(C.c_void_p), n_queries, n, words_per, 0,
                                                None))
        self._qmask_key = key
        self._qmask_ref = allowed

    def _single_device_only(self, what: str) -> None:
        """NotImplementedError, before any device work, for what a multi-device index does not offer yet."""
        if self._multi is not None:
            raise NotImplementedError(f"{what} is not available on a VectorBase over several devices (devices=)")

    def _refuse_multi(self, allowed, subsets) -> None:
        if subsets is not None:
            self._single_device_only("subsets= (per-query subsets)")
        if self._is_query_masks(allowed):
            self._single_device_only("a 2-D allowed= (per-query masks)")

    def _check_queries(self, queries) -> np.ndarray:
        q = np.ascontiguousarray(queries, dtype=np.float32)
        if q.ndim == 1:
            q = q.reshape(1, -1)
        if q.ndim != 2 or q.shape[1] != self._embedding_size:
            raise ValueError(
                f"shapes ({len(self)},{self._embedding_size}) and {tuple(np.shape(queries))} not aligned"
            )
        return q

    def search_arrays(
        self,
        queries: np.ndarray,
        k: int,
        min_score: float = 0.0,
        subset: Sequence[int] | np.ndarray | None = None,
        out: tuple[np.ndarray, np.ndarray, np.ndarray] | None = None,
        allowed: np.ndarray | None = None,
        ties_low_first: bool = False,
        _mask_key=None,
        _mask_owner=None,
        subsets: Sequence[Sequence[int] | np.ndarray] | None = None,
    ) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
        """Batched lookup returning arrays: items int64 [B, k], scores float32 [B, k],
        counts int32 [B] (entries beyond counts[b] are padding: item -1, score 0).  `k` is
        clamped to the number of rows searched.  ``out`` may supply preallocated (e.g. pinned)
        C-contiguous result arrays of exactly those shapes and dtypes.  ``allowed`` (bool [N] or
        bit-packed uint32) restricts the lookup to rows whose bit is set, inside the kernels; a 2-D ``allowed``
        (bool [B, N] or bit-packed uint32 [B, ceil(N / 32)]) gives every query its own mask, in one batched
        search; ``ties_low_first`` orders exactly equal scores by ascending ordinal (row-scan path).
        ``subsets`` (B one-dimensional integer sequences) gives every query its own subset, in one batched
        search: row b equals the one-query search with ``subset=subsets[b]``; `k` is clamped to the longest."""
        self._refuse_multi(allowed, subsets)
        q = self._check_queries(queries)
        b = len(q)
        if k < 1:
            raise ValueError("k must be >= 1")
        n_rows = len(self)
        sub = None
        csr = None
        if subsets is not None:
            if subset is not None or allowed is not None:
                raise ValueError("subsets= cannot be combined with subset= or allowed=")
            csr = self._subsets_csr(subsets, b)
            n_rows = int(np.diff(csr[0]).max()) if b else 0
        elif subset is not None:
            sub = np.ascontiguousarray(subset)
            if sub.size and not np.issubdtype(sub.dtype, np.integer):
                raise IndexError("arrays used as indices must be of integer (or boolean) type")
            sub = sub.astype(np.int64, copy=False).reshape(-1)
            n_rows = len(sub)
        k_eff = max(1, min(k, n_rows))
        if out is not None:
            items, scores, counts = out
            ok = (items.shape == (b, k_eff) and items.dtype == np.int64 and items.flags.c_contiguous
                  and scores.shape == (b, k_eff) and scores.dtype == np.float32 and scores.flags.c_contiguous
                  and counts.shape == (b,) and counts.dtype == np.int32 and counts.flags.c_contiguous)
            if not ok:
                raise ValueError(f"out arrays must be int64/float32 [{b},{k_eff}] and int32 [{b}], C-contiguous")
            counts[:] = 0
        else:
            items = np.full((b, k_eff), -1, dtype=np.int64)
            scores = np.zeros((b, k_eff), dtype=np.float32)
            counts = np.zeros(b, dtype=np.int32)
        floor = _as_f32_scalar(min_score)
        if b == 0 or n_rows == 0 or len(self) == 0 or np.isnan(floor):
            return items, scores, counts
        lib, ix = self._ensure_device()
        if csr is not None:
            offsets, ordinals = csr
            # the hits pass through the index's threshold-search buffers
            with self._single_lock:
                _capi.check(
                    lib.tav_search_subsets(
                        ix, q.ctypes.data_as(C.c_void_p), b, k_eff, C.c_float(float(floor)),
                        _capi.TAV_TIES_LOW_FIRST if ties_low_first else 0, offsets.ctypes.data_as(C.c_void_p),
                        ordinals.ctypes.data_as(C.c_void_p), items.ctypes.data_as(C.c_void_p),
                        scores.ctypes.data_as(C.c_void_p), counts.ctypes.data_as(C.c_void_p), None,
                    )
                )
            return items, scores, counts
        flags = self._flags()
        if allowed is not None:
            if sub is not None:
                raise ValueError("allowed= and subset= cannot be combined")
            if self._is_query_masks(allowed):
                self._use_query_masks(lib, ix, allowed, b)
                flags |= _capi.TAV_USE_QUERY_MASKS
            else:
                self._use_row_mask(lib, ix, allowed, _mask_key, _mask_owner)
                flags |= _capi.TAV_USE_ROW_MASK
        if ties_low_first:
            flags |= _capi.TAV_TIES_LOW_FIRST
        with self._single_lock:
            if self._multi is not None:
                self._multi.topk(lib, q, k_eff, floor, flags, sub, items, scores, counts)
                return items, scores, counts
            _capi.check(
                lib.tav_search(
                    ix, q.ctypes.data_as(C.c_void_p), b, k_eff, C.c_float(float(floor)), flags,
                    sub.ctypes.data_as(C.c_void_p) if sub is not None else None,
                    len(sub) if sub is not None else 0, 0,
                    items.ctypes.data_as(C.c_void_p), scores.ctypes.data_as(C.c_void_p),
                    counts.ctypes.data_as(C.c_void_p), None,
                )
            )
        return items, scores, counts

    def search_range(
        self,
        queries: np.ndarray,
        min_score: float = 0.0,
        subset: Sequence[int] | np.ndarray | None = None,
        allowed: np.ndarray | None = None,
        ties_low_first: bool = False,
        subsets: Sequence[Sequence[int] | np.ndarray] | None = None,
    ) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
        """Threshold (range) search: EVERY row whose score is >= min_score, per query, in one read of
        the rows.  Returns CSR arrays: offsets int64 [B + 1], items int64 [T], scores float32 [T];
        query b's hits are items[offsets[b]:offsets[b + 1]], in the library's order (score descending,
        equal scores higher ordinal first, or lower first with ``ties_low_first``).  ``subset``, ``subsets`` and
        ``allowed`` (1-D, or 2-D: one mask per query) as in ``search_arrays``.  Batches run on the tensor cores (16-bit storage, or float32
        through its fp16 planes), like ``search_arrays``.  The previous call's total sizes the device buffers."""
        self._refuse_multi(allowed, subsets)
        q = self._check_queries(queries)
        b = len(q)
        n_rows = len(self)
        sub = None
        if subsets is not None:
            if subset is not None or allowed is not None:
                raise ValueError("subsets= cannot be combined with subset= or allowed=")
            offsets_in, ordinals = self._subsets_csr(subsets, b)
            offsets = np.zeros(b + 1, dtype=np.int64)
            floor = _as_f32_scalar(min_score)
            if b == 0 or len(ordinals) == 0 or len(self) == 0 or np.isnan(floor):
                return offsets, np.empty(0, np.int64), np.empty(0, np.float32)
            with self._single_lock:
                lib, ix = self._ensure_device()
                _capi.check(
                    lib.tav_range_search_subsets(
                        ix, q.ctypes.data_as(C.c_void_p), b, C.c_float(float(floor)),
                        _capi.TAV_TIES_LOW_FIRST if ties_low_first else 0, offsets_in.ctypes.data_as(C.c_void_p),
                        ordinals.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p), None,
                    )
                )
                return offsets, *self._range_fetch(lib, ix, int(offsets[-1]))
        if subset is not None:
            sub = np.ascontiguousarray(subset)
            if sub.size and not np.issubdtype(sub.dtype, np.integer):
                raise IndexError("arrays used as indices must be of integer (or boolean) type")
            sub = sub.astype(np.int64, copy=False).reshape(-1)
            n_rows = len(sub)
        if allowed is not None and sub is not None:
            raise ValueError("allowed= and subset= cannot be combined")
        offsets = np.zeros(b + 1, dtype=np.int64)
        floor = _as_f32_scalar(min_score)
        if b == 0 or n_rows == 0 or len(self) == 0 or np.isnan(floor):
            return offsets, np.empty(0, np.int64), np.empty(0, np.float32)
        # the hits wait in the index's buffers between the two calls: no other lookup of this object may
        # search in between (ctypes releases the GIL)
        with self._single_lock:
            return self._search_range_locked(q, floor, sub, allowed, ties_low_first, offsets)

    def _search_range_locked(self, q, floor, sub, allowed, ties_low_first, offsets):
        b = len(q)
        lib, ix = self._ensure_device()
        flags = self._flags() & ~_capi.TAV_NO_FUSED_SCAN
        if self._is_query_masks(allowed):
            self._use_query_masks(lib, ix, allowed, b)
            flags |= _capi.TAV_USE_QUERY_MASKS
        elif allowed is not None:
            self._use_row_mask(lib, ix, allowed)
            flags |= _capi.TAV_USE_ROW_MASK
        if ties_low_first:
            flags |= _capi.TAV_TIES_LOW_FIRST
        if self._multi is not None:
            _, items, scores = self._multi.range(lib, q, floor, flags, sub, self._range_hint, offsets)
            self._range_hint = int(offsets[-1])
            return offsets, items, scores
        _capi.check(
            lib.tav_range_search(
                ix, q.ctypes.data_as(C.c_void_p), b, C.c_float(float(floor)), flags,
                sub.ctypes.data_as(C.c_void_p) if sub is not None else None,
                len(sub) if sub is not None else 0, 0, self._range_hint,
                offsets.ctypes.data_as(C.c_void_p), None,
            )
        )
        total = int(offsets[-1])
        items, scores = self._range_fetch(lib, ix, total)
        self._range_hint = total
        return offsets, items, scores

    @staticmethod
    def _range_fetch(lib, ix, total: int) -> tuple[np.ndarray, np.ndarray]:
        """The `total` hits of the index's last threshold search (the caller holds ``_single_lock``)."""
        items = np.empty(total, dtype=np.int64)
        scores = np.empty(total, dtype=np.float32)
        if total:
            _capi.check(lib.tav_range_fetch(ix, 0, total, items.ctypes.data_as(C.c_void_p),
                                            scores.ctypes.data_as(C.c_void_p), 0, None))
        return items, scores

    @staticmethod
    def _subsets_csr(subsets, n_queries: int) -> tuple[np.ndarray, np.ndarray]:
        """B one-dimensional integer sequences -> (offsets int64 [B + 1], ordinals int64 [T]), the layout of
        ``tav_search_subsets``; ValueError when their count is not B, IndexError for a non-integer ordinal."""
        if len(subsets) != n_queries:
            raise ValueError(f"{len(subsets)} subsets for {n_queries} queries")
        parts = []
        for s in subsets:
            a = np.asarray(s)
            if a.size and not np.issubdtype(a.dtype, np.integer):
                raise IndexError("arrays used as indices must be of integer (or boolean) type")
            parts.append(a.astype(np.int64, copy=False).reshape(-1))
        offsets = np.zeros(n_queries + 1, dtype=np.int64)
        np.cumsum([len(p) for p in parts], out=offsets[1:])
        ordinals = np.concatenate(parts) if parts else np.empty(0, np.int64)
        return offsets, np.ascontiguousarray(ordinals, dtype=np.int64)

    def enable_timing(self, enabled: bool = True, main_only: bool = False) -> None:
        """Record CUDA events around the kernels of subsequent lookups (see ``last_timing``);
        ``main_only``: just the dominant kernel and the whole search (cheaper)."""
        self._timing = (2 if main_only else 1) if enabled else 0
        if self._ix is not None:
            _capi.check(_capi.load().tav_set_timing(self._ix, self._timing))

    def last_timing(self) -> dict:
        """Path, launch count and — after ``enable_timing()`` — device times of the last lookup
        (CUDA events inside libtavec; ``scan_ms`` / ``total_ms`` are -1 when timing is off)."""
        lib = _capi.load()
        scan, total = C.c_float(0), C.c_float(0)
        launches, path = C.c_int(0), C.c_int(0)
        _capi.check(lib.tav_last_timing(self._ix, C.byref(scan), C.byref(total), C.byref(launches),
                                        C.byref(path)))
        ms = (C.c_float * 64)()
        kinds = (C.c_int * 64)()
        n = C.c_int(0)
        _capi.check(lib.tav_timing_breakdown(self._ix, ms, kinds, 64, C.byref(n)))
        names = {0: "main", 1: "sample", 2: "aux"}
        breakdown = [(names.get(kinds[i], "?"), ms[i]) for i in range(min(n.value, 64))]
        return {"scan_ms": scan.value, "total_ms": total.value, "launches": launches.value,
                "path": {1: "scan", 2: "mma", 3: "mma_split"}.get(path.value, "none"), "kernels": breakdown}

    # ------------------------------------------------------------------ grouped lookups
    def _check_groups(self, groups):
        """``groups`` -> what ``tav_set_row_groups`` takes: a contiguous int32 array, or the contiguous int32 CUDA
        tensor itself (its values are checked on the device).  ValueError for a wrong length, a non-integer dtype,
        a shape other than 1-D or a value outside [0, 2^31)."""
        n = len(self)
        if getattr(groups, "is_cuda", False):
            import torch

            if not (groups.dtype == torch.int32 and groups.dim() == 1 and groups.is_contiguous()):
                raise ValueError("device groups must be a contiguous 1-D int32 CUDA tensor")
            if groups.device.index != self._device:
                raise ValueError(f"device groups are on cuda:{groups.device.index}, the index on cuda:{self._device}")
            if groups.shape[0] != n:
                raise ValueError(f"groups has {groups.shape[0]} entries for {n} rows")
            return groups
        a = np.asarray(groups)
        if a.ndim != 1:
            raise ValueError(f"groups must be one-dimensional, not of shape {a.shape}")
        if len(a) != n:
            raise ValueError(f"groups has {len(a)} entries for {n} rows")
        if a.size == 0:
            return np.zeros(0, dtype=np.int32)
        if not np.issubdtype(a.dtype, np.integer):
            raise ValueError(f"groups must be integers, not {a.dtype}")
        if int(a.min()) < 0 or int(a.max()) >= 2**31:
            raise ValueError("groups must lie in [0, 2^31)")
        return np.ascontiguousarray(a, dtype=np.int32)

    def _groups_arg(self, groups):
        """(cache key, checked map or None when it is the map on the device): the checks run before any device work."""
        key = (id(groups), self._generation, len(self))
        return key, None if key == self._groups_key else self._check_groups(groups)

    def _use_groups(self, lib, ix, groups, key, checked) -> None:
        """Upload the group map unless it is the one on the device (identity + row generation + rows, as masks)."""
        if self._groups_key == key:
            return
        self._groups_key = None
        g = self._check_groups(groups) if checked is None else checked
        if getattr(g, "is_cuda", False):
            import torch

            stream = torch.cuda.current_stream(g.device).cuda_stream
            _capi.check(lib.tav_set_row_groups(ix, C.c_void_p(g.data_ptr()), len(self), 1, C.c_void_p(stream)))
        else:
            _capi.check(lib.tav_set_row_groups(ix, g.ctypes.data_as(C.c_void_p), len(self), 0, None))
        self._groups_key = key
        self._groups_ref = groups

    def _group_flags(self, lib, ix, allowed, ties_low_first: bool, n_queries: int) -> int:
        flags = self._flags() & ~_capi.TAV_NO_FUSED_SCAN
        if self._is_query_masks(allowed):
            self._use_query_masks(lib, ix, allowed, n_queries)
            flags |= _capi.TAV_USE_QUERY_MASKS
        elif allowed is not None:
            self._use_row_mask(lib, ix, allowed)
            flags |= _capi.TAV_USE_ROW_MASK
        if ties_low_first:
            flags |= _capi.TAV_TIES_LOW_FIRST
        return flags

    def search_groups(
        self,
        queries: np.ndarray,
        k: int,
        groups,
        min_score: float = 0.0,
        allowed: np.ndarray | None = None,
        ties_low_first: bool = False,
    ) -> tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
        """Grouped top-k: the k best groups of rows per query, each scored by its best row (its leader).
        ``groups`` gives the group of every row (a 1-D integer array or sequence of ``len(self)`` values in
        [0, 2^31), or a contiguous int32 CUDA tensor on the index's device); it is uploaded once and reused while
        the same object is passed and the rows do not change.  Row b equals the first occurrence of every group in
        row b of ``search_range`` (same ``min_score``, ``allowed``, ``ties_low_first``), cut to k.  Returns group ids
        int64 [B, k], scores float32 [B, k], leader rows int64 [B, k] and counts int32 [B]; padding is group -1,
        score 0, row -1.  `k` is clamped to the number of rows.  ``last_redone`` holds the number of queries whose
        top rows held fewer than k groups and were answered by the grouped threshold search."""
        self._single_device_only("search_groups")
        q = self._check_queries(queries)
        b = len(q)
        if k < 1:
            raise ValueError("k must be >= 1")
        key, checked = self._groups_arg(groups)
        n = len(self)
        k_eff = max(1, min(k, n))
        group_ids = np.full((b, k_eff), -1, dtype=np.int64)
        scores = np.zeros((b, k_eff), dtype=np.float32)
        rows = np.full((b, k_eff), -1, dtype=np.int64)
        counts = np.zeros(b, dtype=np.int32)
        self.last_redone = 0
        floor = _as_f32_scalar(min_score)
        if b == 0 or n == 0 or np.isnan(floor):
            return group_ids, scores, rows, counts
        redone = C.c_int(0)
        with self._single_lock:  # the leaders pass through the index's threshold-search buffers
            lib, ix = self._ensure_device()
            self._use_groups(lib, ix, groups, key, checked)
            flags = self._group_flags(lib, ix, allowed, ties_low_first, b)
            _capi.check(
                lib.tav_search_groups(
                    ix, q.ctypes.data_as(C.c_void_p), b, k_eff, C.c_float(float(floor)), flags,
                    group_ids.ctypes.data_as(C.c_void_p), scores.ctypes.data_as(C.c_void_p),
                    rows.ctypes.data_as(C.c_void_p), counts.ctypes.data_as(C.c_void_p), None, C.byref(redone),
                )
            )
        self.last_redone = redone.value
        return group_ids, scores, rows, counts

    def search_range_groups(
        self,
        queries: np.ndarray,
        groups,
        min_score: float = 0.0,
        allowed: np.ndarray | None = None,
        ties_low_first: bool = False,
    ) -> tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
        """Grouped threshold search: every group with a row at or above ``min_score``, per query, each once, in
        the order of its leader (its first row in ``search_range``'s list).  ``groups``, ``allowed`` and
        ``ties_low_first`` as in ``search_groups``.  Returns CSR arrays offsets int64 [B + 1], group ids int64 [T],
        scores float32 [T] and leader rows int64 [T]."""
        self._single_device_only("search_range_groups")
        q = self._check_queries(queries)
        b = len(q)
        key, checked = self._groups_arg(groups)
        offsets = np.zeros(b + 1, dtype=np.int64)
        floor = _as_f32_scalar(min_score)
        if b == 0 or len(self) == 0 or np.isnan(floor):
            return offsets, np.empty(0, np.int64), np.empty(0, np.float32), np.empty(0, np.int64)
        with self._single_lock:  # the leaders wait in the index's buffers until they are fetched
            lib, ix = self._ensure_device()
            self._use_groups(lib, ix, groups, key, checked)
            flags = self._group_flags(lib, ix, allowed, ties_low_first, b)
            _capi.check(
                lib.tav_range_search_groups(ix, q.ctypes.data_as(C.c_void_p), b, C.c_float(float(floor)), flags,
                                            self._range_hint, offsets.ctypes.data_as(C.c_void_p), None)
            )
            total = int(offsets[-1])
            group_ids = np.empty(total, dtype=np.int64)
            scores = np.empty(total, dtype=np.float32)
            rows = np.empty(total, dtype=np.int64)
            if total:
                _capi.check(lib.tav_range_fetch_groups(ix, 0, total, group_ids.ctypes.data_as(C.c_void_p),
                                                       scores.ctypes.data_as(C.c_void_p),
                                                       rows.ctypes.data_as(C.c_void_p), 0, None))
        return offsets, group_ids, scores, rows

    def fuzzy_lookup_embedding_grouped(
        self,
        embedding,
        groups,
        max_hits: int | None = None,
        min_score: float | None = None,
    ) -> list[ScoredInt]:
        """``fuzzy_lookup_embedding`` over groups of rows (messages made of chunks): the ``max_hits`` best groups,
        each as ``ScoredInt(group, score of its best row)``, exactly (see ``search_groups``).  The defaults follow
        ``fuzzy_lookup_embedding``: ``max_hits=None`` means 10, ``0`` every group; ``min_score=None`` means 0."""
        self._single_device_only("fuzzy_lookup_embedding_grouped")
        if min_score is None:
            min_score = 0.0
        n = len(self)
        k = self._resolve_k(max_hits, n)
        if n == 0:
            self._check_groups(groups)
            return []
        group_ids, scores, _, counts = self.search_groups(embedding, k, groups, min_score)
        return [ScoredInt(int(group_ids[0, i]), float(scores[0, i])) for i in range(int(counts[0]))]

    # ------------------------------------------------------------------ lookups
    @staticmethod
    def _resolve_k(max_hits: int | None, n_rows: int) -> int:
        if max_hits is None:
            return _DEFAULT_MAX_HITS
        if max_hits < 0:
            raise ValueError("max_hits must be >= 0")
        if max_hits == 0:  # reference quirk: argpartition(x, -0)[-0:] is everything that passes
            return max(n_rows, 1)
        return max_hits

    def fuzzy_lookup_embedding(
        self,
        embedding,
        max_hits: int | None = None,
        min_score: float | None = None,
        predicate: Callable[[int], bool] | None = None,
    ) -> list[ScoredInt]:
        if min_score is None:
            min_score = 0.0
        n = len(self)
        if n == 0:
            return []
        k = self._resolve_k(max_hits, n)
        if predicate is not None:
            if max_hits == 0:  # the reference's predicate path slices `[:0]` (vectorbase.py:201)
                return []
            return self._lookup_with_predicate(embedding, k, min_score, predicate)
        return self._lookup_one(embedding, k, min_score, None)

    def _lookup_one(self, embedding, k: int, min_score: float, subset) -> list[ScoredInt]:
        # the reused result / subset buffers belong to one lookup at a time (ctypes releases the GIL in tav_search)
        with self._single_lock:
            return self._lookup_one_locked(embedding, k, min_score, subset)

    def _lookup_one_locked(self, embedding, k: int, min_score: float, subset) -> list[ScoredInt]:
        """Single-lookup latency path (tools/benchmark_vectorbase.py:97-158 is this call): one host
        query straight into ``tav_search`` — which serves it with ONE kernel launch, the query riding
        in the kernel parameters — with reused result buffers and cached ctypes pointers; none of
        ``search_arrays``' generality (the hits never escape: they are copied into ScoredInt objects)."""
        q = embedding
        if not (type(q) is np.ndarray and q.dtype == np.float32 and q.ndim == 1 and q.flags.c_contiguous):
            q = np.ascontiguousarray(embedding, dtype=np.float32)
            if q.ndim != 1:
                q = q.reshape(-1) if q.ndim == 2 and q.shape[0] == 1 else q
        if q.ndim != 1 or q.shape[0] != self._embedding_size:
            raise ValueError(
                f"shapes ({len(self)},{self._embedding_size}) and {tuple(np.shape(embedding))} not aligned"
            )
        floor = float(np.float32(min_score))
        if floor != floor:  # `scores >= nan` is all-false in the reference
            return []
        n_rows = len(self)
        sub_ptr, sub_len, sub = None, 0, None
        if subset is not None:
            if type(subset) is list:
                pack = _capi.pack_int_list()
                if pack is not None:                 # CPython-API walk of the list: 3.7 us per 1000 ordinals
                    buf = self._subset_buf           # (int64 array, its address): reused across calls
                    if buf is None or len(buf[0]) < len(subset):
                        arr = np.empty(max(4096, 2 * len(subset)), np.int64)
                        buf = self._subset_buf = (arr, arr.ctypes.data)
                    got = pack(subset, buf[1], len(buf[0]))
                    if got >= 0:
                        sub, sub_ptr, n_rows, sub_len = buf[0], buf[1], got, got
                if sub is None:
                    try:
                        sub = np.frombuffer(_array("q", subset), dtype=np.int64)   # 18 us; np.asarray(list): 29 us
                    except (TypeError, OverflowError):
                        sub = None
            if sub is None:
                sub = np.ascontiguousarray(subset)
                if sub.size and not np.issubdtype(sub.dtype, np.integer):
                    raise IndexError("arrays used as indices must be of integer (or boolean) type")
                sub = np.ascontiguousarray(sub.astype(np.int64, copy=False).reshape(-1))
            if sub_ptr is None:
                n_rows = sub_len = len(sub)
                sub_ptr = sub.ctypes.data
        k_eff = max(1, min(k, n_rows))
        out = self._single_out.get(k_eff)
        if out is None:
            if len(self._single_out) > 8:
                self._single_out.clear()
            items, scores, counts = np.empty((1, k_eff), np.int64), np.empty((1, k_eff), np.float32), np.empty(1, np.int32)
            out = self._single_out[k_eff] = (items, scores, counts, items.ctypes.data, scores.ctypes.data,
                                             counts.ctypes.data)
        items, scores, counts, ip, sp, cp = out
        lib, ix = self._ensure_device()
        try:                                 # 0.5 us; ndarray.ctypes.data builds a helper object (1.5 us)
            qp = C.addressof(C.c_char.from_buffer(q))
        except (TypeError, ValueError):      # read-only query buffer
            qp = q.ctypes.data
        if self._multi is not None:
            self._multi.topk(lib, q.reshape(1, -1), k_eff, floor, self._flags(),
                             sub[:sub_len] if sub is not None else None, items, scores, counts)
        else:
            rc = lib.tav_search(ix, qp, 1, k_eff, floor, self._flags(), sub_ptr, sub_len, 0, ip, sp, cp, None)
            if rc < 0:
                _capi.check(rc)
        c = int(counts[0])
        return [ScoredInt(i, s_) for i, s_ in zip(items[0, :c].tolist(), scores[0, :c].tolist())]

    _PREDICATE_MASK_ROWS = 65536  # below this many rows the predicate is evaluated up front

    def _predicate_mask(self, predicate) -> tuple[np.ndarray, tuple]:
        """The predicate over every row, bit-packed and cached per (predicate, rows)."""
        n = len(self)
        key = (id(predicate), self._generation, n)
        hit = self._predicate_masks.get(key)
        if hit is None:
            if len(self._predicate_masks) > 8:
                self._predicate_masks.clear()
            accepted = np.fromiter((bool(predicate(i)) for i in range(n)), dtype=bool, count=n)
            hit = self._predicate_masks[key] = (self.pack_row_mask(accepted), predicate)  # keeps id() alive
        return hit[0], key

    def clear_predicate_cache(self) -> None:
        """Forget the cached predicate bitmasks (and the mask on the device): for predicates whose
        answer changed since they were last used."""
        self._predicate_masks.clear()
        self._mask_key = None
        self._mask_ref = None

    def _lookup_with_predicate(self, embedding, k, min_score, predicate) -> list[ScoredInt]:
        """Reference semantics (vectorbase.py:191-201): every row at or above min_score that
        satisfies the predicate, stable-sorted by descending score, first k.

        The predicate is pushed down as a row bitmask tested inside the scan kernel (one search,
        exact reference order including ties: equal scores -> lower ordinal first).  Small indexes
        evaluate the predicate over all rows at once (cached); large ones first try one unfiltered
        page of hits — enough whenever min_score or the predicate is not very selective — and only
        then build the mask (O(N) predicate calls, what the reference itself spends at
        min_score = 0)."""
        n = len(self)
        if n > self._PREDICATE_MASK_ROWS and (id(predicate), self._generation, n) not in self._predicate_masks:
            fetch = min(n, max(4 * k, 64))
            items, scores, counts = self.search_arrays(embedding, fetch, min_score)
            c = int(counts[0])
            rows, vals = items[0, :c], scores[0, :c]
            order = np.lexsort((rows, -vals.astype(np.float64)))  # score desc, ordinal asc
            accepted = [
                ScoredInt(int(rows[j]), float(vals[j])) for j in order if predicate(int(rows[j]))
            ]
            exhausted = c < fetch or fetch >= n
            # rows tied with the last fetched score may continue beyond the page
            settled = len(accepted) >= k and (c == 0 or accepted[k - 1].score > float(vals[c - 1]))
            if exhausted or settled:
                return accepted[:k]
        mask, key = self._predicate_mask(predicate)
        items, scores, counts = self.search_arrays(embedding, k, min_score, allowed=mask,
                                                   ties_low_first=True, _mask_key=key, _mask_owner=predicate)
        c = int(counts[0])
        return [ScoredInt(i, s_) for i, s_ in zip(items[0, :c].tolist(), scores[0, :c].tolist())]

    def fuzzy_lookup_embedding_in_subset(
        self,
        embedding,
        ordinals_of_subset: list[int],
        max_hits: int | None = None,
        min_score: float | None = None,
    ) -> list[ScoredInt]:
        if min_score is None:
            min_score = 0.0
        if len(ordinals_of_subset) == 0 or len(self) == 0:
            return []
        k = self._resolve_k(max_hits, len(ordinals_of_subset))
        return self._lookup_one(embedding, k, min_score, ordinals_of_subset)

    def fuzzy_lookup_embeddings(
        self,
        embeddings: np.ndarray,
        max_hits: int | None = None,
        min_score: float | None = None,
    ) -> list[list[ScoredInt]]:
        """One batched GPU search for many query embeddings ([B, D]); element b equals
        ``fuzzy_lookup_embedding(embeddings[b], max_hits, min_score)``."""
        if min_score is None:
            min_score = 0.0
        q = np.asarray(embeddings, dtype=np.float32)
        if q.ndim != 2:
            raise ValueError(f"Expected 2D embeddings array, got {q.ndim}D")
        if len(self) == 0:
            return [[] for _ in range(len(q))]
        k = self._resolve_k(max_hits, len(self))
        if max_hits == 0:
            # every passing row: CSR lists from the threshold search instead of [B, N] arrays
            offsets, items, scores = self.search_range(q, min_score)
            il, sl, ol = items.tolist(), scores.tolist(), offsets.tolist()
            return [[ScoredInt(i, s) for i, s in zip(il[ol[b]:ol[b + 1]], sl[ol[b]:ol[b + 1]])]
                    for b in range(len(q))]
        items, scores, counts = self.search_arrays(q, k, min_score)
        # three bulk conversions, then plain list slices: 1.6x faster than slicing the arrays per query
        il, sl, cl = items.tolist(), scores.tolist(), counts.tolist()
        return [[ScoredInt(i, s) for i, s in zip(il[b][:c], sl[b][:c])] for b, c in enumerate(cl)]

    def fuzzy_lookup_embeddings_in_subsets(
        self,
        embeddings: np.ndarray,
        ordinals_of_subsets: Sequence[Sequence[int]],
        max_hits: int | None = None,
        min_score: float | None = None,
    ) -> list[list[ScoredInt]]:
        """One batched GPU search in which query b scores only ``ordinals_of_subsets[b]``; element b equals
        ``fuzzy_lookup_embedding_in_subset(embeddings[b], ordinals_of_subsets[b], max_hits, min_score)``."""
        self._single_device_only("fuzzy_lookup_embeddings_in_subsets (per-query subsets)")
        if min_score is None:
            min_score = 0.0
        q = np.asarray(embeddings, dtype=np.float32)
        if q.ndim != 2:
            raise ValueError(f"Expected 2D embeddings array, got {q.ndim}D")
        if max_hits is not None and max_hits < 0:
            raise ValueError("max_hits must be >= 0")
        if max_hits == 0:
            # every passing entry: CSR lists from the threshold form instead of [B, longest] arrays
            offsets, items, scores = self.search_range(q, min_score, subsets=ordinals_of_subsets)
            il, sl, ol = items.tolist(), scores.tolist(), offsets.tolist()
            return [[ScoredInt(i, s) for i, s in zip(il[ol[b]:ol[b + 1]], sl[ol[b]:ol[b + 1]])]
                    for b in range(len(q))]
        k = _DEFAULT_MAX_HITS if max_hits is None else max_hits
        items, scores, counts = self.search_arrays(q, k, min_score, subsets=ordinals_of_subsets)
        il, sl, cl = items.tolist(), scores.tolist(), counts.tolist()
        return [[ScoredInt(i, s) for i, s in zip(il[b][:c], sl[b][:c])] for b, c in enumerate(cl)]

    async def fuzzy_lookup(
        self,
        key: str,
        max_hits: int | None = None,
        min_score: float | None = None,
        predicate: Callable[[int], bool] | None = None,
    ) -> list[ScoredInt]:
        if max_hits is None:
            max_hits = self.settings.max_matches
        if min_score is None:
            min_score = self.settings.min_score
        embedding = await self.get_embedding(key)
        return self.fuzzy_lookup_embedding(
            embedding, max_hits=max_hits, min_score=min_score, predicate=predicate
        )

    async def fuzzy_lookup_keys(
        self, keys: list[str], max_hits: int | None = None, min_score: float | None = None
    ) -> list[list[ScoredInt]]:
        """Batched ``fuzzy_lookup``: one embedding request, one GPU search."""
        if not keys:
            return []
        if max_hits is None:
            max_hits = self.settings.max_matches
        if min_score is None:
            min_score = self.settings.min_score
        embeddings = await self.get_embeddings(keys)
        return self.fuzzy_lookup_embeddings(embeddings, max_hits=max_hits, min_score=min_score)

    # ------------------------------------------------------------------ torch handles
    @classmethod
    def from_device_tensor(cls, settings, tensor, **kw) -> "VectorBase":
        """Wrap a CUDA tensor [N, D] (float32 / bfloat16 / float16, contiguous) as the
        corpus without copying it and without a host mirror (benchmark-scale corpora)."""
        if kw.get("devices") is not None:
            raise NotImplementedError("from_device_tensor is not available on a VectorBase over several devices "
                                      "(devices=)")
        import torch

        if not (tensor.is_cuda and tensor.dim() == 2 and tensor.is_contiguous()):
            raise ValueError("from_device_tensor needs a contiguous 2-D CUDA tensor")
        names = {torch.float32: "float32", torch.bfloat16: "bfloat16", torch.float16: "float16"}
        if tensor.dtype not in names:
            raise ValueError(f"unsupported dtype {tensor.dtype}")
        self = cls(settings, device=tensor.device.index or 0, storage_dtype=names[tensor.dtype], **kw)
        lib, ix = self._ensure_device()
        self._embedding_size = tensor.shape[1]
        _capi.check(lib.tav_adopt_device(ix, C.c_void_p(tensor.data_ptr()), tensor.shape[0], tensor.shape[1]))
        self._adopted_tensor = tensor  # keep the memory alive
        self._device_only_rows = tensor.shape[0]
        return self

    @staticmethod
    def _device_subsets(subsets, n_queries: int, device):
        """``subsets=(offsets, ordinals)`` of the device forms: contiguous 1-D int64 CUDA tensors on the queries'
        device, offsets of n_queries + 1 entries (their values are checked on the device)."""
        import torch

        if not (isinstance(subsets, (tuple, list)) and len(subsets) == 2):
            raise ValueError("subsets must be (offsets, ordinals) device tensors")
        offsets, ordinals = subsets
        for t, what in ((offsets, "offsets"), (ordinals, "ordinals")):
            if not (getattr(t, "is_cuda", False) and t.dtype == torch.int64 and t.dim() == 1 and t.is_contiguous()):
                raise ValueError(f"subsets {what} must be a contiguous 1-D int64 CUDA tensor")
            if t.device != device:
                raise ValueError(f"subsets {what} is on {t.device}, the queries on {device}")
        if offsets.numel() != n_queries + 1:
            raise ValueError(f"subsets offsets must have {n_queries + 1} entries, not {offsets.numel()}")
        return offsets, ordinals

    def search_device(self, queries, k: int, min_score: float = 0.0, item_offset: int = 0, out=None,
                      defer_check: bool = False, allowed=None, row_to_group=None, subsets=None):
        """Lookup with torch CUDA tensors as handles, enqueued on torch's current stream:
        queries float32 [B, D] -> (items int64 [B,k], scores float32 [B,k], counts int32 [B]) on
        the device.  The tensor-core path normally ends with one host synchronisation (did any
        query need the exact fallback?); with ``defer_check=True`` the call is fully
        asynchronous and ``finish_search()`` must run before the results are trusted.
        ``allowed``: row bitmask, or one per query (see ``search_arrays``; here also a contiguous int32 CUDA
        tensor [B, ceil(N / 32)] of packed words, copied on the current stream).  ``row_to_group``: int32 CUDA tensor [N];
        the hits are then folded on the device like the reference's chunk -> message fold
        (storage/memory/messageindex.py:185-207): first hit per group, items = group ordinals.
        ``subsets=(offsets, ordinals)``: per-query subsets as ``search_arrays(subsets=)`` takes them, in CSR form as
        contiguous 1-D int64 CUDA tensors on the queries' device (offsets [B + 1], ordinals [offsets[-1]]); row b
        equals ``search_arrays(..., subsets=)``'s row b, padded to ``k`` (not clamped: the longest subset is not
        known on the host).  The offsets and ordinals are checked on the device: malformed offsets raise
        ``ValueError`` and an ordinal outside [-N, N) ``IndexError``, from this call, or with ``defer_check=True``
        from ``finish_search()`` (the call then makes no host synchronisation)."""
        self._single_device_only("search_device")
        import torch

        if not (queries.is_cuda and queries.dtype == torch.float32 and queries.is_contiguous()):
            raise ValueError("queries must be a contiguous float32 CUDA tensor")
        if queries.dim() != 2 or queries.shape[1] != self._embedding_size:
            raise ValueError("query width does not match the embedding size")
        b = queries.shape[0]
        if subsets is not None:
            if allowed is not None or row_to_group is not None or item_offset:
                raise ValueError("subsets= cannot be combined with allowed=, row_to_group= or an item_offset")
            if k < 1:
                raise ValueError("k must be >= 1")
            subsets = self._device_subsets(subsets, b, queries.device)
        lib, ix = self._ensure_device()
        if out is None:
            dev = queries.device
            out = (
                torch.empty((b, k), dtype=torch.int64, device=dev),
                torch.empty((b, k), dtype=torch.float32, device=dev),
                torch.empty((b,), dtype=torch.int32, device=dev),
            )
        items, scores, counts = out
        stream = torch.cuda.current_stream(queries.device).cuda_stream
        flags = _capi.TAV_QUERIES_ON_DEVICE | _capi.TAV_OUTPUTS_ON_DEVICE | self._flags()
        if defer_check and row_to_group is None:
            flags |= _capi.TAV_DEFER_RETRY
        if self._is_query_masks(allowed):
            self._use_query_masks(lib, ix, allowed, b, stream)
            flags |= _capi.TAV_USE_QUERY_MASKS
        elif allowed is not None:
            self._use_row_mask(lib, ix, allowed)
            flags |= _capi.TAV_USE_ROW_MASK
        floor = float(np.float32(min_score))
        if subsets is not None:
            offsets, ordinals = subsets
            flags &= _capi.TAV_QUERIES_ON_DEVICE | _capi.TAV_OUTPUTS_ON_DEVICE | _capi.TAV_DEFER_RETRY
            # the hits pass through the index's threshold-search buffers
            with self._single_lock:
                _capi.check(
                    lib.tav_search_subsets_into(
                        ix, C.c_void_p(queries.data_ptr()), b, k, C.c_float(floor), flags,
                        C.c_void_p(offsets.data_ptr()), C.c_void_p(ordinals.data_ptr()), ordinals.numel(),
                        C.c_void_p(items.data_ptr()), C.c_void_p(scores.data_ptr()), C.c_void_p(counts.data_ptr()),
                        C.c_void_p(stream),
                    )
                )
            if flags & _capi.TAV_DEFER_RETRY:
                # the device works on these tensors until finish_search(): keep them alive
                self._pending.append((queries, items, scores, counts, stream, subsets))
            return items, scores, counts
        _capi.check(
            lib.tav_search(ix, C.c_void_p(queries.data_ptr()), b, k, C.c_float(floor),
                           flags, None, 0, item_offset, C.c_void_p(items.data_ptr()),
                           C.c_void_p(scores.data_ptr()), C.c_void_p(counts.data_ptr()),
                           C.c_void_p(stream))
        )
        if row_to_group is not None:
            if not (row_to_group.is_cuda and row_to_group.dtype == torch.int32 and row_to_group.is_contiguous()):
                raise ValueError("row_to_group must be a contiguous int32 CUDA tensor")
            _capi.check(
                lib.tav_fold_groups(self._device, b, k, C.c_void_p(row_to_group.data_ptr()), row_to_group.numel(),
                                    item_offset, C.c_void_p(items.data_ptr()), C.c_void_p(scores.data_ptr()),
                                    C.c_void_p(counts.data_ptr()), C.c_void_p(stream))
            )
        if flags & _capi.TAV_DEFER_RETRY:
            # the library redoes flagged queries into these very buffers at finish_search(): keep them alive
            self._pending.append((queries, items, scores, counts, stream, allowed))
        return items, scores, counts

    def search_range_device(self, queries, min_score: float = 0.0, capacity: int | None = None, *, out=None,
                            defer_check: bool = False, allowed=None, ties_low_first: bool = False, subset=None,
                            expected_hits: int | None = None, item_offset: int = 0, subsets=None):
        """Threshold search with torch CUDA tensors as handles, enqueued on torch's current stream: every row whose
        score is >= min_score, per query, as ``search_range`` finds them, into device tensors
        (offsets int64 [B + 1], items int64 [capacity], scores float32 [capacity]).  The offsets are always
        complete; hits at CSR positions >= ``capacity`` are not written (those slots keep what they held), so when
        ``offsets[-1] > capacity`` the caller may search again with more room.  ``out`` may supply the three
        tensors (``capacity`` then defaults to the room they have).  Items are row ordinals (or subset ordinals)
        + ``item_offset``, as in ``search_device``.  ``queries``: a contiguous float32 CUDA tensor
        [B, D]; ``allowed`` as in ``search_device``; ``subset``: host ordinals as in ``search_range``.
        ``expected_hits`` (default ``capacity``) sizes the device collect regions; it never changes the result.
        The call synchronises once (more when a query overflowed its region); with ``defer_check=True`` it does
        not synchronise at all, and ``finish_search()`` must run before the results are trusted.
        ``subsets=(offsets, ordinals)``: per-query subsets from device tensors as in ``search_device``; the result
        equals ``search_range(..., subsets=)``'s (``expected_hits`` is not used).  A refused search (malformed
        offsets: ``ValueError``; an ordinal outside [-N, N): ``IndexError``) leaves all offsets 0."""
        self._single_device_only("search_range_device")
        import torch

        if not (getattr(queries, "is_cuda", False) and queries.dtype == torch.float32 and queries.is_contiguous()):
            raise ValueError("queries must be a contiguous float32 CUDA tensor")
        if queries.dim() != 2 or queries.shape[1] != self._embedding_size:
            raise ValueError("query width does not match the embedding size")
        b = queries.shape[0]
        dev = queries.device
        if out is not None:
            if len(out) != 3:
                raise ValueError("out must be (offsets, items, scores)")
            offsets, items, scores = out
            for t, dt, what in ((offsets, torch.int64, "offsets"), (items, torch.int64, "items"),
                                (scores, torch.float32, "scores")):
                if not (getattr(t, "is_cuda", False) and t.dtype == dt and t.dim() == 1 and t.is_contiguous()):
                    raise ValueError(f"out {what} must be a contiguous 1-D {dt} CUDA tensor")
                if t.device != dev:
                    raise ValueError(f"out {what} is on {t.device}, the queries on {dev}")
            if offsets.numel() != b + 1:
                raise ValueError(f"out offsets must have {b + 1} entries, not {offsets.numel()}")
            if capacity is None:
                capacity = min(items.numel(), scores.numel())
        if capacity is None:
            raise ValueError("capacity is needed when out is not given")
        if isinstance(capacity, bool) or int(capacity) != capacity or capacity < 0:
            raise ValueError(f"capacity must be a non-negative integer, not {capacity!r}")
        capacity = int(capacity)
        if out is not None and (items.numel() < capacity or scores.numel() < capacity):
            raise ValueError(f"out items / scores hold fewer than capacity = {capacity} hits")
        if expected_hits is None:
            expected_hits = capacity
        if isinstance(expected_hits, bool) or int(expected_hits) != expected_hits or expected_hits < 0:
            raise ValueError(f"expected_hits must be a non-negative integer, not {expected_hits!r}")
        sub = None
        if subsets is not None:
            if subset is not None or allowed is not None or item_offset:
                raise ValueError("subsets= cannot be combined with subset=, allowed= or an item_offset")
            subsets = self._device_subsets(subsets, b, dev)
        if subset is not None:
            if allowed is not None:
                raise ValueError("allowed= and subset= cannot be combined")
            sub = np.ascontiguousarray(subset)
            if sub.size and not np.issubdtype(sub.dtype, np.integer):
                raise IndexError("arrays used as indices must be of integer (or boolean) type")
            sub = sub.astype(np.int64, copy=False).reshape(-1)
        if out is None:
            offsets = torch.empty((b + 1,), dtype=torch.int64, device=dev)
            items = torch.empty((capacity,), dtype=torch.int64, device=dev)
            scores = torch.empty((capacity,), dtype=torch.float32, device=dev)
        lib, ix = self._ensure_device()
        stream = torch.cuda.current_stream(dev).cuda_stream
        flags = _capi.TAV_QUERIES_ON_DEVICE | (self._flags() & ~_capi.TAV_NO_FUSED_SCAN)
        if defer_check:
            flags |= _capi.TAV_DEFER_RETRY
        if self._is_query_masks(allowed):
            self._use_query_masks(lib, ix, allowed, b, stream)
            flags |= _capi.TAV_USE_QUERY_MASKS
        elif allowed is not None:
            self._use_row_mask(lib, ix, allowed)
            flags |= _capi.TAV_USE_ROW_MASK
        if ties_low_first:
            flags |= _capi.TAV_TIES_LOW_FIRST
        floor = float(_as_f32_scalar(min_score))
        if subsets is not None:
            s_offsets, s_ordinals = subsets
            flags &= _capi.TAV_QUERIES_ON_DEVICE | _capi.TAV_DEFER_RETRY | _capi.TAV_TIES_LOW_FIRST
            with self._single_lock:
                _capi.check(
                    lib.tav_range_search_subsets_into(
                        ix, C.c_void_p(queries.data_ptr()), b, C.c_float(floor), flags,
                        C.c_void_p(s_offsets.data_ptr()), C.c_void_p(s_ordinals.data_ptr()), s_ordinals.numel(),
                        capacity, C.c_void_p(offsets.data_ptr()), C.c_void_p(items.data_ptr()),
                        C.c_void_p(scores.data_ptr()), C.c_void_p(stream),
                    )
                )
            if defer_check:
                self._pending.append((queries, items, scores, offsets, stream, subsets))
            return offsets, items, scores
        # the call gives up the index's threshold-search hits: not between a search_range and its fetch
        with self._single_lock:
            _capi.check(
                lib.tav_range_search_into(
                    ix, C.c_void_p(queries.data_ptr()), b, C.c_float(floor), flags,
                    sub.ctypes.data_as(C.c_void_p) if sub is not None else None, len(sub) if sub is not None else 0,
                    int(item_offset), int(expected_hits), capacity, C.c_void_p(offsets.data_ptr()),
                    C.c_void_p(items.data_ptr()), C.c_void_p(scores.data_ptr()), C.c_void_p(stream),
                )
            )
        if defer_check:
            # the library searches flagged queries again into these very tensors at finish_search(): keep them alive
            self._pending.append((queries, items, scores, offsets, stream, allowed))
        return offsets, items, scores

    def finish_search(self) -> int:
        """Complete every outstanding ``search_device(..., defer_check=True)`` and
        ``search_range_device(..., defer_check=True)``: synchronise, redo (exactly) the queries the device search
        flagged, return how many there were.  A deferred ``subsets=`` search that the device checks refused raises
        here (``ValueError`` / ``IndexError``), after every other outstanding search has been completed."""
        self._single_device_only("finish_search")
        if not self._pending:
            return 0
        stream = self._pending[-1][4]
        redone = C.c_int(0)
        try:
            _capi.check(_capi.load().tav_finish_search(self._ix, C.c_void_p(stream), C.byref(redone)))
        finally:
            self._pending.clear()
        return redone.value
