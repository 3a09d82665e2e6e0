"""``EmbeddingIndex`` on the GPU ``VectorBase``.

Same public surface as the reference's thin wrapper (``typeagent.knowpro.fuzzyindex.
EmbeddingIndex``, /root/reference/src/typeagent/knowpro/fuzzyindex.py:12-143: size / get / push /
add_texts / nearest / nearest-in-subset / clear / (de)serialize), plus ``get_indexes_of_nearest_
batch`` — the single batched GPU search that replaces the per-term loop of the related-terms
expansion (storage/memory/reltermsindex.py:320-332).  Most methods are one-line delegations; they
are declared through ``_delegate`` so that the mapping index-method -> VectorBase-method is a
table rather than boilerplate.
"""

from __future__ import annotations

from collections.abc import Callable, Sequence

import numpy as np

from .vectorbase import ScoredInt, TextEmbeddingIndexSettings, VectorBase


def _delegate(target: str, doc: str):
    """A method that forwards positionally to ``self._vector_base.<target>``."""

    def method(self, *args):
        return getattr(self._vector_base, target)(*args)

    method.__name__ = target
    method.__doc__ = doc
    return method


class EmbeddingIndex:
    """Ordinal-addressed embedding store with nearest-neighbour lookups."""

    def __init__(
        self,
        settings: TextEmbeddingIndexSettings,
        embeddings: np.ndarray | None = None,
        **vectorbase_options,
    ):
        # ``_vector_base`` keeps the reference's attribute name: its tests and textlocindex reach into it
        self._vector_base = VectorBase(settings, **vectorbase_options)
        if embeddings is not None:
            self.push(embeddings)

    # -- size ---------------------------------------------------------------------------------
    def __len__(self) -> int:
        return len(self._vector_base)

    async def size(self) -> int:
        return len(self)

    async def is_empty(self) -> bool:
        return len(self) == 0

    # -- rows ---------------------------------------------------------------------------------
    get = _delegate("get_embedding_at", "Row ``pos``; IndexError when out of range.")
    clear = _delegate("clear", "Drop every row (the embedding size is kept).")
    serialize = _delegate("serialize", "The rows as one float32 [N, D] array (a view, no copy).")

    def push(self, embeddings: np.ndarray) -> None:
        """Append rows (float32 [n, D]); no keys are cached."""
        self._vector_base.add_embeddings(None, embeddings)

    async def add_texts(self, texts: list[str]) -> None:
        await self._vector_base.add_keys(texts)

    def remove_at(self, pos: int) -> None:
        """Remove the embedding at ``pos``; the rows after it move up by one (compacted on the device)."""
        if 0 <= pos < len(self._vector_base):
            self._vector_base.remove_embedding_at(pos)
        else:
            raise IndexError(
                f"Index {pos} out of bounds for embedding index of size {len(self._vector_base)}"
            )

    async def get_embedding(self, key: str, cache: bool = True):
        return await self._vector_base.get_embedding(key, cache)

    def deserialize(self, embeddings: np.ndarray) -> None:
        """Adopt a float32 [N, D] array; same input contract as the reference (its asserts)."""
        width = self._vector_base._embedding_size
        assert isinstance(embeddings, np.ndarray), type(embeddings)
        assert embeddings.dtype == np.float32, embeddings.dtype
        assert embeddings.ndim == 2, embeddings.shape
        assert width in (0, embeddings.shape[1]), embeddings.shape
        self._vector_base.deserialize(embeddings)

    # -- lookups ------------------------------------------------------------------------------
    def get_indexes_of_nearest(
        self,
        embedding,
        max_matches: int | None = None,
        min_score: float | None = None,
        predicate: Callable[[int], bool] | None = None,
    ) -> list[ScoredInt]:
        return self._vector_base.fuzzy_lookup_embedding(embedding, max_matches, min_score, predicate)

    def get_indexes_of_nearest_in_subset(
        self,
        embedding,
        ordinals_of_subset: list[int],
        max_matches: int | None = None,
        min_score: float | None = None,
    ) -> list[ScoredInt]:
        return self._vector_base.fuzzy_lookup_embedding_in_subset(
            embedding, ordinals_of_subset, max_matches, min_score
        )

    def get_indexes_of_nearest_batch(
        self,
        embeddings: np.ndarray,
        max_matches: int | None = None,
        min_score: float | None = None,
    ) -> list[list[ScoredInt]]:
        """One GPU search for a [B, D] batch of query embeddings."""
        return self._vector_base.fuzzy_lookup_embeddings(embeddings, max_matches, min_score)

    def get_indexes_of_nearest_in_subsets_batch(
        self,
        embeddings: np.ndarray,
        ordinals_of_subsets: Sequence[Sequence[int]],
        max_matches: int | None = None,
        min_score: float | None = None,
    ) -> list[list[ScoredInt]]:
        """One GPU search in which query b of a [B, D] batch scores only ``ordinals_of_subsets[b]``."""
        return self._vector_base.fuzzy_lookup_embeddings_in_subsets(embeddings, ordinals_of_subsets, max_matches,
                                                                    min_score)
