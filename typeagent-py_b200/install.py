"""Swap the GPU ``VectorBase`` into an importable typeagent, and batch its related-term loops.

The reference has no plugin registry: ``VectorBase`` is a concrete class bound by name at
import time in six modules (SURVEY.md §8b).  ``install()``

* rebinds that name in each module that is importable (the reference's own ``EmbeddingIndex``
  is a pure forwarder and then builds the GPU class), and
* replaces the two one-query-at-a-time loops of the related-terms expansion —
  ``TermEmbeddingIndex.lookup_terms`` (storage/memory/reltermsindex.py:320-332) and
  ``SqliteRelatedTermsFuzzy.lookup_terms`` (storage/sqlite/reltermsindex.py:259-271, "TODO: Some
  kind of batching?") — by ONE embedding request + ONE batched GPU search
  (``VectorBase.fuzzy_lookup_keys``); that is what makes BASELINE config 5 (1 000 query terms
  against the term vocabulary) reachable from ``resolve_related_terms``
  (storage/memory/reltermsindex.py:147-201);

and returns what it patched; ``uninstall()`` restores the originals.  typeagent itself is
optional: without it, ``install()`` patches nothing and says so.
"""

from __future__ import annotations

import importlib

# module -> names bound there (reference: knowpro/fuzzyindex.py:9,23; storage/memory/
# reltermsindex.py:10-14,266; storage/memory/convthreads.py:4,20; storage/sqlite/
# messageindex.py:12,33; storage/sqlite/reltermsindex.py:11,139; aitools/vectorbase.py:82)
_SITES = {
    "typeagent.aitools.vectorbase": ("VectorBase",),
    "typeagent.knowpro.fuzzyindex": ("VectorBase",),
    "typeagent.storage.memory.reltermsindex": ("VectorBase",),
    "typeagent.storage.memory.convthreads": ("VectorBase",),
    "typeagent.storage.sqlite.messageindex": ("VectorBase",),
    "typeagent.storage.sqlite.reltermsindex": ("VectorBase",),
}

_saved: dict[tuple[str, str], object] = {}


def _batched_memory_lookup_terms(original):
    """TermEmbeddingIndex.lookup_terms: same result as the reference's loop of ``fuzzy_lookup`` calls."""

    async def lookup_terms(self, texts, max_hits=None, min_score=None):
        base = self._vectorbase
        if not hasattr(base, "fuzzy_lookup_keys"):   # an index built before install(): leave it alone
            return await original(self, texts, max_hits, min_score)
        if not texts:
            return []
        matches = await base.fuzzy_lookup_keys(list(texts), max_hits=max_hits, min_score=min_score)
        return [self.matches_to_terms(m) for m in matches]

    lookup_terms.__wrapped__ = original
    return lookup_terms


def _batched_sqlite_lookup_terms(original, term_type):
    """SqliteRelatedTermsFuzzy.lookup_terms: ordinals -> Term through ``_terms_list``, as ``lookup_term``
    does (storage/sqlite/reltermsindex.py:158-179)."""

    async def lookup_terms(self, texts, max_hits=None, min_score=None):
        base = self._vector_base
        if not hasattr(base, "fuzzy_lookup_keys"):
            return await original(self, texts, max_hits, min_score)
        if not texts:
            return []
        matches = await base.fuzzy_lookup_keys(list(texts), max_hits=max_hits, min_score=min_score)
        terms = self._terms_list
        return [[term_type(terms[m.item], m.score) for m in hits if m.item < len(terms)] for hits in matches]

    lookup_terms.__wrapped__ = original
    return lookup_terms


def _patch(mod_name: str, owner, name: str, value, patched: list[str], label: str) -> None:
    _saved.setdefault((mod_name, label), (owner, name, getattr(owner, name)))
    setattr(owner, name, value)
    patched.append(f"{mod_name}.{label}")


def install(**vectorbase_options) -> list[str]:
    """Rebind the names; ``vectorbase_options`` (device=, storage_dtype=, normalize=, or devices= for the rows
    of every index in blocks over several GPUs of this process) become the defaults of every VectorBase typeagent
    constructs afterwards."""
    from . import vectorbase

    if vectorbase_options:
        base_cls = type(
            "VectorBase",
            (vectorbase.VectorBase,),
            {"__init__": lambda self, settings, **kw: vectorbase.VectorBase.__init__(
                self, settings, **{**vectorbase_options, **kw})},
        )
    else:
        base_cls = vectorbase.VectorBase
    patched: list[str] = []
    for mod_name, names in _SITES.items():
        try:
            mod = importlib.import_module(mod_name)
        except Exception:
            continue
        for name in names:
            if hasattr(mod, name):
                _patch(mod_name, mod, name, base_cls, patched, name)
        # the sequential related-term loops -> one batched search
        if mod_name == "typeagent.storage.memory.reltermsindex" and hasattr(mod, "TermEmbeddingIndex"):
            cls = mod.TermEmbeddingIndex
            current = cls.__dict__.get("lookup_terms")
            if current is not None and not hasattr(current, "__wrapped__"):
                _patch(mod_name, cls, "lookup_terms", _batched_memory_lookup_terms(current), patched,
                       "TermEmbeddingIndex.lookup_terms")
        if mod_name == "typeagent.storage.sqlite.reltermsindex" and hasattr(mod, "SqliteRelatedTermsFuzzy"):
            cls = mod.SqliteRelatedTermsFuzzy
            current = cls.__dict__.get("lookup_terms")
            if current is not None and not hasattr(current, "__wrapped__"):
                _patch(mod_name, cls, "lookup_terms", _batched_sqlite_lookup_terms(current, mod.interfaces.Term),
                       patched, "SqliteRelatedTermsFuzzy.lookup_terms")
    return patched


def uninstall() -> None:
    for key, (owner, name, original) in list(_saved.items()):
        try:
            setattr(owner, name, original)
        except Exception:
            pass
        del _saved[key]
