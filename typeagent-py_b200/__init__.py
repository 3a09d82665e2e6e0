"""typeagent-py_b200 — H100-native engine for typeagent's VectorBase top-k lookup.

Drop-in for ONE path of microsoft/typeagent-py: ``typeagent.aitools.vectorbase.VectorBase``
(and its thin wrapper ``typeagent.knowpro.fuzzyindex.EmbeddingIndex``), executed by
hand-written sm_90a CUDA kernels behind the C ABI in ``include/tavec.h``.  There is no CPU
fallback: lookups raise ``RuntimeError`` when the CUDA library or a device is missing.
"""

from .vectorbase import (  # noqa: F401
    DEFAULT_MIN_SCORE,
    MODEL_DEFAULT_MIN_SCORES,
    ScoredInt,
    TextEmbeddingIndexSettings,
    VectorBase,
    cosine_to_score,
    get_default_min_score,
)
from .fuzzyindex import EmbeddingIndex  # noqa: F401
from .sharded import ShardedVectorBase  # noqa: F401
from .install import install, uninstall  # noqa: F401

__all__ = [
    "DEFAULT_MIN_SCORE",
    "MODEL_DEFAULT_MIN_SCORES",
    "EmbeddingIndex",
    "ScoredInt",
    "ShardedVectorBase",
    "TextEmbeddingIndexSettings",
    "VectorBase",
    "cosine_to_score",
    "get_default_min_score",
    "install",
    "uninstall",
]
