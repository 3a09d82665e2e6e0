"""Expected search results without tolerances (numpy, CPU only).

``expected_topk`` is the library's result on given float32 dot products: the reference's float32
score map, its ``score >= min_score`` float32 compare, and the library's total order (score bits
descending, then row descending).  Whenever every path computes the same float32 dots, every path
must return exactly this — which ``dyadic_corpus`` arranges: its values are small integers times a
power of two, so every product and every partial sum is exact in float32 in any summation order
(row scan, wgmma, the split planes, the shard merge).  On arbitrary data the tensor-core search must
still equal ``expected_topk`` of the dots its own kernel dumps (``tav_mma_scores``), and those dots
must lie within ``dot_error_bound`` of the exact ones.
"""

from __future__ import annotations

import math

import numpy as np

_ONE, _HALF = np.float32(1.0), np.float32(0.5)
_BLOCK_ELEMS = 1 << 24  # keys built at once (128 MB of uint64)


def scores_of(dots_f32: np.ndarray) -> np.ndarray:
    """clip((x + 1f) * 0.5f, 0, 1) in float32 (== (x + 1) / 2: halving is exact); NaN stays NaN."""
    with np.errstate(invalid="ignore"):
        return np.clip((np.asarray(dots_f32, np.float32) + _ONE) * _HALF, np.float32(0), _ONE)


def expected_topk(dots_f32, k, min_score, allowed=None, item_offset=0):
    """items int64 [B, k], scores float32 [B, k], counts int32 [B] — padding -1 / 0.0 as in
    ``search_arrays``.  Rows qualify when their score is not NaN, ``score >= float32(min_score)``
    (NEP 50: a Python float compares as float32) and ``allowed`` (bool [N]) is set."""
    dots = np.atleast_2d(np.asarray(dots_f32, np.float32))
    b, n = dots.shape
    items = np.full((b, k), -1, np.int64)
    scores = np.zeros((b, k), np.float32)
    counts = np.zeros(b, np.int32)
    floor = np.float32(min_score)
    if n == 0 or np.isnan(floor):
        return items, scores, counts
    take = min(k, n)
    rows = np.arange(n, dtype=np.uint64)
    step = max(1, _BLOCK_ELEMS // n)
    for q0 in range(0, b, step):
        s = scores_of(dots[q0:q0 + step])
        with np.errstate(invalid="ignore"):
            ok = s >= floor  # False for NaN
        if allowed is not None:
            ok &= np.asarray(allowed, bool)[None, :]
        # key + 1 for qualifying rows, 0 for the rest: descending keys = the library's order
        keys = np.where(ok, ((s.view(np.uint32).astype(np.uint64) << np.uint64(32)) | rows) + np.uint64(1),
                        np.uint64(0))
        top = np.partition(keys, n - take, axis=1)[:, n - take:] if take < n else keys
        top = -np.sort(-top.astype(np.int64), axis=1)[:, :take].astype(np.uint64)  # keys < 2^62: int64-safe
        valid = top != 0
        key = top - np.uint64(1)
        blk = slice(q0, q0 + len(top))
        counts[blk] = valid.sum(axis=1)
        items[blk, :take] = np.where(valid, (key & np.uint64(0xFFFFFFFF)).astype(np.int64) + item_offset, -1)
        scores[blk, :take] = np.where(valid, (key >> np.uint64(32)).astype(np.uint32).view(np.float32), 0.0)
    return items, scores, counts


# ---------------------------------------------------------------- exact-arithmetic corpora
PRESETS = {
    # few ties: the widest integers all three storage types hold, dots spread to std ~0.35
    "fine": dict(amp=255, std=0.35),
    # heavy ties (a few hundred distinct dots), dots spread to std ~1: tails clip to scores 0.0 and 1.0
    "coarse": dict(amp=3, std=1.0),
}


def preset(name: str, d: int) -> tuple[int, int]:
    """(amp, exp) of a preset at width d: amp as large as the preset allows with d * amp^2 < 2^24,
    exp the power of two that brings the dots' standard deviation nearest the preset's."""
    p = PRESETS[name]
    amp = min(p["amp"], int(math.isqrt((1 << 24) // d - 1)))
    # integer uniform on [-amp, amp]: E[a^2] = amp (amp + 1) / 3, so std(dot) = sqrt(d) E[a^2] 2^-2exp
    spread = math.sqrt(d) * amp * (amp + 1) / 3.0
    exp = max(0, round(0.5 * math.log2(spread / p["std"])))
    return amp, exp


def dyadic_corpus(n, d, b, amp, exp, seed, dup=()):
    """Corpus float32 [n, d], queries float32 [b, d] with values a * 2^-exp, integer |a| <= amp, and
    their exact dots float32 [b, n].  amp <= 255 and exp <= 24 keep every value exact in bfloat16,
    float16 (whose split form then has lo = 0) and float32; d * amp^2 < 2^24 keeps every partial sum
    of a dot an integer multiple of 2^-2exp below 2^24 of them, i.e. exact in float32 in any order.
    ``dup``: pairs (dst, src) — row dst becomes a copy of row src (exact ties at chosen ranks)."""
    assert d * amp * amp < (1 << 24), "partial sums would not be exact in float32"
    assert amp <= 255 and 0 <= exp <= 24, "values would not be exact in bfloat16 / float16"
    rng = np.random.default_rng(seed)
    vi = rng.integers(-amp, amp + 1, size=(n, d), dtype=np.int64)
    qi = rng.integers(-amp, amp + 1, size=(b, d), dtype=np.int64)
    for dst, src in dup:
        vi[dst] = vi[src]
    scale = np.float32(2.0 ** -exp)
    exact = qi @ vi.T  # |.| < 2^24: exact in float32, and the power-of-two scale is exact too
    dots = exact.astype(np.float32) * np.float32(2.0 ** (-2 * exp))
    return vi.astype(np.float32) * scale, qi.astype(np.float32) * scale, dots


# ---------------------------------------------------------------- rounding-error bound
_U = 2.0 ** -23  # unit roundoff per addition: the tensor cores' adder is not specified to round to nearest,
#                  so a truncating one (error < 1 ulp) is allowed for


def _gamma(m: int) -> float:
    return m * _U / (1.0 - m * _U)


def dot_error_bound(q, v, split=False):
    """float64 [B, N]: a rigorous bound on |computed - exact| of the float32 dots q @ v.T for ANY
    summation order, gamma_d * sum_i |q_i v_i| (inputs taken as exact: pass the storage-rounded ones).
    ``split``: float32 inputs carried as fp16 planes x ~= hi + lo / 2048 — adds their representation
    error (2^-22 relative, plus 2^-36 absolute for fp16 subnormals), the dropped lo * lo' term (<= 2^-22
    relative) and the 2d-term cross accumulator with its final fused combine."""
    q = np.abs(np.asarray(q, np.float64))
    v = np.abs(np.asarray(v, np.float64))
    d = q.shape[1]
    mag = q @ v.T
    if not split:
        return _gamma(d) * mag
    rel = 2.0 ** -22
    eta = 2.0 ** -36
    rep = (2 * rel + rel * rel) * mag + eta * (q.sum(1)[:, None] + v.sum(1)[None, :] + d * eta)
    return (_gamma(2 * d + 1) + rel) * (mag + rep) + rep + _U * (mag + rep)
