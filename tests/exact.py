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
    # benchmark-sized corpora: dots spread to std ~0.15 (0.11 to 0.18 at D = 64 .. 1536), so that even the
    # largest of 10M rows (about 5.3 std) stays below the clip at score 1.0: the sampled admission threshold of
    # the tensor-core path then sits among unclipped scores
    "scale": dict(amp=131, std=0.15),
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


def _gamma(m: int, u: float = _U) -> float:
    return m * u / (1.0 - m * u)


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


# ---------------------------------------------------------------- storage conversion
def round_to(x, dtype: str) -> np.ndarray:
    """float32 values rounded once, to nearest even, to `dtype` and upcast (exactly) back to float32:
    numpy's own conversion for float16, ``round_to_bfloat16`` for bfloat16.  NaN stays NaN."""
    x = np.asarray(x, np.float32)
    if dtype == "float32":
        return x.copy()
    if dtype == "float16":
        with np.errstate(over="ignore"):
            return x.astype(np.float16).astype(np.float32)
    from oracle.vectorbase_oracle import round_to_bfloat16

    return round_to_bfloat16(x)


def to_bits16(x, dtype: str) -> np.ndarray:
    """The uint16 encoding of float32 values already representable in `dtype` (bfloat16 or float16)."""
    x = np.asarray(x, np.float32)
    if dtype == "float16":
        with np.errstate(over="ignore"):
            return x.astype(np.float16).view(np.uint16)
    assert dtype == "bfloat16"
    bits = x.view(np.uint32)
    assert ((bits & 0xFFFF) == 0)[~np.isnan(x)].all(), "not a bfloat16 value"
    return (bits >> 16).astype(np.uint16)


def _f32(bits) -> np.ndarray:
    return np.array(bits, np.uint32).view(np.float32)


def conversion_edges() -> dict[str, np.ndarray]:
    """float32 values where a conversion to bfloat16 or float16 goes wrong first, by class (positive
    values: the sign is added where they are used, except in "zero_inf_nan")."""
    bf = np.array([0x3F80, 0x3F81, 0x4049, 0x404A, 0x0080, 0x0081, 0x0001, 0x0002, 0x7F7E], np.uint32)
    h = np.array([0x3C00, 0x3C01, 0x0001, 0x0002, 0x03FF, 0x7BFE, 0x0400, 0x5BFF], np.uint16)
    h_lo = h.view(np.float16).astype(np.float64)
    h_hi = (h + 1).astype(np.uint16).view(np.float16).astype(np.float64)
    fp16_mid = ((h_lo + h_hi) / 2).astype(np.float32)  # exact in float32
    bf_max, fp_max = _f32([0x7F7F0000])[0], np.float32(65504)
    return {
        # tie at bfloat16 precision: even and odd last bit, normal, subnormal and large; and one float32 ulp off
        "bf16_halfway": _f32(np.concatenate([(bf << 16) | 0x8000, (bf << 16) | 0x7FFF, (bf << 16) | 0x8001])),
        "fp16_halfway": np.concatenate([fp16_mid, np.nextafter(fp16_mid, np.float32(0)),
                                        np.nextafter(fp16_mid, np.float32(np.inf))]),
        # the largest finite value of each format, one float32 ulp past it, half a target ulp past it
        "max_finite": np.array([bf_max, np.nextafter(bf_max, np.float32(np.inf)), _f32([0x7F7F7FFF])[0],
                                _f32([0x7F7F8000])[0], np.finfo(np.float32).max, fp_max,
                                np.nextafter(fp_max, np.float32(np.inf)), 65519.996, 65536.0], np.float32),
        "fp16_overflow": np.array([65520.0, np.nextafter(np.float32(65520), np.float32(0)), 65521.0, 1e5, 1e38],
                                  np.float32),
        "subnormal": np.array([2.0 ** -24, 3 * 2.0 ** -24, 2.0 ** -14, 2.0 ** -14 - 2.0 ** -24, 2.0 ** -133,
                               2.0 ** -126, 2.0 ** -149, 2.0 ** -127 * 3], np.float32),
        "rounds_to_zero": np.array([2.0 ** -25, np.nextafter(np.float32(2.0 ** -25), np.float32(0)),
                                    np.nextafter(np.float32(2.0 ** -25), np.float32(1)), 2.0 ** -26, 2.0 ** -134,
                                    2.0 ** -135, 2.0 ** -149, 1e-30], np.float32),
        "zero_inf_nan": np.array([0.0, -0.0, np.inf, -np.inf, np.nan, -np.nan], np.float32),
    }


_U_RN = 2.0 ** -24  # unit roundoff of the CUDA cores' float32 fma, sqrtf and division (round to nearest)
# storage rounding: (relative unit roundoff, absolute error in the subnormal range)
_STORE = {"float32": (0.0, 0.0), "bfloat16": (2.0 ** -8, 2.0 ** -134), "float16": (2.0 ** -11, 2.0 ** -25)}


def normalize_error_bound(v, storage="float32"):
    """float64 [N, D]: a rigorous bound on |stored - v / ||v||| for rows normalised as the append kernel
    does: v scaled by a power of two (exact), the float32 sum of squares in ANY order (gamma_d relative; at
    most d roundings on any path, plus d * 2^-149 for squares of scaled values below the normal range:
    the scaled sum is >= 1/4), the square root and the division (one rounding each, 2^-148 for a scaled
    value or quotient in the subnormal range), then the storage rounding of that float32 quotient (a second
    rounding on 16-bit storage, bounded separately: the bound holds for double rounding).  Zero rows: 0."""
    v = np.asarray(v, np.float64)
    d = v.shape[1]
    x = np.abs(v) / np.maximum(np.sqrt((v * v).sum(1, keepdims=True)), np.finfo(np.float64).tiny)
    d_ss = _gamma(d, _U_RN) * (1 + _U_RN) + d * 2.0 ** -147
    e_nrm = d_ss + _U_RN + d_ss * _U_RN  # sqrt(1 + a) - 1 <= a: halving the relative error is not needed
    rel = (1 + _U_RN) / (1 - e_nrm) - 1
    err32 = rel * x + 2.0 ** -148
    u_s, abs_s = _STORE[storage]
    return err32 + u_s * (x + err32) + abs_s


def _two_squares_table(amp: int) -> dict[int, tuple[int, int]]:
    t: dict[int, tuple[int, int]] = {}
    for a in range(amp + 1):
        for b in range(a, amp + 1):
            t.setdefault(a * a + b * b, (a, b))
    return t


def four_squares(r: int, amp: int, table=None) -> tuple[int, int, int, int]:
    """Non-negative integers <= amp whose squares sum to r (raises ValueError when there are none)."""
    table = table if table is not None else _two_squares_table(amp)
    for a in range(min(amp, math.isqrt(r)), -1, -1):
        for b in range(min(a, math.isqrt(r - a * a)), -1, -1):
            pair = table.get(r - a * a - b * b)
            if pair is not None:
                return a, b, pair[0], pair[1]
    raise ValueError(f"{r} is not a sum of four squares <= {amp}^2")


def unit_rows(n, d, amp, seed, e_range=(-100, 64)):
    """Integer rows a [n, d] with |a_i| <= amp and sum a_i^2 = 4^m exactly (one m for all rows), each
    multiplied by its own power of two 2^e, e uniform in ``e_range``.  Returns (rows float32 = a * 2^e,
    a int64, m, e int64 [n]).  The normalised row is exactly a / 2^m — held by float32, and with amp <= 255
    (m <= 11) by bfloat16 and float16 too — and dots of two such rows are exact in float32 (d amp^2 < 2^24).
    The first d - 4 coordinates are drawn, adjusted until the remainder to 4^m is at most 2 amp^2, and
    the last four are a four-square decomposition of that remainder."""
    assert d >= 4 and d * amp * amp < (1 << 24)
    rng = np.random.default_rng(seed)
    mean_sq = amp * (amp + 1) / 3.0  # E[a^2] of an integer uniform on [-amp, amp]
    m = max(1, int(math.floor(math.log(max(4.0, (d - 4) * mean_sq + amp * amp), 4))))
    target, cap = 4 ** m, 2 * amp * amp
    a = rng.integers(-amp, amp + 1, size=(n, d), dtype=np.int64)
    a[:, d - 4:] = 0
    free = max(d - 4, 1)
    rem = target - (a * a).sum(1)
    for _ in range(100 * d + 1000):
        over, under = rem < 0, rem > cap
        if not (over.any() or under.any()):
            break
        j = rng.integers(0, free, size=n)
        rows = np.arange(n)
        old = a[rows, j] ** 2
        # too large: zero a coordinate; too small: raise one as far as the remainder allows
        grow = np.minimum(amp, np.sqrt((old + np.maximum(rem, 0)).astype(np.float64)).astype(np.int64))
        new = np.where(over, 0, np.where(under, grow * grow, old))
        sign = np.where(a[rows, j] < 0, -1, 1)
        if d > 4:
            a[rows, j] = sign * np.where(over, 0, np.where(under, grow, np.abs(a[rows, j])))
        rem -= new - old
    assert ((rem >= 0) & (rem <= cap)).all(), "remainders did not settle"
    table = _two_squares_table(amp)
    for i in range(n):
        a[i, d - 4:] = np.array(four_squares(int(rem[i]), amp, table)) * rng.choice([-1, 1], size=4)
    perm = rng.permuted(np.tile(np.arange(d), (n, 1)), axis=1)  # the four fill-ins anywhere in the row
    a = np.take_along_axis(a, perm, axis=1)
    assert ((a * a).sum(1) == target).all() and np.abs(a).max() <= amp
    e = rng.integers(e_range[0], e_range[1] + 1, size=n)
    rows = (a.astype(np.float64) * np.exp2(e.astype(np.float64))[:, None]).astype(np.float32)
    return rows, a, m, e
