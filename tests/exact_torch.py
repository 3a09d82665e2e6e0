"""Expected search results without tolerances, in torch: ``tests/exact.py``'s expectations restated so that
corpora of tens of millions of rows can be checked on the device (they also run on CPU tensors).

Dots come from dyadic corpora (``exact.dyadic_corpus``: values a * 2^-exp, integer |a| <= amp, d * amp^2 < 2^24):
a float64 GEMM of the integer matrices is exact (every partial sum is an integer below 2^53; float64 has no
reduced-precision GEMM mode to fall into), and so is its conversion to float32 and the power-of-two scale.  The
score map and compare are ``exact.scores_of``'s float32 arithmetic.  The order is the library's: int64 keys
``score_bits << 32 | row`` (``~row`` in the low word for ties-low) descending, non-admitted rows key -1.

A dots source is an iterable of (first row, float32 dots [B, rows]) blocks; a plain [B, N] tensor is one block.
"""

from __future__ import annotations

import math

import torch

_BLOCK_BYTES = 1 << 30  # float64 elements of one row block (corpus or dots) converted at once
_LOW = 0xFFFFFFFF


def scores_of(dots: torch.Tensor) -> torch.Tensor:
    """clip((x + 1f) * 0.5f, 0, 1) in float32; NaN stays NaN."""
    return torch.clamp((dots.to(torch.float32) + 1.0) * 0.5, 0.0, 1.0)


def _integers(x: torch.Tensor, exp: int) -> torch.Tensor:
    xi = x.to(torch.float64) * float(2.0 ** exp)
    assert bool((xi == torch.round(xi)).all()), "not a dyadic value a * 2^-exp"
    return xi


def _to_f32(dots_int: torch.Tensor, exp: int) -> torch.Tensor:
    if dots_int.numel():
        assert float(dots_int.abs().max()) < 2.0 ** 24, "an integer dot is not exact in float32"
    return dots_int.to(torch.float32) * float(2.0 ** (-2 * exp))


def dyadic_dots(corpus: torch.Tensor, queries: torch.Tensor, exp: int, block_rows: int | None = None):
    """(r0, float32 dots [B, rows]) for row blocks of ``corpus`` [N, D] (any float dtype, on any device) against
    ``queries`` [B, D], both holding values a * 2^-exp."""
    qi = _integers(queries.to(corpus.device), exp)
    n, d = corpus.shape
    rows = block_rows or max(1, _BLOCK_BYTES // (8 * max(d, len(qi), 1)))
    for r0 in range(0, n, rows):
        vi = _integers(corpus[r0:r0 + rows], exp)
        yield r0, _to_f32(qi @ vi.T, exp)


def subset_dots(corpus: torch.Tensor, queries: torch.Tensor, exp: int, offsets: torch.Tensor, ordinals: torch.Tensor,
                block_entries: int | None = None):
    """(j0, float32 dots [entries]) for blocks of the flat entries of per-query subsets: entry j is the dot of the
    query q with offsets[q] <= j < offsets[q + 1] and row ordinals[j] (negatives wrap like numpy)."""
    dev = corpus.device
    qi = _integers(queries.to(dev), exp)
    offsets, ordinals = offsets.to(dev), ordinals.to(dev)
    n, d = corpus.shape
    step = block_entries or max(1, _BLOCK_BYTES // (8 * d))
    for j0 in range(0, len(ordinals), step):
        j = torch.arange(j0, min(j0 + step, len(ordinals)), device=dev)
        q = torch.searchsorted(offsets, j, right=True) - 1
        vi = _integers(corpus[torch.remainder(ordinals[j0:j0 + len(j)], n)], exp)
        yield j0, _to_f32((vi * qi[q]).sum(1), exp)


def _blocks(source):
    return [(0, source)] if isinstance(source, torch.Tensor) else source


def _floor(min_score) -> float:
    import numpy as np

    return float(np.float32(min_score))


def _keys(scores: torch.Tensor, low: torch.Tensor, ok: torch.Tensor) -> torch.Tensor:
    bits = scores.view(torch.int32).to(torch.int64)  # admitted scores are >= +0: bits < 2^31
    return torch.where(ok, (bits << 32) | low, torch.full_like(bits, -1))


def _low(index: torch.Tensor, ties_low: bool) -> torch.Tensor:
    return (~index) & _LOW if ties_low else index


def _decode(keys: torch.Tensor, ties_low: bool):
    """keys -> (index of the row or entry, float32 score)."""
    low = keys & _LOW
    index = (~low) & _LOW if ties_low else low
    return index, (keys >> 32).to(torch.int32).view(torch.float32)


def _admitted(dots, r0, floor, allowed, ties_low):
    b, rows = dots.shape
    s = scores_of(dots)
    ok = s >= floor  # False for NaN
    if allowed is not None:
        ok &= (allowed[..., r0:r0 + rows] if allowed.dim() == 2 else allowed[r0:r0 + rows][None, :]).to(ok.device)
    row = torch.arange(r0, r0 + rows, device=dots.device, dtype=torch.int64)
    return _keys(s, _low(row, ties_low)[None, :].expand(b, rows), ok)


def topk_ref(source, k: int, min_score, allowed=None, ties_low=False, item_offset=0):
    """items int64 [B, k], scores float32 [B, k], counts int32 [B] — as ``exact.expected_topk``, plus ``ties_low``
    (equal scores: lower row first) and ``allowed`` given per query (bool [B, N]) or shared (bool [N])."""
    best = None
    n = 0
    floor = _floor(min_score)
    for r0, dots in _blocks(source):
        n = max(n, r0 + dots.shape[1])
        if math.isnan(floor):
            continue
        keys = _admitted(dots, r0, floor, allowed, ties_low)
        if best is not None:
            keys = torch.cat([best, keys], dim=1)
        best = torch.topk(keys, min(k, keys.shape[1]), dim=1).values
    b = dots.shape[0]
    dev = dots.device
    items = torch.full((b, k), -1, dtype=torch.int64, device=dev)
    scores = torch.zeros((b, k), dtype=torch.float32, device=dev)
    counts = torch.zeros(b, dtype=torch.int32, device=dev)
    if best is None:
        return items, scores, counts
    valid = best >= 0
    row, s = _decode(best, ties_low)
    take = best.shape[1]
    items[:, :take] = torch.where(valid, row + item_offset, -1)
    scores[:, :take] = torch.where(valid, s, torch.zeros_like(s))
    counts[:] = valid.sum(1).to(torch.int32)
    return items, scores, counts


def _csr(per_query, dev):
    lengths = torch.tensor([len(x) for x in per_query], dtype=torch.int64)
    offsets = torch.zeros(len(per_query) + 1, dtype=torch.int64)
    offsets[1:] = torch.cumsum(lengths, 0)
    keys = torch.cat(per_query) if per_query else torch.empty(0, dtype=torch.int64, device=dev)
    return offsets.to(dev), keys


def range_ref(source, min_score, allowed=None, ties_low=False, item_offset=0):
    """offsets int64 [B + 1], items int64 [T], scores float32 [T]: every admitted row of every query, in the
    library's order (as ``test_gpu_range.expected_range``)."""
    floor = _floor(min_score)
    per_query = None
    for r0, dots in _blocks(source):
        if per_query is None:
            per_query = [[] for _ in range(dots.shape[0])]
        if math.isnan(floor):
            continue
        keys = _admitted(dots, r0, floor, allowed, ties_low)
        for b in range(len(keys)):
            per_query[b].append(keys[b][keys[b] >= 0])
    dev = dots.device
    sorted_keys = [torch.sort(torch.cat(x), descending=True).values if x else torch.empty(0, dtype=torch.int64,
                                                                                            device=dev)
                   for x in per_query]
    offsets, keys = _csr(sorted_keys, dev)
    row, s = _decode(keys, ties_low)
    return offsets, row + item_offset, s


def subsets_ref(entry_source, offsets: torch.Tensor, ordinals: torch.Tensor, k: int, min_score, ties_low=False):
    """Per-query subsets -> ((items [B, k], scores [B, k], counts [B]), (offsets [B + 1], items [T], scores [T])).
    ``entry_source``: (j0, float32 dots [entries]) blocks of the flat entries (``subset_dots``).  Keys are built
    from the flat index j into ``ordinals`` (later entry first among equal scores, earlier with ties-low), items
    are the ordinals as given.  Both forms share one order: the top-k is the head of the threshold list."""
    floor = _floor(min_score)
    dev = ordinals.device
    offsets = offsets.to(dev)
    parts = []
    for j0, dots in entry_source:
        j = torch.arange(j0, j0 + len(dots), device=dev, dtype=torch.int64)
        s = scores_of(dots.to(dev))
        ok = s >= floor if not math.isnan(floor) else torch.zeros_like(s, dtype=torch.bool)
        parts.append(_keys(s, _low(j, ties_low), ok))
    keys = torch.cat(parts) if parts else torch.empty(0, dtype=torch.int64, device=dev)
    off = offsets.tolist()
    per_query = []
    for b in range(len(off) - 1):
        seg = keys[off[b]:off[b + 1]]
        per_query.append(torch.sort(seg[seg >= 0], descending=True).values)
    csr_offsets, flat = _csr(per_query, dev)
    j, s = _decode(flat, ties_low)
    csr = (csr_offsets, ordinals[j], s)
    nq = len(per_query)
    items = torch.full((nq, k), -1, dtype=torch.int64, device=dev)
    scores = torch.zeros((nq, k), dtype=torch.float32, device=dev)
    counts = torch.zeros(nq, dtype=torch.int32, device=dev)
    for b in range(nq):
        c = min(k, len(per_query[b]))
        start = int(csr_offsets[b])
        items[b, :c] = csr[1][start:start + c]
        scores[b, :c] = s[start:start + c]
        counts[b] = c
    return (items, scores, counts), csr
