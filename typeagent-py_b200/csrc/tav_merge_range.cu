// tav_merge_range.cu — merge step of the row-sharded threshold search (tav_merge_range, include/tavec.h).
//
// Input: W per-rank CSR hit lists (tav_range_search results, items already global), each query's hits in the
// library's order.  Output: per query, the union of the W lists in the same order, CSR.  A merge, not a sort:
//
//   * a query's output is cut into tiles of kMrTile hits; a tile's inputs are, in every list g, the hits
//     [a_g, b_g) where a / b are the co-ranks of the tile's first and one-past-last output rank (the split
//     of that rank over the W lists, found by bisection: below);
//   * a CTA loads those W runs into shared memory (each input hit is read from global memory once, by the
//     tile that outputs it), places every hit at its rank inside the tile (its own index in its run plus,
//     per other run, a binary search in shared memory) and writes the tile out contiguously.
//
// Work distribution: a one-CTA plan kernel writes out_offsets (per query the sum of the lists' offsets:
// they already are prefix sums) and the first tile of every query in one flat tile space; the merge kernel
// gives every CTA an equal contiguous run of that space, whatever the queries' sizes — one large query
// spreads over every CTA, many small ones share CTAs.  Inside a run consecutive tiles of a query share
// their boundary, so each boundary's co-rank is searched once, and inside a window one tile wide after the
// previous boundary; only a run's first boundary is searched over the whole lists.
//
// Order: score descending, then item descending (ascending with ties_low).  Scores compare as float32
// values, through a sign-aware key of their bits (the library's are in [0, 1]; NaN has no defined place).
// Exactly equal (score, item) pairs, which distinct global rows never produce, fall back to the list index
// so that the order is total whatever the input.
//
// TAV_MERGE_RANGE_MUTANT (tests only, never set by build.py): 1..5 compile one deliberate defect each, so that
// the GPU test can show its exact checks catch it (tests/test_gpu_sharded_range.py).

#include <stdint.h>

#include <algorithm>

#include "tav_common.cuh"
#include "tav_internal.h"

#ifndef TAV_MERGE_RANGE_MUTANT
#define TAV_MERGE_RANGE_MUTANT 0
#endif

namespace tav {
namespace {

constexpr int kMrThreads = 256;
constexpr int kMrPerThread = 8;
constexpr int kMrTile = kMrThreads * kMrPerThread;  // output hits per tile
constexpr int kMrMaxLists = 32;                     // the co-rank scratch holds W x W counts
constexpr int kMrCtasPerSm = 5;                     // 48 registers per thread: no spills
constexpr int kMrPlanThreads = 1024;

struct MrArgs {
    int n_lists;
    int n_queries;
    const int64_t* offsets;
    int64_t offsets_stride;
    const int64_t* items;
    int64_t items_stride;
    const float* scores;
    int64_t scores_stride;
    int ties_low;
    int64_t* out_offsets;
    int64_t* out_items;
    float* out_scores;
    int64_t* tile_start;  // scratch [n_queries + 1]: first flat tile of every query, then the tile count
};

// list g's hits of query q: [*first, *first + *n) of its arrays
__device__ __forceinline__ void list_hits(const MrArgs& a, int g, int q, int64_t* first, int64_t* n) {
    const int64_t* off = a.offsets + g * a.offsets_stride;
    const int64_t b = off[q];
    int64_t e = off[q + 1];
#if TAV_MERGE_RANGE_MUTANT == 4
    if (q == a.n_queries - 1 && a.items_stride > 0) e = a.items_stride;  // defect: padded counts
#endif
    *first = b;
    *n = max(e - b, static_cast<int64_t>(0));
}

__device__ __forceinline__ int64_t tiles_of(int64_t hits) {
#if TAV_MERGE_RANGE_MUTANT == 5
    return hits / kMrTile;  // defect: last partial tile dropped
#else
    return (hits + kMrTile - 1) / kMrTile;
#endif
}

// float32 bits -> unsigned key in the order of the values (negative values below positive ones)
__device__ __forceinline__ uint32_t order_key(uint32_t bits) {
    return (bits & 0x80000000u) ? ~bits : (bits | 0x80000000u);
}

// hit (sa, ia) of list ga comes before hit (sb, ib) of list gb; scores as raw float32 bits
__device__ __forceinline__ bool precedes(uint32_t sa, int64_t ia, int ga, uint32_t sb, int64_t ib, int gb,
                                         int ties_low) {
    if (sa != sb) return order_key(sa) > order_key(sb);
#if TAV_MERGE_RANGE_MUTANT == 1
    return ga < gb;  // defect: equal scores ordered by list instead of item
#endif
#if TAV_MERGE_RANGE_MUTANT == 2
    ties_low = 0;    // defect: ties-low ignored
#endif
    if (ia != ib) return ties_low ? ia < ib : ia > ib;
    return ga < gb;
}

// the CTA's scratch for a co-rank search
struct CorankSmem {
    int64_t lo[kMrMaxLists], hi[kMrMaxLists], mid[kMrMaxLists], rank[kMrMaxLists];
    int64_t piv_item[kMrMaxLists];
    uint32_t piv_score[kMrMaxLists];
    int open[kMrMaxLists];
    int64_t p[kMrMaxLists * kMrMaxLists];  // [pivot list g][list h]: hits of h before g's pivot (window-clamped)
};

// Co-rank of output rank r of one query (the whole CTA calls it): split[g] = how many of list g's n[g] hits come
// among the query's first r outputs.  Bisection on every list at once, keeping lo[g] <= split[g] <= hi[g]: each
// round the midpoint of every open window is a pivot P; its rank among all hits is the sum over the lists h of
// the number of h's hits before P, each found by a binary search (one thread per (pivot, list) pair) inside h's
// window — clamping to the window does not change whether rank < r (P is among the first r outputs).  If it is,
// every hit before P is too: each lo[h] rises to that count (and past P in P's own list); if not, each hi[h]
// falls to it.  Every window at least halves per round.  `floor` (or nullptr): the co-rank of an earlier rank
// r - span of the same query, which bounds every window to [floor[g], floor[g] + span].
__device__ __forceinline__ void corank(const MrArgs& a, int W, const int64_t* base, const int64_t* n, int64_t r,
                                       int64_t total, const int64_t* floor, int64_t span, CorankSmem& sm,
                                       int64_t* split) {
    const int tid = threadIdx.x;
    int64_t lo = 0, hi = 0;
    if (tid < W) {
        hi = min(n[tid], r);
        lo = max(static_cast<int64_t>(0), r - (total - n[tid]));
        if (floor) {
            lo = max(lo, floor[tid]);
            hi = min(hi, floor[tid] + span);
        }
    }
    for (;;) {
        const bool open = tid < W && lo < hi;
        if (tid < W) {
            sm.lo[tid] = lo;
            sm.hi[tid] = hi;
            sm.rank[tid] = 0;
            sm.open[tid] = open;
            if (open) {
                const int64_t mid = lo + (hi - lo) / 2;
                sm.mid[tid] = mid;
                sm.piv_score[tid] = __float_as_uint(a.scores[tid * a.scores_stride + base[tid] + mid]);
                sm.piv_item[tid] = a.items[tid * a.items_stride + base[tid] + mid];
            }
        }
        if (!__syncthreads_or(open)) break;
        for (int pr = tid; pr < W * W; pr += kMrThreads) {
            const int g = pr / W, h = pr - g * W;
            if (!sm.open[g]) continue;
            int64_t p = sm.mid[g];
            if (h != g) {
                const uint32_t ps = sm.piv_score[g];
                const int64_t pi = sm.piv_item[g];
                const float* sc = a.scores + h * a.scores_stride + base[h];
                const int64_t* it = a.items + h * a.items_stride + base[h];
                int64_t L = sm.lo[h], H = sm.hi[h];
                while (L < H) {
                    const int64_t m = L + (H - L) / 2;
                    if (precedes(__float_as_uint(sc[m]), it[m], h, ps, pi, g, a.ties_low))
                        L = m + 1;
                    else
                        H = m;
                }
                p = L;
            }
            sm.p[pr] = p;
            atomicAdd(reinterpret_cast<unsigned long long*>(&sm.rank[g]), static_cast<unsigned long long>(p));
        }
        __syncthreads();
        if (tid < W) {
            for (int g = 0; g < W; ++g) {
                if (!sm.open[g]) continue;
                const int64_t p = sm.p[g * W + tid];
                if (sm.rank[g] < r)
                    lo = max(lo, p + (g == tid ? 1 : 0));
                else
                    hi = min(hi, p);
            }
        }
        __syncthreads();
    }
#if TAV_MERGE_RANGE_MUTANT == 3
    if (tid == 0 && r > 0 && r < total && lo < n[0]) lo += 1;  // defect: one list's co-rank off by one
#endif
    if (tid < W) split[tid] = lo;
    __syncthreads();
}

// one CTA: out_offsets, and the flat tile space (tile_start[q] = first tile of query q, tile_start[B] = tiles)
__global__ void __launch_bounds__(kMrPlanThreads) merge_range_plan(const MrArgs a) {
    __shared__ int64_t s_sum[kMrPlanThreads];
    const int B = a.n_queries, W = a.n_lists, tid = threadIdx.x;
    const int per = (B + kMrPlanThreads - 1) / kMrPlanThreads;
    const int q0 = min(B, tid * per), q1 = min(B, q0 + per);
    auto query = [&](int q, int64_t* out, int64_t* hits) {
        int64_t o = 0, t = 0;
        for (int g = 0; g < W; ++g) {
            int64_t first, n;
            list_hits(a, g, q, &first, &n);
            o += first;
            t += n;
        }
        *out = o;
        *hits = t;
    };
    int64_t mine = 0;
    for (int q = q0; q < q1; ++q) {
        int64_t out, hits;
        query(q, &out, &hits);
        a.out_offsets[q] = out;
        mine += tiles_of(hits);
        if (q == B - 1) a.out_offsets[B] = out + hits;
    }
    s_sum[tid] = mine;
    __syncthreads();
    for (int off = 1; off < kMrPlanThreads; off <<= 1) {  // inclusive scan
        const int64_t v = tid >= off ? s_sum[tid - off] : 0;
        __syncthreads();
        s_sum[tid] += v;
        __syncthreads();
    }
    int64_t run = s_sum[tid] - mine;
    for (int q = q0; q < q1; ++q) {
        int64_t out, hits;
        query(q, &out, &hits);
        a.tile_start[q] = run;
        run += tiles_of(hits);
    }
    if (tid == kMrPlanThreads - 1) a.tile_start[B] = s_sum[tid];
}

__global__ void __launch_bounds__(kMrThreads, kMrCtasPerSm) merge_range_kernel(const MrArgs a) {
    __shared__ int64_t t_items[kMrTile];
    __shared__ uint32_t t_scores[kMrTile];
    __shared__ CorankSmem cs;
    __shared__ int64_t s_base[kMrMaxLists], s_n[kMrMaxLists], s_a[kMrMaxLists], s_b[kMrMaxLists];
    __shared__ int s_start[kMrMaxLists + 1];
    __shared__ int64_t s_total, s_out;
    // the run's end and the loaded query's state live in shared memory (kept in registers across the tile loop,
    // ptxas spills them)
    __shared__ int64_t s_t_end, s_tile0, s_tile1;
    __shared__ int s_q, s_carried;  // the loaded query; s_a holds the co-rank of this tile's first rank
    const int W = a.n_lists, B = a.n_queries, tid = threadIdx.x;
    const int64_t n_tiles = a.tile_start[B];
    const int64_t per = (n_tiles + gridDim.x - 1) / gridDim.x;
    const int64_t t_begin = blockIdx.x * per;
    if (t_begin >= n_tiles) return;
    if (tid == 0) {  // the query of the run's first tile: the last q with tile_start[q] <= t_begin
        int lo = 0, hi = B - 1;
        while (lo < hi) {
            const int m = (lo + hi + 1) >> 1;
            if (a.tile_start[m] <= t_begin)
                lo = m;
            else
                hi = m - 1;
        }
        s_t_end = min(n_tiles, t_begin + per);
        s_q = lo - 1;
        s_tile1 = -1;
    }
    __syncthreads();
    for (int64_t t = t_begin; t < s_t_end; ++t) {
        if (t >= s_tile1) {  // next query with tiles (uniform: every thread reads the same words)
            int q = s_q + 1;
            while (a.tile_start[q + 1] <= t) ++q;
            __syncthreads();  // every thread has read s_tile1 / s_q; the previous tile's readers of s_base / s_n are done
            if (tid < W) list_hits(a, tid, q, &s_base[tid], &s_n[tid]);
            __syncthreads();
            if (tid == 0) {
                int64_t total = 0;
                for (int g = 0; g < W; ++g) total += s_n[g];
                s_total = total;
                s_out = a.out_offsets[q];
                s_tile0 = a.tile_start[q];
                s_tile1 = a.tile_start[q + 1];
                s_q = q;
                s_carried = 0;
            }
            __syncthreads();
        }
        const int64_t total = s_total, out_base = s_out;
        const int64_t r0 = (t - s_tile0) * kMrTile, r1 = min(r0 + kMrTile, total);
        if (r0 == 0) {
            if (tid < W) s_a[tid] = 0;
        } else if (!s_carried) {
            corank(a, W, s_base, s_n, r0, total, nullptr, 0, cs, s_a);
        }
        if (r1 == total) {
            if (tid < W) s_b[tid] = s_n[tid];
        } else {
            __syncthreads();  // s_a complete before it bounds the windows
            corank(a, W, s_base, s_n, r1, total, s_a, r1 - r0, cs, s_b);
        }
        __syncthreads();
        if (tid == 0) {  // run g of the tile: list g's hits [s_a[g], s_a[g] + len), at s_start[g] in shared memory
            int start = 0;
            for (int g = 0; g < W; ++g) {
                const int64_t lo = min(max(s_a[g], static_cast<int64_t>(0)), s_n[g]);
                const int64_t hi = min(max(s_b[g], lo), s_n[g]);
                const int len = static_cast<int>(min(hi - lo, static_cast<int64_t>(kMrTile - start)));
                s_a[g] = lo;
                s_start[g] = start;
                start += len;
            }
            s_start[W] = start;
        }
        __syncthreads();
        const int n_tile = s_start[W];
        for (int g = 0; g < W; ++g) {
            const int s0 = s_start[g], len = s_start[g + 1] - s0;
            const int64_t src = s_base[g] + s_a[g];
            const int64_t* it = a.items + g * a.items_stride + src;
            const float* sc = a.scores + g * a.scores_stride + src;
            for (int i = tid; i < len; i += kMrThreads) {
                t_items[s0 + i] = it[i];
                t_scores[s0 + i] = __float_as_uint(sc[i]);
            }
        }
        __syncthreads();
        int64_t my_item[kMrPerThread];
        uint32_t my_score[kMrPerThread];
        int my_pos[kMrPerThread];
#pragma unroll
        for (int j = 0; j < kMrPerThread; ++j) {
            const int i = tid + j * kMrThreads;
            my_pos[j] = -1;
            my_item[j] = 0;
            my_score[j] = 0;
            if (i < n_tile) {
                int g = 0;
                while (i >= s_start[g + 1]) ++g;
                const uint32_t s = t_scores[i];
                const int64_t item = t_items[i];
                int pos = i - s_start[g];
                for (int h = 0; h < W; ++h) {
                    if (h == g) continue;
                    int L = s_start[h], H = s_start[h + 1];
                    const int h0 = L;
                    while (L < H) {
                        const int m = (L + H) >> 1;
                        if (precedes(t_scores[m], t_items[m], h, s, item, g, a.ties_low))
                            L = m + 1;
                        else
                            H = m;
                    }
                    pos += L - h0;
                }
                my_pos[j] = pos;
                my_item[j] = item;
                my_score[j] = s;
            }
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < kMrPerThread; ++j) {
            if (my_pos[j] >= 0) {
                t_items[my_pos[j]] = my_item[j];
                t_scores[my_pos[j]] = my_score[j];
            }
        }
        __syncthreads();
        const int n_out = static_cast<int>(min(static_cast<int64_t>(n_tile), r1 - r0));
        int64_t* oi = a.out_items + out_base + r0;
        float* os = a.out_scores + out_base + r0;
        for (int i = tid; i < n_out; i += kMrThreads) {
            oi[i] = t_items[i];
            os[i] = __uint_as_float(t_scores[i]);
        }
        if (tid < W) s_a[tid] = s_b[tid];  // the next tile of this query starts where this one ends
        if (tid == 0) s_carried = 1;
        __syncthreads();
    }
}

}  // namespace

#define TAVM_CUDA(expr)                                                                            \
    do {                                                                                           \
        cudaError_t _e = (expr);                                                                   \
        if (_e != cudaSuccess) {                                                                   \
            set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return _e == cudaErrorMemoryAllocation ? TAV_ERR_OOM : TAV_ERR_CUDA;                   \
        }                                                                                          \
    } while (0)

}  // namespace tav

using namespace tav;

extern "C" int tav_merge_range(int device, int n_lists, int n_queries, const int64_t* offsets, int64_t offsets_stride,
                               const int64_t* items, int64_t items_stride, const float* scores, int64_t scores_stride,
                               int ties_low_first, int64_t* out_offsets, int64_t* out_items, float* out_scores,
                               void* stream) {
    if (n_lists < 1 || n_lists > kMrMaxLists || n_queries < 0 || offsets_stride < 0 || items_stride < 0 ||
        scores_stride < 0) {
        set_error("tav_merge_range: invalid argument (1 <= n_lists <= %d, strides >= 0)", kMrMaxLists);
        return TAV_ERR_INVALID;
    }
    if (n_queries == 0) return TAV_OK;
    if (!offsets || !items || !scores || !out_offsets || !out_items || !out_scores) {
        set_error("tav_merge_range: null pointer");
        return TAV_ERR_INVALID;
    }
    TAVM_CUDA(cudaSetDevice(device));
    int sms = 0;
    TAVM_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    // the flat tile space: stream-ordered scratch, so concurrent merges on other streams never share it
    int64_t* tile_start = nullptr;
    TAVM_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&tile_start), (static_cast<size_t>(n_queries) + 1) * sizeof(int64_t),
                              s));
    MrArgs a{n_lists, n_queries, offsets, offsets_stride, items, items_stride, scores, scores_stride,
             ties_low_first ? 1 : 0, out_offsets, out_items, out_scores, tile_start};
    merge_range_plan<<<1, kMrPlanThreads, 0, s>>>(a);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) {
        merge_range_kernel<<<kMrCtasPerSm * sms, kMrThreads, 0, s>>>(a);  // one resident wave over all tiles
        e = cudaGetLastError();
    }
    const cudaError_t f = cudaFreeAsync(tile_start, s);
    TAVM_CUDA(e);
    TAVM_CUDA(f);
    return TAV_OK;
}
