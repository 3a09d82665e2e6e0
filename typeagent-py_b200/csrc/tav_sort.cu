// tav_sort.cu — segmented sort of the threshold search's hits (tav_range_search): every query's
// admitted keys, unsorted, in one segment each -> descending key order, decoded into CSR items / scores.
//
// Keys are the library's unique 64-bit (score_bits << 32 | position) keys (tav_common.cuh), so sorting
// them exactly gives the library's total order, ties in score included, without a stable sort.
//   * segments of at most kSmallSortMax keys: one CTA each, bitonic sort in shared memory;
//   * larger segments: a multi-CTA LSD radix sort over 8-bit digits, all large segments in the same
//     launches.  Only the digits below the highest bit that varies inside a segment (min key XOR max
//     key) are sorted: keys sharing their upper bits need no pass over them.  A pass is histogram per
//     tile of kRadixTile keys -> per-segment prefix over (digit, tile) -> stable scatter.  Descending
//     order comes from sorting the bucket 255 - digit ascending.
//
// Device-planned form (tav_range_search_into): range_plan_kernel turns the collect counters into the CSR
// offsets, the segments, the large-segment list and the tile map on the device; the sort kernels are then
// launched over host-known upper bounds, their CTAs past the plan's counts return at once, and the decode
// writes only CSR positions below the caller's capacity.  Each kernel body is one template: the <false>
// instantiation is the host-planned kernel, unchanged.

#include <algorithm>

#include "tav_common.cuh"
#include "tav_internal.h"

namespace tav {

constexpr int kSortThreads = 256;
constexpr int kRadixBuckets = 256;
constexpr int kMaxRadixPasses = 8;  // 64-bit keys

// the device-planned kernels' extra argument: the plan's counts, and the capacity of the caller's outputs
struct SortBound {
    const int* sizes;  // device [2]: large segments, radix tiles
    int64_t cap;       // CSR positions >= cap are not written
};

__device__ __forceinline__ void decode_store(uint64_t key, const SortArgs& a, int64_t at) {
    const uint32_t kp = key_pos(key);
    const uint32_t pos = a.ties_low ? ~kp : kp;
    a.out_items[at] = (a.subset ? a.subset[pos] : static_cast<int64_t>(pos)) + a.item_offset;
    a.out_scores[at] = key_score(key);
}

__device__ __forceinline__ int radix_passes(const uint64_t* minmax, int l) {
    const uint64_t v = minmax[2 * l] ^ minmax[2 * l + 1];
    return v ? (64 - __clzll(static_cast<long long>(v)) + 7) / 8 : 0;
}

__device__ __forceinline__ uint32_t bucket_of(uint64_t key, int pass) {
#if TAV_SCALE_MUTANT == 3
    if (pass == 3) return 0u;
#endif
    return 255u - static_cast<uint32_t>((key >> (8 * pass)) & 0xFFu);
}

// ---- small segments: one CTA, shared memory ---------------------------------------------------------
template <bool kDev>
__device__ __forceinline__ void small_sort(const SortArgs& a, const SortBound& bd) {
    __shared__ uint64_t keys[kSmallSortMax];
    const SortSeg seg = a.segs[blockIdx.x];
    if (seg.n == 0 || seg.n > kSmallSortMax) return;
    if (kDev && seg.out >= bd.cap) return;
    const int n = static_cast<int>(seg.n);
    int cap = 2;
    while (cap < n) cap <<= 1;
    for (int i = threadIdx.x; i < cap; i += kSortThreads) keys[i] = i < n ? seg.keys[i] : 0;  // 0: below every key
    bitonic_sort_desc<kSortThreads>(keys, cap);
    for (int i = threadIdx.x; i < n; i += kSortThreads)
        if (!kDev || seg.out + i < bd.cap) decode_store(keys[i], a, seg.out + i);
}
__global__ void __launch_bounds__(kSortThreads) small_sort_kernel(const SortArgs a) { small_sort<false>(a, SortBound{}); }
__global__ void __launch_bounds__(kSortThreads) small_sort_dev_kernel(const SortArgs a, const SortBound bd) {
    small_sort<true>(a, bd);
}

// ---- large segments: LSD radix sort -------------------------------------------------------------------
struct TileRef {
    SortSeg seg;
    int l;          // index into a.large
    int64_t first;  // first key of the tile inside the segment
    int n;          // keys in the tile
};
__device__ __forceinline__ TileRef tile_ref(const SortArgs& a, int64_t t) {
    TileRef r;
    r.l = a.tile_seg[t];
    r.seg = a.segs[a.large[r.l]];
    r.first = (t - r.seg.tile0) * kRadixTile;
    r.n = static_cast<int>(min(static_cast<int64_t>(kRadixTile), r.seg.n - r.first));
    return r;
}
// device-planned: this CTA's tile (or large segment, which = 1) is past the plan's count
template <bool kDev>
__device__ __forceinline__ bool past_plan(const SortBound& bd, int which) {
    return kDev && static_cast<int>(blockIdx.x) >= bd.sizes[which];
}

template <bool kDev>
__device__ __forceinline__ void radix_minmax(const SortArgs& a, const SortBound& bd) {
    if (past_plan<kDev>(bd, 1)) return;
    const TileRef r = tile_ref(a, blockIdx.x);
    unsigned long long lo = ~0ull, hi = 0ull;
    for (int i = threadIdx.x; i < r.n; i += kSortThreads) {
        const unsigned long long k = r.seg.keys[r.first + i];
        lo = min(lo, k);
        hi = max(hi, k);
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
        lo = min(lo, __shfl_xor_sync(0xFFFFFFFFu, lo, off));
        hi = max(hi, __shfl_xor_sync(0xFFFFFFFFu, hi, off));
    }
    if ((threadIdx.x & 31) == 0) {
        atomicMin(reinterpret_cast<unsigned long long*>(a.minmax + 2 * r.l), lo);
        atomicMax(reinterpret_cast<unsigned long long*>(a.minmax + 2 * r.l + 1), hi);
    }
}
__global__ void __launch_bounds__(kSortThreads) radix_minmax_kernel(const SortArgs a) { radix_minmax<false>(a, SortBound{}); }
__global__ void __launch_bounds__(kSortThreads) radix_minmax_dev_kernel(const SortArgs a, const SortBound bd) {
    radix_minmax<true>(a, bd);
}

// pass p reads the keys from `keys` when p is even, from `tmp` when odd (and writes the other one)
__device__ __forceinline__ const uint64_t* pass_src(const SortSeg& s, int p) { return (p & 1) ? s.tmp : s.keys; }
__device__ __forceinline__ uint64_t* pass_dst(const SortSeg& s, int p) { return (p & 1) ? s.keys : s.tmp; }

template <bool kDev>
__device__ __forceinline__ void radix_hist(const SortArgs& a, const SortBound& bd, int pass) {
    __shared__ uint32_t h[kRadixBuckets];
    if (past_plan<kDev>(bd, 1)) return;
    const TileRef r = tile_ref(a, blockIdx.x);
    if (pass >= radix_passes(a.minmax, r.l)) return;
    h[threadIdx.x] = 0;
    __syncthreads();
    const uint64_t* src = pass_src(r.seg, pass) + r.first;
    for (int i = threadIdx.x; i < r.n; i += kSortThreads) atomicAdd(&h[bucket_of(src[i], pass)], 1u);
    __syncthreads();
    a.hist[static_cast<size_t>(blockIdx.x) * kRadixBuckets + threadIdx.x] = h[threadIdx.x];
}
__global__ void __launch_bounds__(kSortThreads) radix_hist_kernel(const SortArgs a, int pass) {
    radix_hist<false>(a, SortBound{}, pass);
}
__global__ void __launch_bounds__(kSortThreads) radix_hist_dev_kernel(const SortArgs a, const SortBound bd, int pass) {
    radix_hist<true>(a, bd, pass);
}

// one CTA per large segment, thread b = bucket b: offs[tile][b] = keys of the segment in buckets < b
// + keys in bucket b of the segment's earlier tiles
template <bool kDev>
__device__ __forceinline__ void radix_offsets(const SortArgs& a, const SortBound& bd, int pass) {
    __shared__ uint32_t s_warp[kRadixBuckets / 32];
    if (past_plan<kDev>(bd, 0)) return;
    const int l = blockIdx.x;
    if (pass >= radix_passes(a.minmax, l)) return;
    const SortSeg seg = a.segs[a.large[l]];
    const int64_t nt = (seg.n + kRadixTile - 1) / kRadixTile;
    const int b = threadIdx.x, lane = b & 31, warp = b >> 5;
    const uint32_t* h = a.hist + static_cast<size_t>(seg.tile0) * kRadixBuckets + b;
    uint32_t total = 0;
    for (int64_t t = 0; t < nt; t += 8) {  // eight independent loads in flight
        uint32_t v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) v[u] = t + u < nt ? h[(t + u) * kRadixBuckets] : 0u;
#pragma unroll
        for (int u = 0; u < 8; ++u) total += v[u];
    }
    // exclusive scan of the bucket totals over the CTA
    uint32_t incl = total;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, incl, off);
        if (lane >= off) incl += y;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    uint32_t run = incl - total;
    for (int w = 0; w < warp; ++w) run += s_warp[w];
    uint32_t* o = a.offs + static_cast<size_t>(seg.tile0) * kRadixBuckets + b;
    for (int64_t t = 0; t < nt; t += 8) {
        uint32_t v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) v[u] = t + u < nt ? h[(t + u) * kRadixBuckets] : 0u;
#pragma unroll
        for (int u = 0; u < 8; ++u)
            if (t + u < nt) {
                o[(t + u) * kRadixBuckets] = run;
                run += v[u];
            }
    }
}
__global__ void __launch_bounds__(kRadixBuckets) radix_offsets_kernel(const SortArgs a, int pass) {
    radix_offsets<false>(a, SortBound{}, pass);
}
__global__ void __launch_bounds__(kRadixBuckets) radix_offsets_dev_kernel(const SortArgs a, const SortBound bd, int pass) {
    radix_offsets<true>(a, bd, pass);
}

// stable scatter: the tile is walked in chunks of 256 keys; inside a chunk a key's rank among equal
// buckets is (earlier warps' count) + (earlier lanes of its warp, from __match_any_sync)
template <bool kDev>
__device__ __forceinline__ void radix_scatter(const SortArgs& a, const SortBound& bd, int pass) {
    constexpr int kWarps = kSortThreads / 32;
    __shared__ uint32_t s_base[kRadixBuckets];
    __shared__ uint32_t s_wcnt[kWarps][kRadixBuckets];
    if (past_plan<kDev>(bd, 1)) return;
    const TileRef r = tile_ref(a, blockIdx.x);
    if (pass >= radix_passes(a.minmax, r.l)) return;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    s_base[tid] = a.offs[static_cast<size_t>(blockIdx.x) * kRadixBuckets + tid];
#pragma unroll
    for (int w = 0; w < kWarps; ++w) s_wcnt[w][tid] = 0;
    __syncthreads();
    const uint64_t* src = pass_src(r.seg, pass) + r.first;
    uint64_t* dst = pass_dst(r.seg, pass);
    for (int c0 = 0; c0 < r.n; c0 += kSortThreads) {
        const int i = c0 + tid;
        const bool valid = i < r.n;
        const uint64_t key = valid ? src[i] : 0;
        const uint32_t b = valid ? bucket_of(key, pass) : kRadixBuckets;
        const unsigned peers = __match_any_sync(0xFFFFFFFFu, b);
        const int rank = __popc(peers & ((1u << lane) - 1u));
        if (valid && rank == 0) s_wcnt[warp][b] = __popc(peers);
        __syncthreads();
        if (valid) {
            uint32_t at = s_base[b] + rank;
            for (int w = 0; w < warp; ++w) at += s_wcnt[w][b];
            dst[at] = key;
        }
        __syncthreads();
        uint32_t add = 0;
#pragma unroll
        for (int w = 0; w < kWarps; ++w) {
            add += s_wcnt[w][tid];
            s_wcnt[w][tid] = 0;
        }
        s_base[tid] += add;
        __syncthreads();
    }
}
__global__ void __launch_bounds__(kSortThreads) radix_scatter_kernel(const SortArgs a, int pass) {
    radix_scatter<false>(a, SortBound{}, pass);
}
__global__ void __launch_bounds__(kSortThreads) radix_scatter_dev_kernel(const SortArgs a, const SortBound bd, int pass) {
    radix_scatter<true>(a, bd, pass);
}

template <bool kDev>
__device__ __forceinline__ void radix_decode(const SortArgs& a, const SortBound& bd) {
    if (past_plan<kDev>(bd, 1)) return;
    const TileRef r = tile_ref(a, blockIdx.x);
    const int np = radix_passes(a.minmax, r.l);
    const uint64_t* src = ((np & 1) ? r.seg.tmp : r.seg.keys) + r.first;  // where the last pass left them
    for (int i = threadIdx.x; i < r.n; i += kSortThreads)
        if (!kDev || r.seg.out + r.first + i < bd.cap) decode_store(src[i], a, r.seg.out + r.first + i);
}
__global__ void __launch_bounds__(kSortThreads) radix_decode_kernel(const SortArgs a) { radix_decode<false>(a, SortBound{}); }
__global__ void __launch_bounds__(kSortThreads) radix_decode_dev_kernel(const SortArgs a, const SortBound bd) {
    radix_decode<true>(a, bd);
}

cudaError_t launch_segmented_sort(const SortArgs& a, cudaStream_t s, int* launches) {
    int n = 0;
    if (a.n_segs > 0) {
        small_sort_kernel<<<a.n_segs, kSortThreads, 0, s>>>(a);
        ++n;
    }
    if (a.n_large > 0) {
        cudaError_t e = cudaMemsetAsync(a.minmax, 0, 2 * sizeof(uint64_t) * a.n_large, s);
        if (e != cudaSuccess) return e;
        // min starts at ~0: the even words
        e = cudaMemset2DAsync(a.minmax, 2 * sizeof(uint64_t), 0xFF, sizeof(uint64_t), a.n_large, s);
        if (e != cudaSuccess) return e;
        const unsigned tiles = static_cast<unsigned>(a.n_tiles);
        radix_minmax_kernel<<<tiles, kSortThreads, 0, s>>>(a);
        for (int p = 0; p < kMaxRadixPasses; ++p) {
            radix_hist_kernel<<<tiles, kSortThreads, 0, s>>>(a, p);
            radix_offsets_kernel<<<a.n_large, kRadixBuckets, 0, s>>>(a, p);
            radix_scatter_kernel<<<tiles, kSortThreads, 0, s>>>(a, p);
        }
        radix_decode_kernel<<<tiles, kSortThreads, 0, s>>>(a);
        n += 2 + 3 * kMaxRadixPasses;
    }
    if (launches) *launches += n;
    return cudaGetLastError();
}

// ---- the device plan (tav_range_search_into) ------------------------------------------------------------
constexpr int kPlanThreads = 512;  // (1024 threads would spill)

// exclusive scan of one value per thread over the CTA; *total = the sum (every thread)
__device__ __forceinline__ int64_t plan_scan(int64_t v, int64_t* s_warp, int64_t* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int64_t incl = v;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const int64_t y = __shfl_up_sync(0xFFFFFFFFu, incl, off);
        if (lane >= off) incl += y;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        int64_t w = lane < kPlanThreads / 32 ? s_warp[lane] : 0;
        int64_t wi = w;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const int64_t y = __shfl_up_sync(0xFFFFFFFFu, wi, off);
            if (lane >= off) wi += y;
        }
        s_warp[32 + lane] = wi - w;
        if (lane == 31) s_warp[64] = wi;
    }
    __syncthreads();
    const int64_t excl = s_warp[32 + warp] + incl - v;
    *total = s_warp[64];
    __syncthreads();  // s_warp is reused by the next scan
    return excl;
}

// One CTA; thread t owns the queries [t * per, (t + 1) * per).  A query overflowed when fill[q] > cap: its count
// is still exact (the collect counters count past their regions), so it takes its place in the offsets, but its
// keys are incomplete: flagged, sorted with n = 0 (nothing written) and, packed, not gathered (dst_off -1).  When
// an abandon word is set (the split form met a value beyond the fp16 range) no query is sorted or gathered: the
// whole search is redone, and nothing of this pass may reach the caller's outputs.
__global__ void __launch_bounds__(kPlanThreads) range_plan_kernel(const RangePlanArgs a) {
    __shared__ int64_t s_warp[65];
    const bool abandon = (a.abandon[0] && *a.abandon[0]) || (a.abandon[1] && *a.abandon[1]);
    const int per = (a.nq + kPlanThreads - 1) / kPlanThreads;
    const int q0 = min(a.nq, static_cast<int>(threadIdx.x) * per), q1 = min(a.nq, q0 + per);
    int64_t hits = 0, kept = 0, large = 0, tiles = 0, over = 0;
    for (int q = q0; q < q1; ++q) {
        const int64_t n = a.count[q];
        hits += n;
        if (abandon || a.fill[q] > a.cap) {
            over += abandon ? 0 : 1;
            continue;
        }
        kept += n;
        if (n > kSmallSortMax) {
            ++large;
            tiles += (n + kRadixTile - 1) / kRadixTile;
        }
    }
    int64_t t_hits, t_kept, t_large, t_tiles, t_over;
    int64_t o_hits = plan_scan(hits, s_warp, &t_hits);
    int64_t o_kept = plan_scan(kept, s_warp, &t_kept);
    int64_t o_large = plan_scan(large, s_warp, &t_large);
    int64_t o_tiles = plan_scan(tiles, s_warp, &t_tiles);
    plan_scan(over, s_warp, &t_over);
    for (int q = q0; q < q1; ++q) {
        const int64_t n = a.count[q];
        const bool o = a.fill[q] > a.cap;
        const bool skip = abandon || o;
        SortSeg g;
        const int64_t koff = a.key_stride ? static_cast<int64_t>(q) * a.key_stride : o_kept;
        g.keys = a.keys + koff;
        g.tmp = a.tmp + koff;
        g.out = a.out_base ? a.out_base[q] : o_hits;
        g.n = skip ? 0 : n;
        g.tile0 = o_tiles;
        if (a.out_offsets) a.out_offsets[q] = o_hits;
        if (a.flags) a.flags[q] = (o && !abandon) ? static_cast<int32_t>(min(static_cast<uint32_t>(a.fill[q]), 0x7FFFFFFFu)) : 0;
        if (a.dst_off) a.dst_off[q] = skip ? -1 : o_kept;
        if (!skip && n > kSmallSortMax) {
            const int64_t nt = (n + kRadixTile - 1) / kRadixTile;
            a.large[o_large] = q;
            a.minmax[2 * o_large] = ~0ull;
            a.minmax[2 * o_large + 1] = 0ull;
            for (int64_t t = 0; t < nt; ++t) a.tile_seg[o_tiles + t] = static_cast<int>(o_large);
            ++o_large;
            o_tiles += nt;
        }
        if (!skip) o_kept += n;
        o_hits += n;
        a.segs[q] = g;
    }
    if (threadIdx.x == 0) {
        if (a.out_offsets) a.out_offsets[a.nq] = t_hits;
        a.sizes[0] = static_cast<int>(t_large);
        a.sizes[1] = static_cast<int>(t_tiles);
        if (a.n_flagged) *a.n_flagged = static_cast<int32_t>(t_over);
        if (a.n_flagged_host) *a.n_flagged_host = static_cast<int32_t>(t_over);
    }
}

cudaError_t launch_range_plan(const RangePlanArgs& a, cudaStream_t s) {
    range_plan_kernel<<<1, kPlanThreads, 0, s>>>(a);
    return cudaGetLastError();
}

// The plan of the sort of per-query subsets (tav_search_subsets_into): as range_plan_kernel over regions that never
// overflow, query q's keys (and radix scratch) at keys + key_off[q].  When an abandon word (the search's status) is
// set the search is refused: every query counts 0 hits, so the offsets are all 0 and nothing is sorted.
__global__ void __launch_bounds__(kPlanThreads, 1) range_plan_subsets_kernel(const RangePlanArgs a, const int64_t* key_off) {
    __shared__ int64_t s_warp[65];
    const bool refused = ((a.abandon[0] && *a.abandon[0]) || (a.abandon[1] && *a.abandon[1]));
    const int per = (a.nq + kPlanThreads - 1) / kPlanThreads;
    const int q0 = min(a.nq, static_cast<int>(threadIdx.x) * per), q1 = min(a.nq, q0 + per);
    int64_t hits = 0, large = 0, tiles = 0;
    for (int q = q0; q < q1; ++q) {
        if (refused && TAV_SUBSETS_DEVICE_MUTANT != 3) continue;
        const int64_t n = a.count[q];
        hits += n;
        if (!refused && n > kSmallSortMax) {
            ++large;
            tiles += (n + kRadixTile - 1) / kRadixTile;
        }
    }
    int64_t t_hits, t_large, t_tiles;
    int64_t o_hits = plan_scan(hits, s_warp, &t_hits);
    int64_t o_large = plan_scan(large, s_warp, &t_large);
    int64_t o_tiles = plan_scan(tiles, s_warp, &t_tiles);
    for (int q = q0; q < q1; ++q) {
        const int64_t n = refused && TAV_SUBSETS_DEVICE_MUTANT != 3 ? 0 : a.count[q];
        SortSeg g;
        g.keys = a.keys + key_off[q];
        g.tmp = a.tmp + key_off[q];
        g.out = o_hits;
        g.n = refused ? 0 : n;
        g.tile0 = o_tiles;
        a.out_offsets[q] = o_hits;
        if (g.n > kSmallSortMax) {
            const int64_t nt = (n + kRadixTile - 1) / kRadixTile;
            a.large[o_large] = q;
            a.minmax[2 * o_large] = ~0ull;
            a.minmax[2 * o_large + 1] = 0ull;
            for (int64_t t = 0; t < nt; ++t) a.tile_seg[o_tiles + t] = static_cast<int>(o_large);
            ++o_large;
            o_tiles += nt;
        }
        o_hits += n;
        a.segs[q] = g;
    }
    if (threadIdx.x == 0) {
        a.out_offsets[a.nq] = t_hits;
        a.sizes[0] = static_cast<int>(t_large);
        a.sizes[1] = static_cast<int>(t_tiles);
    }
}

cudaError_t launch_range_plan_subsets(const RangePlanArgs& a, const int64_t* key_off, cudaStream_t s) {
    range_plan_subsets_kernel<<<1, kPlanThreads, 0, s>>>(a, key_off);
    return cudaGetLastError();
}

// ---- the work plan of per-query subsets from device offsets (tav_search_subsets_into) ----------------------
// One CTA; thread t owns the queries [t * per, (t + 1) * per).  The offsets must start at 0, never decrease and end
// at n_ordinals; otherwise the status word is set and no work is planned, so nothing reads the ordinals.  Query q's
// work items are its tiles of kSubsetTile entries, [work0[q], work0[q + 1]).
__global__ void __launch_bounds__(kPlanThreads) subset_plan_kernel(const SubsetPlanArgs a) {
    __shared__ int64_t s_warp[65];
    const int per = (a.nq + kPlanThreads - 1) / kPlanThreads;
    const int q0 = min(a.nq, static_cast<int>(threadIdx.x) * per), q1 = min(a.nq, q0 + per);
    auto tiles_of = [](int64_t len) {
        int64_t t = (len + kSubsetTile - 1) / kSubsetTile;
#if TAV_SUBSETS_DEVICE_MUTANT == 1
        if (len > 0 && len % kSubsetTile == 0) --t;
#endif
        return t;
    };
    bool bad = threadIdx.x == 0 && (a.offsets[0] != 0 || a.offsets[a.nq] != a.n_ordinals);
    int64_t tiles = 0;
    for (int q = q0; q < q1; ++q) {  // each offset in [0, n_ordinals] first: no difference below can wrap
        const int64_t lo = a.offsets[q], hi = a.offsets[q + 1];
        if (lo < 0 || hi > a.n_ordinals || hi < lo) bad = true;
        else tiles += tiles_of(hi - lo);
    }
    if (__syncthreads_or(bad)) {  // CTA-uniform
        if (threadIdx.x == 0) {
            atomicOr(a.status, kSubsetBadOffsets);
            *a.n_work = 0;
        }
        return;
    }
    int64_t total;
    int64_t w = plan_scan(tiles, s_warp, &total);
    for (int q = q0; q < q1; ++q) {
        a.work0[q] = w;
        w += tiles_of(a.offsets[q + 1] - a.offsets[q]);
    }
    if (threadIdx.x == 0) {
        a.work0[a.nq] = total;
        *a.n_work = total;
    }
}

cudaError_t launch_subset_plan(const SubsetPlanArgs& a, cudaStream_t s) {
    subset_plan_kernel<<<1, kPlanThreads, 0, s>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_segmented_sort_dev(const SortArgs& a, const int* sizes, int64_t cap, cudaStream_t s, int* launches) {
    const SortBound bd{sizes, cap};
    int n = 0;
    if (a.n_segs > 0 && cap > 0) {
        small_sort_dev_kernel<<<a.n_segs, kSortThreads, 0, s>>>(a, bd);
        ++n;
    }
    if (a.n_large > 0 && a.n_tiles > 0 && cap > 0) {
        const unsigned tiles = static_cast<unsigned>(a.n_tiles);
        radix_minmax_dev_kernel<<<tiles, kSortThreads, 0, s>>>(a, bd);
        for (int p = 0; p < kMaxRadixPasses; ++p) {
            radix_hist_dev_kernel<<<tiles, kSortThreads, 0, s>>>(a, bd, p);
            radix_offsets_dev_kernel<<<a.n_large, kRadixBuckets, 0, s>>>(a, bd, p);
            radix_scatter_dev_kernel<<<tiles, kSortThreads, 0, s>>>(a, bd, p);
        }
        radix_decode_dev_kernel<<<tiles, kSortThreads, 0, s>>>(a, bd);
        n += 2 + 3 * kMaxRadixPasses;
    }
    if (launches) *launches += n;
    return cudaGetLastError();
}

}  // namespace tav
