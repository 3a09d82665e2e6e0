// tav_leaders.cu — grouped lookups (tav_search_groups / tav_range_search_groups): the kernels that turn a query's
// unsorted library keys into the keys of its groups' leaders, and the group map's check.
//
// A group's leader is its row whose key is largest (keys are unique, and their descending order is the library's
// hit order), so the grouped result is the leaders' keys sorted by the segmented sort of the threshold search.
// Leader reduction, per query segment of n keys: an open-addressing table of 2^ceil(log2(2n)) slots (int32 group,
// uint64 key; 12 bytes a slot), so the scratch is O(keys) and never O(queries x groups).
//   claim:   every key claims its group's slot (linear probing, atomicCAS on the group word) and atomicMax-es its
//            key into it; the table is at most half full, so probe runs stay short;
//   compact: every occupied slot holds exactly its group's leader, which is appended to the segment's own keys
//            (in place: the segment is only read by the claim launch before it) through the query's counter.
// Both launches walk a flat space of tiles over every query's keys (slots), so one query with millions of hits is
// spread over the GPU like many small ones.

#include <algorithm>

#include "tav_common.cuh"
#include "tav_internal.h"

namespace tav {

constexpr int kLeaderThreads = 256;
constexpr int kLeaderTile = kLeaderTileKeys;  // keys (slots) per CTA

__device__ __forceinline__ uint32_t group_hash(uint32_t g) {
    g ^= g >> 16;
    g *= 0x7feb352du;
    g ^= g >> 15;
    g *= 0x846ca68bu;
    g ^= g >> 16;
    return g;
}

// the segment of flat tile t: the last q with tile0(q) <= t (segments in ascending tile order)
template <bool kSlots>
__device__ __forceinline__ int leader_seg_of(const LeaderSeg* segs, int nq, int64_t t) {
    int lo = 0, hi = nq - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        const int64_t t0 = kSlots ? segs[mid].slot_tile0 : segs[mid].key_tile0;
        if (t0 <= t) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(kLeaderThreads) leader_claim_kernel(const LeaderSeg* segs, int nq, int64_t n_tiles,
                                                                       const int32_t* groups, int ties_low,
                                                                       int32_t* tgroup, unsigned long long* tkey) {
    for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const LeaderSeg sg = segs[leader_seg_of<false>(segs, nq, t)];
        const int64_t first = (t - sg.key_tile0) * kLeaderTile;
        const int64_t end = min(first + kLeaderTile, sg.n);
        for (int64_t i = first + threadIdx.x; i < end; i += kLeaderThreads) {
            const uint64_t key = sg.keys[i];
            const uint32_t kp = key_pos(key);
            const int32_t g = groups[ties_low ? ~kp : kp];
            uint32_t h = group_hash(static_cast<uint32_t>(g)) & sg.slot_mask;
            for (;;) {
                const int64_t at = sg.slot0 + h;
                const int32_t prev = atomicCAS(&tgroup[at], -1, g);
                if (prev == -1 || prev == g) {
                    atomicMax(&tkey[at], static_cast<unsigned long long>(key));
                    break;
                }
                h = (h + 1) & sg.slot_mask;
            }
        }
    }
}

__global__ void __launch_bounds__(kLeaderThreads) leader_compact_kernel(const LeaderSeg* segs, int nq, int64_t n_tiles,
                                                                         const int32_t* tgroup,
                                                                         const unsigned long long* tkey,
                                                                         uint32_t* counts) {
    __shared__ uint32_t s_n, s_base;
    for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const int q = leader_seg_of<true>(segs, nq, t);
        const LeaderSeg sg = segs[q];
        const int64_t first = (t - sg.slot_tile0) * kLeaderTile;
        const int64_t end = min(first + kLeaderTile, static_cast<int64_t>(sg.slot_mask) + 1);
        if (threadIdx.x == 0) s_n = 0;
        __syncthreads();
        // a tile's leaders are counted in shared memory first (one global atomic per tile), then written
        uint32_t n_mine = 0;
        for (int64_t j = first + threadIdx.x; j < end; j += kLeaderThreads) n_mine += tgroup[sg.slot0 + j] != -1;
        const uint32_t at = n_mine ? atomicAdd(&s_n, n_mine) : 0;
        __syncthreads();
        if (threadIdx.x == 0) s_base = s_n ? atomicAdd(&counts[q], s_n) : 0;
        __syncthreads();
        uint32_t w = s_base + at;
        for (int64_t j = first + threadIdx.x; j < end; j += kLeaderThreads)
            if (tgroup[sg.slot0 + j] != -1) sg.keys[w++] = tkey[sg.slot0 + j];
        __syncthreads();
    }
}

static int leader_grid(int64_t n_tiles) {
    return static_cast<int>(std::min<int64_t>(n_tiles, 132 * 16));
}

cudaError_t launch_leaders(const LeaderSeg* segs, int nq, int64_t key_tiles, int64_t slot_tiles, const int32_t* groups,
                           int ties_low, int32_t* tgroup, uint64_t* tkey, uint32_t* counts, cudaStream_t s) {
    if (nq <= 0 || slot_tiles <= 0) return cudaSuccess;
    auto* tk = reinterpret_cast<unsigned long long*>(tkey);
    if (key_tiles > 0)
        leader_claim_kernel<<<leader_grid(key_tiles), kLeaderThreads, 0, s>>>(segs, nq, key_tiles, groups, ties_low,
                                                                               tgroup, tk);
    leader_compact_kernel<<<leader_grid(slot_tiles), kLeaderThreads, 0, s>>>(segs, nq, slot_tiles, tgroup, tk, counts);
    return cudaGetLastError();
}

// the group map's check: stat[0] |= 1 for a negative value, stat[1] = runs of equal consecutive values
__global__ void group_check_kernel(const int32_t* groups, int64_t n, unsigned long long* stat) {
    unsigned long long bad = 0, runs = 0;
    for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int32_t g = groups[i];
        bad |= g < 0;
        runs += i == 0 || groups[i - 1] != g;
    }
    for (int o = 16; o > 0; o >>= 1) {
        bad |= __shfl_xor_sync(0xffffffffu, bad, o);
        runs += __shfl_xor_sync(0xffffffffu, runs, o);
    }
    if ((threadIdx.x & 31) == 0) {
        if (bad) atomicOr(&stat[0], 1ull);
        if (runs) atomicAdd(&stat[1], runs);
    }
}

cudaError_t launch_group_check(const int32_t* groups, int64_t n, uint64_t* stat, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    const int grid = static_cast<int>(std::min<int64_t>((n + 255) / 256, 132 * 8));
    group_check_kernel<<<grid, 256, 0, s>>>(groups, n, reinterpret_cast<unsigned long long*>(stat));
    return cudaGetLastError();
}

// [nq, k] top-k hits (rows, scores, counts) -> the library's keys of each query's hits, query q's at keys + q * k
__global__ void topk_keys_kernel(int k, const int64_t* rows, const float* scores, const int32_t* counts, int ties_low,
                                 uint64_t* keys) {
    const int q = blockIdx.x;
    const int n = counts[q];
    const size_t base = static_cast<size_t>(q) * k;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const uint32_t p = static_cast<uint32_t>(rows[base + i]);
        keys[base + i] = make_key(scores[base + i], ties_low ? ~p : p);
    }
}

cudaError_t launch_topk_keys(int nq, int k, const int64_t* rows, const float* scores, const int32_t* counts,
                             int ties_low, uint64_t* keys, cudaStream_t s) {
    if (nq <= 0) return cudaSuccess;
    topk_keys_kernel<<<nq, 256, 0, s>>>(k, rows, scores, counts, ties_low, keys);
    return cudaGetLastError();
}

// out_groups[i] = groups[rows[i]] for every row >= 0, -1 for padding
__global__ void group_decode_kernel(int64_t n, const int64_t* rows, const int32_t* groups, int64_t* out_groups) {
    for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int64_t r = rows[i];
        out_groups[i] = r >= 0 ? static_cast<int64_t>(groups[r]) : int64_t(-1);
    }
}

cudaError_t launch_group_decode(int64_t n, const int64_t* rows, const int32_t* groups, int64_t* out_groups,
                                cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    const int grid = static_cast<int>(std::min<int64_t>((n + 255) / 256, 132 * 8));
    group_decode_kernel<<<grid, 256, 0, s>>>(n, rows, groups, out_groups);
    return cudaGetLastError();
}

}  // namespace tav
