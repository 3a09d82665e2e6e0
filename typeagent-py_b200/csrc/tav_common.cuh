// tav_common.cuh — shared device/host helpers of libtavec (sm_90a).
//
// Candidate keys.  Every (row, score) candidate travels as one 64-bit key
//     key = (float_bits(score) << 32) | position
// where score = clip((x + 1) / 2, 0, 1) in float32 (reference: aitools/vectorbase.py:44-47)
// is non-negative, so its IEEE bit pattern is monotone in its value, and `position` is the
// row ordinal (or the position inside the caller's subset).  Sorting keys descending gives
// the library's total order: higher score first, equal scores -> higher position first
// (what numpy's reversed argsort yields for small tied groups, vectorbase.py:184-187).
// Keys are unique per scanned row, which makes the multi-pass "next page" search exact.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace tav {

constexpr int kPassK = 2048;        // most hits one pass returns per query (TAV_PASS_K)
constexpr int kScanThreads = 256;   // row-scan CTA: 8 warps
constexpr int kScanWarps = kScanThreads / 32;
constexpr int kSelectThreads = 256;

// score map, exactly the reference's float32 arithmetic: (x + 1.0f) / 2.0f == (x + 1.0f) * 0.5f
// bit for bit (scaling by a power of two is exact), with the add kept un-fused.
__device__ __forceinline__ float score_from_dot(float x) {
    float s = __fmul_rn(__fadd_rn(x, 1.0f), 0.5f);
    s = s < 0.0f ? 0.0f : s;   // NaN falls through both clamps and is rejected by `s >= floor`
    s = s > 1.0f ? 1.0f : s;
    return s;
}

__device__ __forceinline__ uint64_t make_key(float score, uint32_t pos) {
    return (static_cast<uint64_t>(__float_as_uint(score)) << 32) | pos;
}
__device__ __forceinline__ float key_score(uint64_t key) {
    return __uint_as_float(static_cast<uint32_t>(key >> 32));
}
__device__ __forceinline__ uint32_t key_pos(uint64_t key) { return static_cast<uint32_t>(key); }

// In-place bitonic sort, descending, of n (power of two) keys in shared memory by the whole
// CTA.  Callers pad unused slots with 0 (the smallest key; a real key 0 ties harmlessly).
template <int THREADS>
__device__ __forceinline__ void bitonic_sort_desc(uint64_t* a, int n) {
    for (int size = 2; size <= n; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            __syncthreads();
            for (int t = threadIdx.x; t < (n >> 1); t += THREADS) {
                const int lo = 2 * t - (t & (stride - 1));
                const int hi = lo + stride;
                const bool desc = (lo & size) == 0;
                const uint64_t x = a[lo], y = a[hi];
                if ((x < y) == desc) {
                    a[lo] = y;
                    a[hi] = x;
                }
            }
        }
    }
    __syncthreads();
}

// Shared-memory candidate list of one query, owned by a CTA.  Protocol: pushes happen only
// between two CTA-wide barriers ("a round") and a round pushes at most `round_max` keys.
// list_push() reports whether the list has risen above its watermark (cap - round_max); the
// CTA ORs those reports at the round barrier (__syncthreads_or — exact, because the final
// count is the largest slot any pusher was given) and, when set, every thread takes the slow
// path together and compacts the lists that need it (sort, keep best k, raise the admission
// threshold to just above the k-th key).  One barrier per round in the common case.
struct CandList {
    uint64_t* keys;  // [cap]
    int* count;      // number of keys pushed so far this epoch
    uint64_t* admit; // keys >= *admit are admitted
};

// ---- rank selection: the k best of a SHORT unsorted list without sorting it ------------------------------
// The owner of a key counts the keys greater than it (broadcast reads of shared memory).  Keys are unique,
// so the counts are a permutation and a key of rank < k belongs at out[rank].  O(n^2 / lanes) compares but
// no dependent shuffle chains and next to no barriers: for the <= 256-key lists of the latency path this
// costs a few hundred cycles where a bitonic sort of 128 slots costs 28 CTA barriers (~3 us) and k rounds
// of a shuffle arg-max ~2 us.
__device__ __forceinline__ int rank_among(const uint64_t* in, int n, uint64_t mine) {
    int rank = 0, i = 0;
    for (; i + 2 <= n; i += 2) {  // `in` is 16-byte aligned: one LDS.128 per two keys
        const ulonglong2 p = *reinterpret_cast<const ulonglong2*>(in + i);
        rank += (p.x > mine) + (p.y > mine);
    }
    if (i < n) rank += in[i] > mine;
    return rank;
}

// One warp: the min(n, k) largest of n <= 64 keys, descending, into out (which must not overlap in[0..n)).
__device__ __forceinline__ void warp_rank_select(const uint64_t* in, int n, int k, uint64_t* out) {
    const int lane = threadIdx.x & 31;
    const uint64_t m0 = lane < n ? in[lane] : 0, m1 = lane + 32 < n ? in[lane + 32] : 0;
    int r0 = 0, r1 = 0, i = 0;
    for (; i + 2 <= n; i += 2) {
        const ulonglong2 p = *reinterpret_cast<const ulonglong2*>(in + i);
        r0 += (p.x > m0) + (p.y > m0);
        r1 += (p.x > m1) + (p.y > m1);
    }
    if (i < n) {
        const uint64_t o = in[i];
        r0 += o > m0;
        r1 += o > m1;
    }
    if (lane < n && r0 < k) out[r0] = m0;
    if (lane + 32 < n && r1 < k) out[r1] = m1;
}

// The k (<= 32) largest of `total` <= 4096 unique keys at keys[0..total), by a 256-thread CTA: levels of
// 64-key slices, each reduced to its k best by one warp, until <= 256 keys are left for one CTA-wide rank
// selection.  Every slice but the last is full (64 >= k keys), so the slices' outputs are dense and the next
// level needs no padding.  keys[] must have room for 8192 entries (upper half = ping-pong buffer) and is
// clobbered; callers barrier before (keys filled); out[0..min(total, k)) is valid after the call.
__device__ __forceinline__ void block_rank_topk(uint64_t* keys, int total, int k, uint64_t* out) {
    const int warp = threadIdx.x >> 5;
    uint64_t* in = keys;
    uint64_t* tmp = keys + 4096;
    int n = total;
    while (n > kSelectThreads) {
        const int slices = (n + 63) >> 6;
        for (int s = warp; s < slices; s += kSelectThreads / 32)
            warp_rank_select(in + 64 * s, min(64, n - 64 * s), k, tmp + s * k);
        __syncthreads();
        n = (slices - 1) * k + min(n - 64 * (slices - 1), k);
        uint64_t* t = in;
        in = tmp;
        tmp = t;
    }
    if (static_cast<int>(threadIdx.x) < n) {
        const uint64_t mine = in[threadIdx.x];
        const int rank = rank_among(in, n, mine);
        if (rank < k) out[rank] = mine;
    }
    __syncthreads();
}

template <int THREADS>
__device__ __forceinline__ void list_compact(CandList l, int cap, int k, uint64_t floor_key) {
    // all threads call; *l.count is stable (callers barrier first)
    const int n = min(*l.count, cap);
    if (cap <= THREADS) {
        // short list (one key per thread): rank selection in place, three barriers
        uint64_t mine = 0;
        int rank = k;
        if (static_cast<int>(threadIdx.x) < n) {
            mine = l.keys[threadIdx.x];
            rank = rank_among(l.keys, n, mine);
        }
        __syncthreads();  // every key is in a register, every rank counted
        if (rank < k) l.keys[rank] = mine;
        __syncthreads();
        if (threadIdx.x == 0) {
            const int kept = min(n, k);
            *l.count = kept;
            *l.admit = (kept == k) ? l.keys[k - 1] + 1 : floor_key;
        }
        __syncthreads();
        return;
    }
    for (int i = n + threadIdx.x; i < cap; i += THREADS) l.keys[i] = 0;
    bitonic_sort_desc<THREADS>(l.keys, cap);
    if (threadIdx.x == 0) {
        const int kept = min(n, k);
        *l.count = kept;
        *l.admit = (kept == k) ? l.keys[k - 1] + 1 : floor_key;
    }
    __syncthreads();
}

// returns 1 when the list is now above `watermark` (compaction needed before the next round)
__device__ __forceinline__ int list_push(CandList l, uint64_t key, int watermark) {
    const int slot = atomicAdd(l.count, 1);
    l.keys[slot] = key;  // room guaranteed by the round protocol
    return slot + 1 > watermark;
}

// Warp-aggregated push for kernels where a whole warp feeds ONE list (select / finalize / merge):
// every lane calls it (convergently) with its own `want`; one shared-memory atomic per warp instead
// of one per key.
__device__ __forceinline__ int list_push_warp(CandList l, uint64_t key, bool want, int watermark) {
    const unsigned lanes = __ballot_sync(0xFFFFFFFFu, want);
    if (lanes == 0) return 0;
    const int lane = threadIdx.x & 31;
    const int leader = __ffs(lanes) - 1;
    int base = 0;
    if (lane == leader) base = atomicAdd(l.count, __popc(lanes));
    base = __shfl_sync(0xFFFFFFFFu, base, leader);
    if (want) l.keys[base + __popc(lanes & ((1u << lane) - 1u))] = key;
    return base + __popc(lanes) > watermark;
}

// k largest of `total` unsorted keys in shared memory, WITHOUT sorting them all: a histogram of the
// score bits (kSelBuckets linear buckets between the smallest and the largest score present) locates the
// bucket that holds the k-th key; keys in higher buckets are certain winners, the boundary bucket is
// kept whole, and only those (k + a few) keys are sorted.  ~10 CTA barriers instead of the ~80 of a
// full bitonic sort of 4096 keys.  Returns the number of keys left in `out` (sorted descending, >= k
// unless total < k), or -1 when the survivors do not fit `out_cap` (massive ties: the caller sorts all).
constexpr int kSelBuckets = 1024;
template <int THREADS>
__device__ int select_topk_smem(const uint64_t* keys, int total, int k, uint32_t* hist, uint64_t* out, int out_cap) {
    __shared__ uint32_t s_lo, s_hi, s_bstar, s_n;
    const int tid = threadIdx.x;
    if (tid == 0) {
        s_lo = 0xFFFFFFFFu;
        s_hi = 0u;
        s_n = 0;
    }
    for (int i = tid; i < kSelBuckets; i += THREADS) hist[i] = 0;
    __syncthreads();
    uint32_t lo = 0xFFFFFFFFu, hi = 0u;
    for (int i = tid; i < total; i += THREADS) {
        const uint32_t sb = static_cast<uint32_t>(keys[i] >> 32);
        lo = min(lo, sb);
        hi = max(hi, sb);
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
        lo = min(lo, __shfl_xor_sync(0xFFFFFFFFu, lo, off));
        hi = max(hi, __shfl_xor_sync(0xFFFFFFFFu, hi, off));
    }
    if ((tid & 31) == 0) {
        atomicMin(&s_lo, lo);
        atomicMax(&s_hi, hi);
    }
    __syncthreads();
    lo = s_lo;
    const uint64_t span = static_cast<uint64_t>(s_hi - lo) + 1;
    auto bucket = [&](uint64_t key) {
        return static_cast<uint32_t>((static_cast<uint64_t>(static_cast<uint32_t>(key >> 32) - lo) * kSelBuckets) / span);
    };
    for (int i = tid; i < total; i += THREADS) atomicAdd(&hist[bucket(keys[i])], 1u);
    __syncthreads();
    if (tid < 32) {
        // lane L owns buckets [32L, 32L+32); walk from the top until k keys are covered
        uint32_t mine = 0;
#pragma unroll 8
        for (int j = 0; j < 32; ++j) mine += hist[tid * 32 + j];
        uint32_t above = 0;  // keys in the buckets of the lanes above this one (uniform loop: full-mask shuffles)
        for (int l = 31; l >= 0; --l) {
            const uint32_t m = __shfl_sync(0xFFFFFFFFu, mine, l);
            if (l > tid) above += m;
        }
        if (above < static_cast<uint32_t>(k) && above + mine >= static_cast<uint32_t>(k)) {
            uint32_t acc = above;
            int bsel = tid * 32;
            for (int j = 31; j >= 0; --j) {
                acc += hist[tid * 32 + j];
                if (acc >= static_cast<uint32_t>(k)) {
                    bsel = tid * 32 + j;
                    break;
                }
            }
            s_bstar = static_cast<uint32_t>(bsel);
        }
        if (tid == 0 && total < k) s_bstar = 0;  // fewer keys than k: keep everything
    }
    __syncthreads();
    const uint32_t bstar = s_bstar;
    for (int i0 = 0; i0 < total; i0 += THREADS) {
        const int i = i0 + tid;
        const uint64_t key = i < total ? keys[i] : 0;
        const bool keep = i < total && bucket(key) >= bstar;
        const unsigned m = __ballot_sync(0xFFFFFFFFu, keep);
        if (m) {
            uint32_t base = 0;
            if ((tid & 31) == 0) base = atomicAdd(&s_n, __popc(m));
            base = __shfl_sync(0xFFFFFFFFu, base, 0);
            const uint32_t slot = base + __popc(m & ((1u << (tid & 31)) - 1u));
            if (keep && slot < static_cast<uint32_t>(out_cap)) out[slot] = key;
        }
    }
    __syncthreads();
    const int n = static_cast<int>(s_n);
    if (n > out_cap) return -1;
    int cap = 32;
    while (cap < n) cap <<= 1;
    for (int i = n + tid; i < cap; i += THREADS) out[i] = 0;
    if (cap <= 64) {
        // a handful of survivors: one warp sorts them with warp-level barriers only (a CTA barrier per
        // bitonic pass costs more than the pass)
        __syncthreads();
        if (tid < 32) {
            for (int size = 2; size <= cap; size <<= 1) {
                for (int stride = size >> 1; stride > 0; stride >>= 1) {
                    __syncwarp();
                    for (int t = tid; t < (cap >> 1); t += 32) {
                        const int lo2 = 2 * t - (t & (stride - 1));
                        const int hi2 = lo2 + stride;
                        const bool desc = (lo2 & size) == 0;
                        const uint64_t x = out[lo2], y = out[hi2];
                        if ((x < y) == desc) {
                            out[lo2] = y;
                            out[hi2] = x;
                        }
                    }
                }
            }
        }
        __syncthreads();
    } else {
        bitonic_sort_desc<THREADS>(out, cap);
    }
    return n;
}

// ---- system-scope flags between GPUs (csrc/tav_group.cu: peer-memory candidate exchange) -------------
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
constexpr long long kSpinLimit = 8000000000ll;  // ~4 s of clock64: a lost peer traps instead of hanging the box
// returns once *p has reached `want` (sequence numbers wrap: compared as a signed distance)
__device__ __forceinline__ void spin_until(const uint32_t* p, uint32_t want) {
    const long long t0 = clock64();
    while (static_cast<int32_t>(ld_acquire_sys(p) - want) < 0) {
        if (clock64() - t0 > kSpinLimit) __trap();
        __nanosleep(64);
    }
}

// What a merge of a sharded search waits for and signals (all device pointers; arrive == nullptr: plain merge)
struct MergeSync {
    const uint32_t* arrive;    // [world] sequence number of the last list every rank published into THIS rank's region
    int world;
    uint32_t seq;              // the search being merged
    uint32_t* ack[16];         // ack[w]: this rank's acknowledgement word in rank w's region
    int me;
    uint32_t* ticket;          // device counter (zero on entry, self-resetting): last-CTA-done
    const char* tails;         // slot tails of the world's lists: tails + r * slot_bytes, word 0 = "still to be
                               // corrected", word 1 = status (1: the rank's local search failed, its list is empty)
    size_t slot_bytes;
    uint32_t* flagged_host;    // mapped pinned word receiving the world-wide sum of the tails' word 0
    uint32_t* status_host;     // mapped pinned word receiving the world-wide sum of the tails' word 1
};

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) costs a driver call; remember, per device, the
// largest size already granted to a kernel and only call again to raise it.
template <typename Kernel>
inline cudaError_t ensure_dynamic_smem(Kernel kern, size_t bytes, int (&granted)[16]) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < 16 && static_cast<size_t>(granted[dev]) >= bytes) return cudaSuccess;
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes));
    if (e == cudaSuccess && dev >= 0 && dev < 16) granted[dev] = static_cast<int>(bytes);
    return e;
}

inline int next_pow2(int v) {
    int p = 1;
    while (p < v) p <<= 1;
    return p;
}

// element loaders: storage type -> float
__device__ __forceinline__ float to_float(float v) { return v; }
__device__ __forceinline__ float to_float(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float to_float(__half v) { return __half2float(v); }

}  // namespace tav
