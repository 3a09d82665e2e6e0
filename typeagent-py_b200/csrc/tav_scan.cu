// tav_scan.cu — the CUDA-core "row scan" path of libtavec: exact float32 dot products for a
// handful of queries at a time, HBM-bound (reads every corpus row once per pass).
//
// Replaces, on the GPU, the body of the reference's VectorBase.fuzzy_lookup_embedding /
// fuzzy_lookup_embedding_in_subset (aitools/vectorbase.py:163-230):
//     np.dot(V, e) -> cosine_to_score -> flatnonzero(>= min_score) -> argpartition/argsort
// as ONE fused kernel (dot + score map + threshold + running top-k in shared memory) plus a
// one-CTA-per-query select kernel that merges the per-CTA survivors.  No score vector, mask
// or gather copy is ever materialised.
//
// Layout: corpus row-major [N, D] in HBM (float32 / bf16 / fp16), queries float32 [nq, D]
// staged in shared memory, one warp per row, 4 rows in flight per warp, 16-byte vector loads
// (float4 / 8 x 16-bit) with a scalar fallback for rows that are not 16-byte multiples.
// Algorithmic bytes per pass: n_scan * D * sizeof(storage) (+ nq*D*4 queries, + hits).

#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>

#include "tav_common.cuh"
#include "tav_internal.h"
#include <cstdlib>

namespace tav {

constexpr int kRowsPerWarp = 4;
constexpr int kRoundRows = kScanWarps * kRowsPerWarp;  // 32 rows per CTA round
constexpr int kScanSmemBudget = 160 * 1024;

static inline int scan_cap(int k) {
    int c = next_pow2(2 * k);
    if (c < 128) c = 128;  // >= k + kRoundRows always
    return c;
}
static inline size_t scan_smem_bytes(int qb, int dim, int k, bool fused = false) {
    size_t q_bytes = (static_cast<size_t>(qb) * dim * sizeof(float) + 15) & ~size_t(15);
    size_t lists = static_cast<size_t>(qb) * scan_cap(k) * sizeof(uint64_t);
    // single-launch form: the last CTA's merge needs all survivors + the selection's output and histogram
    if (fused)
        lists = std::max(lists, static_cast<size_t>(kFusedSelectMax) * sizeof(uint64_t) + kFusedSelOut * sizeof(uint64_t) +
                                    kSelBuckets * sizeof(uint32_t));
    return q_bytes + lists;
}

int scan_max_queries(int dim, int k) {
    for (int qb = 8; qb >= 1; qb >>= 1)
        if (scan_smem_bytes(qb, dim, k) <= static_cast<size_t>(kScanSmemBudget)) return qb;
    return 0;
}

// ---- 16-byte row chunk -> floats ---------------------------------------------------------
template <typename T>
struct Vec;
template <>
struct Vec<float> {
    static constexpr int kElems = 4;
    __device__ static __forceinline__ void load(const float* p, float (&f)[4]) {
        const float4 v = __ldcs(reinterpret_cast<const float4*>(p));
        f[0] = v.x, f[1] = v.y, f[2] = v.z, f[3] = v.w;
    }
};
template <>
struct Vec<__nv_bfloat16> {
    static constexpr int kElems = 8;
    __device__ static __forceinline__ void load(const __nv_bfloat16* p, float (&f)[8]) {
        const uint4 v = __ldcs(reinterpret_cast<const uint4*>(p));
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            f[2 * i] = __uint_as_float(w[i] << 16);
            f[2 * i + 1] = __uint_as_float(w[i] & 0xFFFF0000u);
        }
    }
};
template <>
struct Vec<__half> {
    static constexpr int kElems = 8;
    __device__ static __forceinline__ void load(const __half* p, float (&f)[8]) {
        const uint4 v = __ldcs(reinterpret_cast<const uint4*>(p));
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 t = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
            f[2 * i] = t.x, f[2 * i + 1] = t.y;
        }
    }
};

// Butterfly that leaves, in every lane, the warp-wide sum of value (lane >> (5 - log2 NV)):
// 31 shuffles for 32 values instead of 160.
template <int NV>
__device__ __forceinline__ void warp_transpose_reduce(float (&v)[NV], int lane) {
    constexpr unsigned kFull = 0xFFFFFFFFu;
    int n = NV;
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
        if (n > 1) {
            n >>= 1;
            const bool upper = (lane & off) != 0;
#pragma unroll
            for (int i = 0; i < NV / 2; ++i) {
                if (i < n) {
                    const float send = upper ? v[i] : v[i + n];
                    const float keep = upper ? v[i + n] : v[i];
                    v[i] = keep + __shfl_xor_sync(kFull, send, off);
                }
            }
        } else {
            v[0] += __shfl_xor_sync(kFull, v[0], off);
        }
    }
}

// Single-lookup latency form (BLOB != NoBlob): the query vector — and a short subset — travel as
// KERNEL PARAMETERS (no H2D copy, no staging buffer: the launch itself carries them), and the CTA
// that finishes last merges every CTA's survivors and writes the hits (no second launch).
struct NoBlob {
    float q[1];
    int32_t sub[1];
};
template <int QN, int SN>
struct alignas(16) ParamBlob {
    float q[QN];
    int32_t sub[SN > 0 ? SN : 1];
};

// the general form with per-query masks (a.qmask): a tag type, so that the other instantiations stay as they are
struct NoBlobQM : NoBlob {};

template <typename BLOB>
struct BlobTraits {
    static constexpr bool kHas = true;
    static constexpr bool kQMask = false;
};
template <>
struct BlobTraits<NoBlob> {
    static constexpr bool kHas = false;
    static constexpr bool kQMask = false;
};
template <>
struct BlobTraits<NoBlobQM> {
    static constexpr bool kHas = false;
    static constexpr bool kQMask = true;
};

// bit `row` of query q's mask (q < a.nq)
__device__ __forceinline__ bool qmask_bit(const QueryMasks& m, int q, int64_t row) {
    const int64_t r = m.map ? m.map[q] : q;
    return (m.bits[r * m.stride + (row >> 5)] >> (row & 31)) & 1u;
}

__device__ __forceinline__ unsigned long long global_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
#define TAV_STAMP(slot)                                                   \
    do {                                                                  \
        if (a.trace && threadIdx.x == 0) a.trace[(slot)] = global_ns();   \
    } while (0)

// COLLECT (threshold search): no running top-k; every admitted key is appended to its query's region
// (a.cand_keys + q * a.collect_stride) through a per-query counter that keeps counting past the region.
template <typename T, int QB, bool VEC, typename BLOB, bool COLLECT = false>
__global__ void __launch_bounds__(kScanThreads)
scan_rows_kernel(const ScanArgs a, const __grid_constant__ BLOB blob) {
    constexpr bool kBlob = BlobTraits<BLOB>::kHas;
    if (blockIdx.x == 0) TAV_STAMP(0);
    extern __shared__ __align__(16) unsigned char smem_raw[];
    constexpr int NV = kRowsPerWarp * QB;
    const int dim = a.dim;
    const int cap = max(128, 1 << (32 - __clz(2 * a.k - 1)));  // == scan_cap(k)
    float* sq = reinterpret_cast<float*>(smem_raw);
    const size_t q_bytes = (static_cast<size_t>(QB) * dim * sizeof(float) + 15) & ~size_t(15);
    uint64_t* skeys = reinterpret_cast<uint64_t*>(smem_raw + q_bytes);
    __shared__ int s_cnt[QB];
    __shared__ uint64_t s_admit[QB];
    __shared__ uint32_t s_base[QB];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint64_t floor_key = 0;  // the floor itself is tested in float (NaN-safe)

    // stage the queries (zero-fill unused slots)
    if constexpr (kBlob) {
        // 16-byte constant-bank loads (LDC.128): a divergent-index LDC is serialised per lane
        const float4* bq = reinterpret_cast<const float4*>(blob.q);
        float4* sq4 = reinterpret_cast<float4*>(sq);
        for (int i = tid; i < (dim + 3) / 4; i += kScanThreads) sq4[i] = bq[i];
    } else {
        for (int i = tid; i < QB * dim; i += kScanThreads) {
            const int q = i / dim;
            sq[i] = q < a.nq ? a.queries[i] : 0.0f;
        }
    }
    if (tid < QB) {
        s_cnt[tid] = 0;
        s_admit[tid] = floor_key;
    }
    if (blockIdx.x == 0) {
        __syncthreads();
        TAV_STAMP(1);  // query staged
    }

    const T* corpus = reinterpret_cast<const T*>(a.corpus);
    const int64_t n_tiles = (a.n_scan + kRoundRows - 1) / kRoundRows;
    if constexpr (COLLECT) __syncthreads();  // queries staged (no round barriers in this mode)

    int need = 0;  // my last push left a list above its watermark
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        // round barrier: previous pushes visible (first round: queries staged)
        if (!COLLECT && __syncthreads_or(need)) {
            need = 0;
#pragma unroll
            for (int q = 0; q < QB; ++q) {
                if (s_cnt[q] > cap - kRoundRows) {  // CTA-uniform: nobody pushes in here
                    CandList l{skeys + static_cast<size_t>(q) * cap, &s_cnt[q], &s_admit[q]};
                    list_compact<kScanThreads>(l, cap, a.k, floor_key);
                }
            }
        }

        const int64_t pos0 = tile * kRoundRows + warp * kRowsPerWarp;
        const T* rp[kRowsPerWarp];
        int64_t rrow[kRowsPerWarp];
#pragma unroll
        for (int r = 0; r < kRowsPerWarp; ++r) {
            const int64_t pos = pos0 + r;
            int64_t row = 0;
            if (pos < a.n_scan) {
                row = pos;
                if (kBlob && a.subset_in_params) {
                    row = blob.sub[pos];
                    if (row < 0) row += a.n_corpus;
                } else if (a.subset) {
                    row = a.subset[pos];
                    if (row < 0) row += a.n_corpus;  // numpy-style negative ordinals
                }
            }
            rrow[r] = row;
            rp[r] = corpus + row * dim;
        }

        float acc[NV];
#pragma unroll
        for (int i = 0; i < NV; ++i) acc[i] = 0.0f;

        if constexpr (VEC) {
            constexpr int E = Vec<T>::kElems;
            const int nvec = dim / E;
            for (int c = lane; c < nvec; c += 32) {
                float f[kRowsPerWarp][E];
#pragma unroll
                for (int r = 0; r < kRowsPerWarp; ++r) Vec<T>::load(rp[r] + c * E, f[r]);
#pragma unroll
                for (int q = 0; q < QB; ++q) {
                    const float4* q4 = reinterpret_cast<const float4*>(sq + q * dim + c * E);
#pragma unroll
                    for (int h = 0; h < E / 4; ++h) {
                        const float4 qv = q4[h];
#pragma unroll
                        for (int r = 0; r < kRowsPerWarp; ++r) {
                            float s = acc[r * QB + q];
                            s = fmaf(f[r][4 * h + 0], qv.x, s);
                            s = fmaf(f[r][4 * h + 1], qv.y, s);
                            s = fmaf(f[r][4 * h + 2], qv.z, s);
                            s = fmaf(f[r][4 * h + 3], qv.w, s);
                            acc[r * QB + q] = s;
                        }
                    }
                }
            }
        } else {
            for (int c = lane; c < dim; c += 32) {
                float f[kRowsPerWarp];
#pragma unroll
                for (int r = 0; r < kRowsPerWarp; ++r) f[r] = to_float(rp[r][c]);
#pragma unroll
                for (int q = 0; q < QB; ++q) {
                    const float qv = sq[q * dim + c];
#pragma unroll
                    for (int r = 0; r < kRowsPerWarp; ++r)
                        acc[r * QB + q] = fmaf(f[r], qv, acc[r * QB + q]);
                }
            }
        }

        warp_transpose_reduce<NV>(acc, lane);

        constexpr int kLanesPerValue = 32 / NV;
        if constexpr (COLLECT) {
            // same admission as below; the appends of a warp are aggregated per query (one atomic each)
            const int idx = lane / kLanesPerValue;
            const int r = idx / QB, q = idx % QB;
            const int64_t pos = pos0 + r;
            bool want = (lane & (kLanesPerValue - 1)) == 0 && pos < a.n_scan && q < a.nq;
            if (!BlobTraits<BLOB>::kQMask && want && a.row_mask) {
                int64_t row = rrow[0];
#pragma unroll
                for (int rr = 1; rr < kRowsPerWarp; ++rr) row = (r == rr) ? rrow[rr] : row;
                want = (a.row_mask[row >> 5] >> (row & 31)) & 1u;
            }
            if constexpr (BlobTraits<BLOB>::kQMask) {
                if (want) {  // this lane's query's own mask
                    int64_t row = rrow[0];
#pragma unroll
                    for (int rr = 1; rr < kRowsPerWarp; ++rr) row = (r == rr) ? rrow[rr] : row;
                    want = qmask_bit(a.qmask, q, row);
                }
            }
            const float s = score_from_dot(acc[0]);
            want = want && s >= a.floor_score;  // float32 compare, NaN rejected
            const uint32_t p32 = static_cast<uint32_t>(pos);
            const uint64_t key = make_key(s, a.ties_low ? ~p32 : p32);
#pragma unroll
            for (int qq = 0; qq < QB; ++qq) {
                const unsigned m = __ballot_sync(0xFFFFFFFFu, want && q == qq);
                if (m == 0) continue;
                const int leader = __ffs(m) - 1;
                uint32_t base = 0;
                if (lane == leader) base = atomicAdd(&a.cand_count[qq], static_cast<uint32_t>(__popc(m)));
                base = __shfl_sync(0xFFFFFFFFu, base, leader);
                if (want && q == qq) {
                    const uint64_t slot = static_cast<uint64_t>(base) + __popc(m & ((1u << lane) - 1u));
                    if (slot < static_cast<uint64_t>(a.collect_stride))
                        a.cand_keys[static_cast<size_t>(qq) * a.collect_stride + slot] = key;
                }
            }
        } else if ((lane & (kLanesPerValue - 1)) == 0) {
            const int idx = lane / kLanesPerValue;
            const int r = idx / QB, q = idx % QB;
            const int64_t pos = pos0 + r;
            bool allowed = true;
            if (!BlobTraits<BLOB>::kQMask && a.row_mask) {  // predicate pushdown (vectorbase.py:191-201): one bit per corpus row
                int64_t row = rrow[0];
#pragma unroll
                for (int rr = 1; rr < kRowsPerWarp; ++rr) row = (r == rr) ? rrow[rr] : row;
                allowed = (a.row_mask[row >> 5] >> (row & 31)) & 1u;
            }
            if constexpr (BlobTraits<BLOB>::kQMask) {
                if (pos < a.n_scan && q < a.nq) {  // this lane's query's own mask (padding lanes read nothing)
                    int64_t row = rrow[0];
#pragma unroll
                    for (int rr = 1; rr < kRowsPerWarp; ++rr) row = (r == rr) ? rrow[rr] : row;
                    allowed = qmask_bit(a.qmask, q, row);
                }
            }
            if (pos < a.n_scan && q < a.nq && allowed) {
                const float s = score_from_dot(acc[0]);
                if (s >= a.floor_score) {  // float32 compare, as vectorbase.py:179
                    // ties_low: among equal scores the LOWER position sorts first (the reference's
                    // stable sort on the predicate path), else the higher one (its argsort path)
                    const uint32_t p32 = static_cast<uint32_t>(pos);
                    const uint64_t key = make_key(s, a.ties_low ? ~p32 : p32);
                    if (key >= s_admit[q] && (a.bound == nullptr || key < a.bound[q])) {
                        CandList l{skeys + static_cast<size_t>(q) * cap, &s_cnt[q], &s_admit[q]};
                        need |= list_push(l, key, cap - kRoundRows);
                    }
                }
            }
        }
    }

    if constexpr (COLLECT) return;

    // hand the CTA's best k per query to the global candidate buffers
    __syncthreads();
    if (blockIdx.x == 0) TAV_STAMP(2);  // rows scanned
#pragma unroll
    for (int q = 0; q < QB; ++q) {
        if (q >= a.nq) break;
        CandList l{skeys + static_cast<size_t>(q) * cap, &s_cnt[q], &s_admit[q]};
        // Hand over the CTA's best k (rank selection when the list is short: three barriers, no sort), so that
        // the last CTA of the single-launch form merges grid * k keys and not grid * (a round's worth).
        const int have = s_cnt[q];  // read by every thread BEFORE thread 0 may rewrite it (racecheck: the branch
        __syncthreads();            // below must see one value in all warps, or the barriers inside it diverge)
        if (have > a.k) list_compact<kScanThreads>(l, cap, a.k, floor_key);  // CTA-uniform
        const int n = s_cnt[q];
        if (tid == 0 && n > 0) s_base[q] = atomicAdd(&a.cand_count[q], static_cast<uint32_t>(n));
        __syncthreads();
        if (n > 0) {
            uint64_t* dst = a.cand_keys + static_cast<size_t>(q) * a.cand_stride + s_base[q];
            for (int i = tid; i < n; i += kScanThreads) dst[i] = l.keys[i];
        }
    }

    if (a.fused) {
        // ---- last CTA done: merge every CTA's survivors, write the hits, raise the host flag ----
        __shared__ int s_is_last;
        __threadfence();
        __syncthreads();
        if (tid == 0) {
            const uint32_t t = atomicAdd(a.fused_ticket, 1u);
            s_is_last = t == gridDim.x - 1;
            if (s_is_last) *a.fused_ticket = 0;  // ready for the next search
        }
        __syncthreads();
        if (blockIdx.x == 0) TAV_STAMP(3);  // survivors handed over
        if (!s_is_last) return;
        TAV_STAMP(4);  // last CTA starts the merge
        __threadfence();
        uint64_t* keys = skeys;  // the lists are dead now; room for kFusedSelectMax keys was reserved
        for (int q = 0; q < a.nq; ++q) {
            const int total = static_cast<int>(min(__ldcg(&a.cand_count[q]), static_cast<uint32_t>(a.cand_stride)));
            int cap2 = 32;
            while (cap2 < total) cap2 <<= 1;
            const uint64_t* in = a.cand_keys + static_cast<size_t>(q) * a.cand_stride;
            __syncthreads();
            for (int i0 = tid; i0 < total; i0 += 4 * kScanThreads) {  // four independent loads in flight per thread
                uint64_t e[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) e[u] = i0 + u * kScanThreads < total ? __ldcg(&in[i0 + u * kScanThreads]) : 0;
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    if (i0 + u * kScanThreads < total) keys[i0 + u * kScanThreads] = e[u];
            }
            __syncthreads();
            // k best of the survivors: histogram selection (a dozen barriers) instead of a full sort
            uint64_t* sel_out = keys + kFusedSelectMax;
            uint32_t* hist = reinterpret_cast<uint32_t*>(sel_out + kFusedSelOut);
            const uint64_t* result = keys;
            int n = -1;
            if (a.k <= 32 && total <= 4096) {
                // the latency case (few survivors, small k): levels of rank selection, no sort
                block_rank_topk(keys, total, a.k, sel_out);
                result = sel_out;
                n = min(total, a.k);
            } else if (total > 256 && a.k <= kFusedSelOut / 2) {
                const int got = select_topk_smem<kScanThreads>(keys, total, a.k, hist, sel_out, kFusedSelOut);
                if (got >= 0) {
                    n = min(got, a.k);
                    result = sel_out;
                }
            }
            if (n < 0) {
                for (int i = total + tid; i < cap2; i += kScanThreads) keys[i] = 0;
                bitonic_sort_desc<kScanThreads>(keys, cap2);
                n = min(total, a.k);
            }
            int64_t* items = a.out_items + static_cast<size_t>(q) * a.k;
            float* scores = a.out_scores + static_cast<size_t>(q) * a.k;
            for (int j = tid; j < a.k; j += kScanThreads) {
                int64_t item = -1;
                float sc = 0.0f;
                if (j < n) {
                    const uint32_t kp = key_pos(result[j]);
                    const uint32_t pos = a.ties_low ? ~kp : kp;
                    if (a.items_as_positions) item = pos;
                    else if (kBlob && a.subset_in_params) item = blob.sub[pos];
                    else item = a.subset ? a.subset[pos] : static_cast<int64_t>(pos);
                    item += a.item_offset;
                    sc = key_score(result[j]);
                }
                items[j] = item;
                scores[j] = sc;
            }
            if (tid == 0) {
                a.out_counts[q] = n;
                a.cand_count[q] = 0;
            }
        }
        TAV_STAMP(5);  // hits written
        if (a.done_flag) {
            // ONE system-scope fence, by the thread that raises the completion word: the barrier orders the
            // other threads' result stores before it (a membar.sys per thread cost ~20 us here: each waits
            // for the outstanding PCIe writes)
            __syncthreads();
            if (tid == 0) {
                __threadfence_system();
                *reinterpret_cast<volatile uint32_t*>(a.done_flag) = a.done_seq;
            }
        }
        TAV_STAMP(6);  // completion word raised
    }
}

int scan_grid(int device, int dtype, int dim, int nq, int k, int64_t n_scan) {
    (void)dtype;
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    const size_t smem = scan_smem_bytes(nq, dim, k);
    int per_sm = static_cast<int>((200 * 1024) / (smem + 1024));
    if (per_sm > 4) per_sm = 4;   // 32 warps x 4 rows in flight already covers HBM latency
    if (per_sm < 1) per_sm = 1;
    int64_t tiles = (n_scan + kRoundRows - 1) / kRoundRows;
    int64_t g = static_cast<int64_t>(sms) * per_sm;
    if (g > tiles) g = tiles;
    if (g < 1) g = 1;
    return static_cast<int>(g);
}

template <typename T, int QB, typename BLOB>
static cudaError_t launch_scan_t(const ScanArgs& a, const BLOB& blob, cudaStream_t s) {
    const size_t row_bytes = static_cast<size_t>(a.dim) * sizeof(T);
    const bool vec = (row_bytes % 16 == 0) && (reinterpret_cast<uintptr_t>(a.corpus) % 16 == 0);
    const size_t smem = scan_smem_bytes(QB, a.dim, a.k, a.fused != 0);
    auto kern = vec ? scan_rows_kernel<T, QB, true, BLOB> : scan_rows_kernel<T, QB, false, BLOB>;
    static int granted[2][16] = {};
    cudaError_t e = ensure_dynamic_smem(kern, smem, granted[vec ? 1 : 0]);
    if (e != cudaSuccess) return e;
    kern<<<a.grid, kScanThreads, smem, s>>>(a, blob);
    return cudaGetLastError();
}

template <typename T, typename BLOB>
static cudaError_t launch_scan_b(const ScanArgs& a, cudaStream_t s) {
    const BLOB none{};
    if (a.nq <= 1) return launch_scan_t<T, 1>(a, none, s);
    if (a.nq <= 2) return launch_scan_t<T, 2>(a, none, s);
    if (a.nq <= 4) return launch_scan_t<T, 4>(a, none, s);
    return launch_scan_t<T, 8>(a, none, s);
}

template <typename T>
static cudaError_t launch_scan_q(const ScanArgs& a, cudaStream_t s) {
    if (a.qmask.bits) return launch_scan_b<T, NoBlobQM>(a, s);
    return launch_scan_b<T, NoBlob>(a, s);
}

cudaError_t launch_scan(const ScanArgs& a, cudaStream_t s) {
    switch (a.dtype) {
        case TAV_F32: return launch_scan_q<float>(a, s);
        case TAV_BF16: return launch_scan_q<__nv_bfloat16>(a, s);
        case TAV_F16: return launch_scan_q<__half>(a, s);
    }
    return cudaErrorInvalidValue;
}

// ---- collect mode (threshold search): shared memory holds only the queries ---------------------
static inline size_t collect_smem_bytes(int qb, int dim) {
    return (static_cast<size_t>(qb) * dim * sizeof(float) + 15) & ~size_t(15);
}

int scan_collect_max_queries(int dim) {
    for (int qb = 8; qb >= 1; qb >>= 1)
        if (collect_smem_bytes(qb, dim) <= static_cast<size_t>(kScanSmemBudget)) return qb;
    return 0;
}

int scan_collect_grid(int device, int dim, int nq, int64_t n_scan) {
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    int per_sm = static_cast<int>((200 * 1024) / (collect_smem_bytes(nq, dim) + 1024));
    per_sm = std::max(1, std::min(per_sm, 4));
    const int64_t tiles = (n_scan + kRoundRows - 1) / kRoundRows;
    return static_cast<int>(std::max<int64_t>(1, std::min<int64_t>(tiles, static_cast<int64_t>(sms) * per_sm)));
}

template <typename T, int QB, typename BLOB>
static cudaError_t launch_collect_t(const ScanArgs& a, cudaStream_t s) {
    const size_t row_bytes = static_cast<size_t>(a.dim) * sizeof(T);
    const bool vec = (row_bytes % 16 == 0) && (reinterpret_cast<uintptr_t>(a.corpus) % 16 == 0);
    const size_t smem = collect_smem_bytes(QB, a.dim);
    auto kern = vec ? scan_rows_kernel<T, QB, true, BLOB, true> : scan_rows_kernel<T, QB, false, BLOB, true>;
    static int granted[2][16] = {};
    cudaError_t e = ensure_dynamic_smem(kern, smem, granted[vec ? 1 : 0]);
    if (e != cudaSuccess) return e;
    kern<<<a.grid, kScanThreads, smem, s>>>(a, BLOB{});
    return cudaGetLastError();
}

template <typename T, typename BLOB>
static cudaError_t launch_collect_b(const ScanArgs& a, cudaStream_t s) {
    if (a.nq <= 1) return launch_collect_t<T, 1, BLOB>(a, s);
    if (a.nq <= 2) return launch_collect_t<T, 2, BLOB>(a, s);
    if (a.nq <= 4) return launch_collect_t<T, 4, BLOB>(a, s);
    return launch_collect_t<T, 8, BLOB>(a, s);
}

template <typename T>
static cudaError_t launch_collect_q(const ScanArgs& a, cudaStream_t s) {
    if (a.qmask.bits) return launch_collect_b<T, NoBlobQM>(a, s);
    return launch_collect_b<T, NoBlob>(a, s);
}

// one CTA per mask row: the set bits of its first n_rows
__global__ void __launch_bounds__(256)
mask_popcount_kernel(const uint32_t* __restrict__ bits, int64_t n_rows, int64_t stride, uint32_t* pop) {
    __shared__ uint32_t s_part[8];
    const int tid = threadIdx.x, lane = tid & 31;
    const uint32_t* row = bits + static_cast<int64_t>(blockIdx.x) * stride;
    const int64_t words = (n_rows + 31) / 32;
    const uint32_t last = (n_rows & 31) ? (1u << (n_rows & 31)) - 1u : 0xFFFFFFFFu;
    uint32_t c = 0;
    for (int64_t i = tid; i < words; i += 256) c += __popc(i == words - 1 ? row[i] & last : row[i]);
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) c += __shfl_xor_sync(0xFFFFFFFFu, c, off);
    if (lane == 0) s_part[tid >> 5] = c;
    __syncthreads();
    if (tid == 0) {
        uint32_t t = 0;
        for (int w = 0; w < 8; ++w) t += s_part[w];
        pop[blockIdx.x] = t;
    }
}

cudaError_t launch_mask_popcount(const uint32_t* bits, int n_masks, int64_t n_rows, int64_t stride, uint32_t* pop,
                                 cudaStream_t s) {
    if (n_masks <= 0) return cudaSuccess;
    mask_popcount_kernel<<<n_masks, 256, 0, s>>>(bits, n_rows, stride, pop);
    return cudaGetLastError();
}

cudaError_t launch_scan_collect(const ScanArgs& a, cudaStream_t s) {
    switch (a.dtype) {
        case TAV_F32: return launch_collect_q<float>(a, s);
        case TAV_BF16: return launch_collect_q<__nv_bfloat16>(a, s);
        case TAV_F16: return launch_collect_q<__half>(a, s);
    }
    return cudaErrorInvalidValue;
}

// ---- per-query subsets: one gather over a batch whose queries score different rows ---------------
// Each (query, entry) dot is computed as the row scan computes it with one query per pass (QB = 1): the same
// lane-strided loads, fmaf order and warp_transpose_reduce<4> tree, so row b of a batch equals the one-query
// subset search bit for bit.  A CTA walks work items (query, tile); it stages a query only when the query changes.
// The device-planned form (kDev, tav_search_subsets_into) reads the planned item count and checks each ordinal
// against [-n_corpus, n_corpus) before it forms a row address: an entry outside sets the status word and row 0 is
// read in its place (the search is refused).  The <false> instantiation is the host-planned kernel, unchanged.
struct SubsetDev {
    const int64_t* n_work;  // device: the planned item count
    int* status;
};
template <typename T, bool VEC, bool kDev>
__device__ __forceinline__ void subset_gather(const SubsetArgs& a, const SubsetDev& d) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* sq = reinterpret_cast<float*>(smem_raw);
    __shared__ int s_q;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int dim = a.dim;
    const T* corpus = reinterpret_cast<const T*>(a.corpus);
    const int64_t n_work = kDev ? *d.n_work : a.n_work;
    int cur = -1;
    for (int64_t w = blockIdx.x; w < n_work; w += gridDim.x) {
        __syncthreads();  // the previous item is done with s_q and sq
        if (tid == 0) {   // the query of item w: the last q with work0[q] <= w
            int lo = 0, hi = a.nq - 1;
            while (lo < hi) {
                const int mid = (lo + hi + 1) >> 1;
                if (a.work0[mid] <= w) lo = mid;
                else hi = mid - 1;
            }
            s_q = lo;
        }
        __syncthreads();
        const int q = s_q;
        if (q != cur) {  // CTA-uniform
            for (int i = tid; i < dim; i += kScanThreads) sq[i] = a.queries[static_cast<size_t>(q) * dim + i];
            __syncthreads();
            cur = q;
        }
        const int64_t q_begin = a.offsets[q], q_end = a.offsets[q + 1];
        int64_t begin = q_begin + (w - a.work0[q]) * kSubsetTile;
#if TAV_SUBSETS_MUTANT == 1
        if (w > a.work0[q] && (q_end - q_begin) % kSubsetTile != 0) ++begin;
#endif
        const int64_t end = min(begin + kSubsetTile, q_end);
        uint64_t* qkeys = a.keys + q_begin;
        for (int64_t pos0 = begin + warp * kRowsPerWarp; pos0 < end; pos0 += kRoundRows) {  // warp-uniform
            const T* rp[kRowsPerWarp];
#pragma unroll
            for (int r = 0; r < kRowsPerWarp; ++r) {
                int64_t row = 0;
                if (pos0 + r < end) {
                    row = a.ordinals[pos0 + r];
                    if (kDev && (row < -a.n_corpus || row >= a.n_corpus)) {
                        atomicOr(d.status, kSubsetBadOrdinal);
                        row = 0;
                    }
                    if (row < 0) row += a.n_corpus;  // numpy-style negative ordinals
                }
                rp[r] = corpus + row * dim;
            }
            float acc[kRowsPerWarp];
#pragma unroll
            for (int r = 0; r < kRowsPerWarp; ++r) acc[r] = 0.0f;
            if constexpr (VEC) {
                constexpr int E = Vec<T>::kElems;
                const int nvec = dim / E;
                for (int c = lane; c < nvec; c += 32) {
                    float f[kRowsPerWarp][E];
#pragma unroll
                    for (int r = 0; r < kRowsPerWarp; ++r) Vec<T>::load(rp[r] + c * E, f[r]);
                    const float4* q4 = reinterpret_cast<const float4*>(sq + c * E);
#pragma unroll
                    for (int h = 0; h < E / 4; ++h) {
                        const float4 qv = q4[h];
#pragma unroll
                        for (int r = 0; r < kRowsPerWarp; ++r) {
                            float s = acc[r];
                            s = fmaf(f[r][4 * h + 0], qv.x, s);
                            s = fmaf(f[r][4 * h + 1], qv.y, s);
                            s = fmaf(f[r][4 * h + 2], qv.z, s);
                            s = fmaf(f[r][4 * h + 3], qv.w, s);
                            acc[r] = s;
                        }
                    }
                }
            } else {
                for (int c = lane; c < dim; c += 32) {
                    float f[kRowsPerWarp];
#pragma unroll
                    for (int r = 0; r < kRowsPerWarp; ++r) f[r] = to_float(rp[r][c]);
                    const float qv = sq[c];
#pragma unroll
                    for (int r = 0; r < kRowsPerWarp; ++r) acc[r] = fmaf(f[r], qv, acc[r]);
                }
            }
            warp_transpose_reduce<kRowsPerWarp>(acc, lane);

            // lane 8r holds entry pos0 + r; the warp's admitted keys take one atomic
            constexpr int kLanesPerValue = 32 / kRowsPerWarp;
            const int64_t pos = pos0 + lane / kLanesPerValue;
            const float s = score_from_dot(acc[0]);
            const bool want = (lane & (kLanesPerValue - 1)) == 0 && pos < end && s >= a.floor_score;  // NaN rejected
            const unsigned m = __ballot_sync(0xFFFFFFFFu, want);
            if (m == 0) continue;
            const int leader = __ffs(m) - 1;
            uint32_t base = 0;
            if (lane == leader) base = atomicAdd(&a.counts[q], static_cast<uint32_t>(__popc(m)));
            base = __shfl_sync(0xFFFFFFFFu, base, leader);
            if (want) {
                const uint32_t j = static_cast<uint32_t>(pos)  // flat index into the ordinals (< 2^32)
#if TAV_SCALE_MUTANT == 2
                                   & 0xFFFFFFu
#endif
                    ;
                qkeys[base + __popc(m & ((1u << lane) - 1u))] = make_key(s, a.ties_low ? ~j : j);
            }
        }
    }
}

template <typename T, bool VEC>
__global__ void __launch_bounds__(kScanThreads) subset_gather_kernel(const SubsetArgs a) {
    subset_gather<T, VEC, false>(a, SubsetDev{});
}
template <typename T, bool VEC>
__global__ void __launch_bounds__(kScanThreads) subset_gather_dev_kernel(const SubsetArgs a, const SubsetDev d) {
    subset_gather<T, VEC, true>(a, d);
}

// one wave of as many CTAs as fit per SM (at most 4, the row scan's occupancy); the items are grid-strided
template <typename Kern, typename... Args>
static cudaError_t launch_gather_wave(Kern kern, int (&granted)[16], size_t smem, int64_t n_work, cudaStream_t s,
                                      Args... args) {
    cudaError_t e = ensure_dynamic_smem(kern, smem, granted);
    if (e != cudaSuccess) return e;
    int device = 0, sms = 132, per_sm = 1;
    if ((e = cudaGetDevice(&device)) != cudaSuccess) return e;
    if ((e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device)) != cudaSuccess) return e;
    if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kScanThreads, smem)) != cudaSuccess) return e;
    per_sm = std::max(1, std::min(per_sm, 4));
    const int grid = static_cast<int>(std::min<int64_t>(n_work, static_cast<int64_t>(sms) * per_sm));
    kern<<<grid, kScanThreads, smem, s>>>(args...);
    return cudaGetLastError();
}

// d: the device-planned form (nullptr: the host-planned one)
template <typename T>
static cudaError_t launch_subset_gather_t(const SubsetArgs& a, const SubsetDev* d, cudaStream_t s) {
    const size_t row_bytes = static_cast<size_t>(a.dim) * sizeof(T);
    const bool vec = (row_bytes % 16 == 0) && (reinterpret_cast<uintptr_t>(a.corpus) % 16 == 0);
    const size_t smem = collect_smem_bytes(1, a.dim);
    static int granted[4][16] = {};
    int (&g)[16] = granted[(vec ? 1 : 0) + (d ? 2 : 0)];
    if (d)
        return launch_gather_wave(vec ? subset_gather_dev_kernel<T, true> : subset_gather_dev_kernel<T, false>, g, smem,
                                  a.n_work, s, a, *d);
    return launch_gather_wave(vec ? subset_gather_kernel<T, true> : subset_gather_kernel<T, false>, g, smem, a.n_work, s,
                              a);
}

static cudaError_t launch_subset_gather_any(const SubsetArgs& a, const SubsetDev* d, cudaStream_t s) {
    if (a.n_work == 0) return cudaSuccess;
    switch (a.dtype) {
        case TAV_F32: return launch_subset_gather_t<float>(a, d, s);
        case TAV_BF16: return launch_subset_gather_t<__nv_bfloat16>(a, d, s);
        case TAV_F16: return launch_subset_gather_t<__half>(a, d, s);
    }
    return cudaErrorInvalidValue;
}

cudaError_t launch_subset_gather(const SubsetArgs& a, cudaStream_t s) { return launch_subset_gather_any(a, nullptr, s); }

cudaError_t launch_subset_gather_dev(const SubsetArgs& a, const int64_t* n_work, int* status, cudaStream_t s) {
    const SubsetDev d{n_work, status};
    return launch_subset_gather_any(a, &d, s);
}

// one CTA per query
__global__ void __launch_bounds__(256)
subset_topk_layout_kernel(int k, const int64_t* __restrict__ csr_offsets, const int64_t* __restrict__ hits,
                          const float* __restrict__ hit_scores, int64_t* out_items, float* out_scores,
                          int32_t* out_counts) {
    const int q = blockIdx.x;
    const int64_t first = csr_offsets[q];
    const int n = static_cast<int>(min(static_cast<int64_t>(k), csr_offsets[q + 1] - first));
    int64_t* items = out_items + static_cast<size_t>(q) * k;
    float* scores = out_scores + static_cast<size_t>(q) * k;
    for (int j = threadIdx.x; j < k; j += 256) {
        items[j] = j < n ? hits[first + j] : -1;
        scores[j] = j < n ? hit_scores[first + j] : 0.0f;
    }
    if (threadIdx.x == 0) out_counts[q] = n;
}

cudaError_t launch_subset_topk_layout(int nq, int k, const int64_t* csr_offsets, const int64_t* hits,
                                      const float* hit_scores, int64_t* out_items, float* out_scores,
                                      int32_t* out_counts, cudaStream_t s) {
    if (nq <= 0) return cudaSuccess;
    subset_topk_layout_kernel<<<nq, 256, 0, s>>>(k, csr_offsets, hits, hit_scores, out_items, out_scores, out_counts);
    return cudaGetLastError();
}

// ---- single-lookup latency form: query (and a short subset) in the kernel parameters ----------
using SmallBlob = ParamBlob<kParamQuerySmall, 0>;                   // 4 KB of parameters
using MidBlob = ParamBlob<kParamQuerySmall, kParamSubsetSmall>;    // 8 KB
using BigBlob = ParamBlob<kParamQueryBig, kParamSubsetMax>;        // 28 KB

bool scan1_fits(int dim, int k, int64_t n_scan, int64_t subset_len, bool has_subset) {
    if (dim > kParamQueryBig) return false;
    if (has_subset && subset_len > kParamSubsetMax) return false;
    // the last CTA sorts every CTA's k survivors at once: a full wave of CTAs must fit its buffer
    const int64_t tiles = (n_scan + kRoundRows - 1) / kRoundRows;
    return static_cast<int64_t>(k) * std::min<int64_t>(tiles, 132) <= kFusedSelectMax;
}

int scan1_grid(int device, int dim, int k, int64_t n_scan) {
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    int64_t tiles = (n_scan + kRoundRows - 1) / kRoundRows;
    // up to 4 CTAs per SM (the general form's occupancy), one round of rows per CTA while the rows last.  The
    // last CTA merges grid * k survivors: its buffer bounds the grid, and for the rank-selection merge (k <= 32)
    // so does its cost, which grows with the survivors; 2048 survivors balance that merge against the rounds of
    // rows per CTA (TAV_SCAN1_SURVIVORS overrides it).
    int64_t g = std::min<int64_t>(tiles, 4ll * sms);
    static const int64_t survivors_env = [] {
        const char* e = getenv("TAV_SCAN1_SURVIVORS");  // tuning knob for that sweep
        return e ? std::max<int64_t>(atoll(e), 0) : 0;
    }();
    int64_t survivors_max = k <= 32 ? 2048 : kFusedSelectMax;
    if (survivors_env > 0) survivors_max = std::min<int64_t>(survivors_env, kFusedSelectMax);
    g = std::min<int64_t>(g, survivors_max / std::max(k, 1));
    (void)dim;
    return static_cast<int>(std::max<int64_t>(g, 1));
}

template <typename T, typename BLOB>
static cudaError_t launch_scan1_t(const ScanArgs& a, const float* q_host, const int64_t* sub_host, cudaStream_t s) {
    // the blob is filled on the host stack and copied into the launch's parameter buffer
    static thread_local BLOB blob;
    memcpy(blob.q, q_host, static_cast<size_t>(a.dim) * sizeof(float));
    if (sub_host)
        for (int64_t i = 0; i < a.n_scan; ++i) blob.sub[i] = static_cast<int32_t>(sub_host[i]);
    return launch_scan_t<T, 1>(a, blob, s);
}

template <typename T>
static cudaError_t launch_scan1_d(const ScanArgs& a, const float* q_host, const int64_t* sub_host, cudaStream_t s) {
    // the smallest parameter blob that holds the query (and the subset): the launch copies all of it
    if (a.dim <= kParamQuerySmall && !sub_host) return launch_scan1_t<T, SmallBlob>(a, q_host, sub_host, s);
    if (a.dim <= kParamQuerySmall && a.n_scan <= kParamSubsetSmall) return launch_scan1_t<T, MidBlob>(a, q_host, sub_host, s);
    return launch_scan1_t<T, BigBlob>(a, q_host, sub_host, s);
}

cudaError_t launch_scan1(const ScanArgs& a, const float* q_host, const int64_t* sub_host, cudaStream_t s) {
    switch (a.dtype) {
        case TAV_F32: return launch_scan1_d<float>(a, q_host, sub_host, s);
        case TAV_BF16: return launch_scan1_d<__nv_bfloat16>(a, q_host, sub_host, s);
        case TAV_F16: return launch_scan1_d<__half>(a, q_host, sub_host, s);
    }
    return cudaErrorInvalidValue;
}

// ---- select: per query, best k of the global candidate buffer, sorted, decoded -----------
static inline int select_cap(int k) { return next_pow2(k + kSelectThreads); }

__global__ void __launch_bounds__(kSelectThreads) select_kernel(const SelectArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint64_t* keys = reinterpret_cast<uint64_t*>(smem_raw);
    __shared__ int s_cnt;
    __shared__ uint64_t s_admit;
    const int q = blockIdx.x, tid = threadIdx.x;
    const int cap = 1 << (32 - __clz(a.k + kSelectThreads - 1));
    const uint32_t total = min(a.cand_count[q], static_cast<uint32_t>(a.cand_stride));
    const uint64_t* in = a.cand_keys + static_cast<size_t>(q) * a.cand_stride;
    if (tid == 0) {
        s_cnt = 0;
        s_admit = 0;
    }
    CandList l{keys, &s_cnt, &s_admit};
    int need = 0;
    for (uint32_t base = 0; base < total; base += kSelectThreads) {
        if (__syncthreads_or(need)) {
            need = 0;
            list_compact<kSelectThreads>(l, cap, a.k, 0);
        }
        const uint32_t i = base + tid;
        const uint64_t key = i < total ? in[i] : 0;
        need |= list_push_warp(l, key, i < total && key >= s_admit, cap - kSelectThreads);
    }
    __syncthreads();
    list_compact<kSelectThreads>(l, cap, a.k, 0);  // final sort (also when total == 0)
    const int n = s_cnt;
    int64_t* items = a.out_items + static_cast<size_t>(q) * a.out_stride + a.out_offset;
    float* scores = a.out_scores + static_cast<size_t>(q) * a.out_stride + a.out_offset;
    for (int j = tid; j < a.k; j += kSelectThreads) {
        if (j < n) {
            const uint64_t key = keys[j];
            const uint32_t pos = a.ties_low ? ~key_pos(key) : key_pos(key);
            const int64_t item = a.subset ? a.subset[pos] : static_cast<int64_t>(pos);
            items[j] = item + a.item_offset;
            scores[j] = key_score(key);
        } else {
            items[j] = -1;
            scores[j] = 0.0f;
        }
    }
    if (tid == 0) {
        a.out_counts[q] = a.accumulate ? a.out_counts[q] + n : n;
        if (a.bound_out) a.bound_out[q] = (n == a.k) ? keys[a.k - 1] : 0;
        a.cand_count_reset[q] = 0;  // ready for the next pass: no memset between launches
    }
}

cudaError_t launch_select(const SelectArgs& a, cudaStream_t s) {
    const size_t smem = static_cast<size_t>(select_cap(a.k)) * sizeof(uint64_t);
    static int granted[16] = {};
    cudaError_t e = ensure_dynamic_smem(select_kernel, smem, granted);
    if (e != cudaSuccess) return e;
    select_kernel<<<a.nq, kSelectThreads, smem, s>>>(a);
    return cudaGetLastError();
}

// ---- merge of per-shard results (after the candidate all-gather) -------------------------
// ORDER 0: key low word = list * k + (k - 1 - j): among equal scores a later shard (higher rows) and,
// inside a shard, an earlier slot (higher row) sorts first — the same total order as one GPU.
// ORDER 1: ~(list * k + j): an earlier shard and an earlier slot first (lists searched ties-low-first).
// ORDER 2 / 3: the item itself (a global subset position < 2^32), or its complement: higher / lower first;
// the decoded item is the key's low word, the items array is only read for the keys.
template <int ORDER>
__global__ void __launch_bounds__(kSelectThreads)
merge_kernel(int n_lists, int n_queries, int k, const int64_t* items, const float* scores,
             const int32_t* counts, int64_t items_stride, int64_t scores_stride,
             int64_t counts_stride, int64_t* out_items, float* out_scores, int32_t* out_counts, const MergeSync sync) {
    constexpr bool kPosKey = ORDER >= 2 && TAV_SHARDED_FILTER_MUTANT != 2;
    constexpr bool kLowFirst = ORDER == 1 || (ORDER == 3 && !kPosKey);
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint64_t* keys = reinterpret_cast<uint64_t*>(smem_raw);
    __shared__ int s_cnt;
    __shared__ uint64_t s_admit;
    const int q = blockIdx.x, tid = threadIdx.x;
    if (sync.arrive) {  // sharded search: every rank's list for this search must have landed in this rank's region
        if (tid < sync.world) spin_until(sync.arrive + tid, sync.seq);
        __syncthreads();
    }
    const int cap = 1 << (32 - __clz(k + kSelectThreads - 1));
    if (tid == 0) {
        s_cnt = 0;
        s_admit = 0;
    }
    CandList l{keys, &s_cnt, &s_admit};
    const int64_t total = static_cast<int64_t>(n_lists) * k;
    int need = 0;
    for (int64_t base = 0; base < total; base += kSelectThreads) {
        if (__syncthreads_or(need)) {
            need = 0;
            list_compact<kSelectThreads>(l, cap, k, 0);
        }
        const int64_t i = base + tid;
        uint64_t key = 0;
        bool want = false;
        if (i < total) {
            const int g = static_cast<int>(i / k), j = static_cast<int>(i % k);
            if (j < counts[g * counts_stride + q]) {
                const float sc = scores[g * scores_stride + static_cast<size_t>(q) * k + j];
                uint32_t low;
                if constexpr (kPosKey) {
                    const uint32_t it = static_cast<uint32_t>(items[g * items_stride + static_cast<size_t>(q) * k + j]);
                    low = ORDER == 2 ? it : ~it;
                } else if constexpr (kLowFirst) {
                    low = ~static_cast<uint32_t>(g * k + j);
                } else {
                    low = static_cast<uint32_t>(g * k + (k - 1 - j));
                }
                key = make_key(sc, low);
                want = key >= s_admit;
            }
        }
        need |= list_push_warp(l, key, want, cap - kSelectThreads);
    }
    __syncthreads();
    list_compact<kSelectThreads>(l, cap, k, 0);
    const int n = s_cnt;
    for (int j = tid; j < k; j += kSelectThreads) {
        int64_t item = -1;
        float sc = 0.0f;
        if (j < n) {
            const uint32_t low = key_pos(keys[j]);
            if constexpr (kPosKey) {
                item = static_cast<int64_t>(ORDER == 2 ? low : ~low);
            } else if constexpr (kLowFirst) {
                const uint32_t t = ~low;
                const int g = t / k, jj = static_cast<int>(t % k);
                item = items[g * items_stride + static_cast<size_t>(q) * k + jj];
            } else {
                const int g = low / k, jj = k - 1 - static_cast<int>(low % k);
                item = items[g * items_stride + static_cast<size_t>(q) * k + jj];
            }
            sc = key_score(keys[j]);
        }
        out_items[static_cast<size_t>(q) * k + j] = item;
        out_scores[static_cast<size_t>(q) * k + j] = sc;
    }
    if (tid == 0) out_counts[q] = n;
    if (sync.arrive) {
        // last CTA done: nobody on this rank reads the slots of `seq` any more -> acknowledge to every peer
        // (their next publish into this slot waits for it) and add up the "still to be corrected" tails
        __shared__ int s_last_cta;
        __threadfence();
        __syncthreads();
        if (tid == 0) {
            const uint32_t t = atomicAdd(sync.ticket, 1u);
            s_last_cta = t == gridDim.x - 1;
            if (s_last_cta) *sync.ticket = 0;
        }
        __syncthreads();
        if (s_last_cta) {
            __threadfence();
            if (tid < sync.world && tid != sync.me) st_release_sys(sync.ack[tid], sync.seq);
            if (tid == 0) {
                uint32_t sum = 0, status = 0;
                for (int r = 0; r < sync.world; ++r) {
                    const volatile uint32_t* tail =
                        reinterpret_cast<const volatile uint32_t*>(sync.tails + static_cast<size_t>(r) * sync.slot_bytes);
                    sum += tail[0];
                    status += tail[1];
                }
                *sync.flagged_host = sum;
                *sync.status_host = TAV_PEER_FILTER_MUTANT == 2 ? 0u : status;
            }
        }
    }
}

template <int ORDER>
static cudaError_t launch_merge_t(int n_lists, int n_queries, int k, const int64_t* items, const float* scores,
                                  const int32_t* counts, int64_t items_stride, int64_t scores_stride,
                                  int64_t counts_stride, int64_t* out_items, float* out_scores, int32_t* out_counts,
                                  cudaStream_t s, const MergeSync& sync) {
    const size_t smem = static_cast<size_t>(select_cap(k)) * sizeof(uint64_t);
    static int granted[16] = {};
    cudaError_t e = ensure_dynamic_smem(merge_kernel<ORDER>, smem, granted);
    if (e != cudaSuccess) return e;
    merge_kernel<ORDER><<<n_queries, kSelectThreads, smem, s>>>(n_lists, n_queries, k, items, scores, counts,
                                                                items_stride, scores_stride, counts_stride, out_items,
                                                                out_scores, out_counts, sync);
    return cudaGetLastError();
}

cudaError_t launch_merge_ordered(int n_lists, int n_queries, int k, const int64_t* items, const float* scores,
                                 const int32_t* counts, int64_t items_stride, int64_t scores_stride,
                                 int64_t counts_stride, int order, int64_t* out_items, float* out_scores,
                                 int32_t* out_counts, cudaStream_t s, const MergeSync* sync) {
    if (items_stride == 0) items_stride = static_cast<int64_t>(n_queries) * k;
    if (scores_stride == 0) scores_stride = static_cast<int64_t>(n_queries) * k;
    if (counts_stride == 0) counts_stride = n_queries;
#if TAV_SHARDED_FILTER_MUTANT == 1
    order = 0;
#endif
    const MergeSync none{};
    switch (order) {
        case 0: return launch_merge_t<0>(n_lists, n_queries, k, items, scores, counts, items_stride, scores_stride,
                                         counts_stride, out_items, out_scores, out_counts, s, sync ? *sync : none);
        case 1: return launch_merge_t<1>(n_lists, n_queries, k, items, scores, counts, items_stride, scores_stride,
                                         counts_stride, out_items, out_scores, out_counts, s, sync ? *sync : none);
        case 2: return launch_merge_t<2>(n_lists, n_queries, k, items, scores, counts, items_stride, scores_stride,
                                         counts_stride, out_items, out_scores, out_counts, s, sync ? *sync : none);
        case 3: return launch_merge_t<3>(n_lists, n_queries, k, items, scores, counts, items_stride, scores_stride,
                                         counts_stride, out_items, out_scores, out_counts, s, sync ? *sync : none);
    }
    return cudaErrorInvalidValue;
}

// tav_merge_topk's merge is order 0 of the ordered merge: one launch path, so that merge_kernel<0> has one record
// of the shared memory it was granted (two records of one kernel's attribute could lower it under the other's feet)
cudaError_t launch_merge(int n_lists, int n_queries, int k, const int64_t* items,
                         const float* scores, const int32_t* counts, int64_t items_stride,
                         int64_t scores_stride, int64_t counts_stride, int64_t* out_items,
                         float* out_scores, int32_t* out_counts, cudaStream_t s) {
    if (items_stride == 0) items_stride = static_cast<int64_t>(n_queries) * k;
    if (scores_stride == 0) scores_stride = static_cast<int64_t>(n_queries) * k;
    if (counts_stride == 0) counts_stride = n_queries;
    return launch_merge_t<0>(n_lists, n_queries, k, items, scores, counts, items_stride, scores_stride, counts_stride,
                             out_items, out_scores, out_counts, s, MergeSync{});
}

// ---- items[i] = table[items[i]] (subset positions -> global positions -> the caller's ordinals) --------
__global__ void __launch_bounds__(256)
map_items_kernel(int64_t n, const int64_t* __restrict__ table, int64_t table_len, int64_t* __restrict__ items) {
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        const int64_t v = items[i];
        if (v >= 0 && v < table_len) items[i] = table[v];
    }
}

cudaError_t launch_map_items(int64_t n, const int64_t* table, int64_t table_len, int64_t* items, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    const int64_t blocks = std::min<int64_t>((n + 255) / 256, 132 * 8);
    map_items_kernel<<<static_cast<unsigned>(blocks), 256, 0, s>>>(n, table, table_len, items);
    return cudaGetLastError();
}

// ---- chunk -> message fold of a hit list (storage/memory/messageindex.py:185-207) --------------
// The reference folds AFTER the top-k over chunks: walking the hits in score order, the first hit of
// a message carries its best score; later hits of the same message are dropped.  One CTA per query,
// in place: items become group (message) ordinals, order preserved, tail padded with -1 / 0.
__global__ void __launch_bounds__(256)
fold_groups_kernel(int k, const int32_t* row_to_group, int64_t n_rows, int64_t item_offset, int64_t* items_all,
                   float* scores_all, int32_t* counts) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    int32_t* grp = reinterpret_cast<int32_t*>(smem_raw);         // [k]
    float* sc = reinterpret_cast<float*>(grp + k);               // [k]
    __shared__ int s_base, s_warp[8];
    const int q = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int64_t* items = items_all + static_cast<size_t>(q) * k;
    float* scores = scores_all + static_cast<size_t>(q) * k;
    const int n = min(counts[q], k);
    for (int j = tid; j < n; j += 256) {
        const int64_t row = items[j] - item_offset;
        grp[j] = (row >= 0 && row < n_rows) ? row_to_group[row] : -1 - j;  // unmapped rows stay distinct
        sc[j] = scores[j];
    }
    if (tid == 0) s_base = 0;
    __syncthreads();
    for (int j0 = 0; j0 < n; j0 += 256) {
        const int j = j0 + tid;
        bool keep = j < n;
        if (keep) {
            const int g = grp[j];
            for (int i = 0; i < j; ++i)
                if (grp[i] == g) {
                    keep = false;
                    break;
                }
        }
        const unsigned m = __ballot_sync(0xFFFFFFFFu, keep);
        if (lane == 0) s_warp[warp] = __popc(m);
        __syncthreads();
        int before = s_base;
        for (int w = 0; w < warp; ++w) before += s_warp[w];
        if (keep) {
            const int dst = before + __popc(m & ((1u << lane) - 1u));
            items[dst] = grp[j] < 0 ? -1 : static_cast<int64_t>(grp[j]);  // dst <= j; inputs were copied to smem
            scores[dst] = sc[j];
        }
        __syncthreads();
        if (tid == 0) {
            int total = 0;
            for (int w = 0; w < 8; ++w) total += s_warp[w];
            s_base += total;
        }
        __syncthreads();
    }
    const int kept = s_base;
    for (int j = kept + tid; j < k; j += 256) {
        items[j] = -1;
        scores[j] = 0.0f;
    }
    if (tid == 0) counts[q] = kept;
}

cudaError_t launch_fold_groups(int n_queries, int k, const int32_t* row_to_group, int64_t n_rows,
                               int64_t item_offset, int64_t* items, float* scores, int32_t* counts,
                               cudaStream_t s) {
    if (n_queries == 0) return cudaSuccess;
    const size_t smem = static_cast<size_t>(k) * 8;
    static int granted[16] = {};
    cudaError_t e = ensure_dynamic_smem(fold_groups_kernel, smem, granted);
    if (e != cudaSuccess) return e;
    fold_groups_kernel<<<n_queries, 256, smem, s>>>(k, row_to_group, n_rows, item_offset, items, scores, counts);
    return cudaGetLastError();
}

// ---- convert-on-append (fused optional L2 normalisation) ---------------------------------
template <typename S, typename D>
__device__ __forceinline__ D convert_elem(S v);
template <> __device__ __forceinline__ float convert_elem<float, float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 convert_elem<float, __nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ __half convert_elem<float, __half>(float v) { return __float2half_rn(v); }

template <typename S, typename D>
__global__ void __launch_bounds__(256) convert_rows_kernel(const S* src, D* dst, int64_t n, int dim,
                                                          int normalize) {
    // one warp per row
    const int lane = threadIdx.x & 31;
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t n_warps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    for (int64_t row = warp; row < n; row += n_warps) {
        const S* s = src + row * dim;
        D* d = dst + row * dim;
        float inv = 1.0f;
        int shift = 0;
        if (normalize) {
            // Scale by 2^-shift, the power of two of the largest magnitude, so that the sum of squares of
            // the scaled row lies in [1/4, dim] whatever the row's scale: without it rows below ~1e-19
            // underflow to a zero or subnormal sum and rows above ~1e19 overflow it.  The scaling is exact,
            // so rows whose squares stay in the normal range get the same bits as unscaled arithmetic.
            // fmaxf skips NaN; an infinite maximum leaves the row unscaled (its quotients are then NaN or 0).
            float amax = 0.0f;
            for (int c = lane; c < dim; c += 32) amax = fmaxf(amax, fabsf(to_float(s[c])));
#pragma unroll
            for (int off = 16; off >= 1; off >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xFFFFFFFFu, amax, off));
            if (amax > 0.0f && isfinite(amax)) frexpf(amax, &shift);
            float ss = 0.0f;
            for (int c = lane; c < dim; c += 32) {
                const float v = ldexpf(to_float(s[c]), -shift);
                ss = fmaf(v, v, ss);
            }
#pragma unroll
            for (int off = 16; off >= 1; off >>= 1) ss += __shfl_xor_sync(0xFFFFFFFFu, ss, off);
            const float nrm = sqrtf(ss);
            inv = nrm > 0.0f ? nrm : 1.0f;  // the divisor; zero rows stay zero (model_adapters.py:182)
            if (!(nrm > 0.0f)) shift = 0;   // zero rows and rows with a NaN are stored as they are
        }
        for (int c = lane; c < dim; c += 32) {
            float v = to_float(s[c]);
            if (normalize) v = ldexpf(v, -shift) / inv;
            d[c] = convert_elem<float, D>(v);
        }
    }
}

template <typename S>
static cudaError_t launch_convert_s(const S* src, void* dst, int dst_dtype, int64_t n, int dim,
                                    int normalize, cudaStream_t s) {
    int64_t blocks = (n + 7) / 8;
    if (blocks > 132 * 16) blocks = 132 * 16;
    if (blocks < 1) blocks = 1;
    const int g = static_cast<int>(blocks);
    switch (dst_dtype) {
        case TAV_F32: convert_rows_kernel<S, float><<<g, 256, 0, s>>>(src, static_cast<float*>(dst), n, dim, normalize); break;
        case TAV_BF16: convert_rows_kernel<S, __nv_bfloat16><<<g, 256, 0, s>>>(src, static_cast<__nv_bfloat16*>(dst), n, dim, normalize); break;
        case TAV_F16: convert_rows_kernel<S, __half><<<g, 256, 0, s>>>(src, static_cast<__half*>(dst), n, dim, normalize); break;
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

cudaError_t launch_convert(const void* src, int src_dtype, void* dst, int dst_dtype, int64_t n,
                           int dim, int normalize, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    switch (src_dtype) {
        case TAV_F32: return launch_convert_s(static_cast<const float*>(src), dst, dst_dtype, n, dim, normalize, s);
        case TAV_BF16: return launch_convert_s(static_cast<const __nv_bfloat16*>(src), dst, dst_dtype, n, dim, normalize, s);
        case TAV_F16: return launch_convert_s(static_cast<const __half*>(src), dst, dst_dtype, n, dim, normalize, s);
    }
    return cudaErrorInvalidValue;
}

}  // namespace tav
