// tav_mma.cu — the tensor-core path of libtavec: batched query x corpus similarity as a dense
// bf16/fp16 contraction on Hopper warpgroup MMAs (wgmma, fp32 accumulators in registers) fed by
// TMA tiles from HBM, with the score threshold and top-k candidate selection fused into the
// epilogue that reads the accumulators.
//
// Reference semantics (aitools/vectorbase.py:163-190, per query): x = dot(row, q) in float32;
// score = clip((x+1)/2, 0, 1); keep score >= min_score; k best by score.  Products of bf16/fp16
// values are exact in float32, so on storage-rounded inputs only the summation order differs
// from the reference's sgemv.
//
// Shape of one CTA (persistent, one per SM, 288 threads):
//   warps 0-7  two consumer warpgroups.  Warpgroup g owns queries [64g, 64g+64) of the unit's
//              128-query chunk: per 64-wide K slice it issues four wgmma m64nNk16 (N = 256 corpus
//              rows, or 128 in the split form) on the query slice and the corpus slice in shared
//              memory, keeping one group in flight while it releases the previous slot.  After the
//              last K slice of a tile its accumulators are screened in registers: a thread holds two
//              queries (rows r and r+8 of its warp's 16) and, of every 8 corpus rows, two neighbours.
//              Per 32 rows of a query: the maximum of its 8 dots against the query's admission
//              threshold; only a group that holds an admitted row runs its 8 predicated compare-and-
//              append steps, (dot, row) keys going to the thread's PRIVATE segment of the query's
//              candidate buffer (register counter, no atomics; admit_group).
//   warp 8     TMA producer: per (corpus tile, query chunk, 64-wide K slice) loads the query slice
//              [128 x 64] and the corpus slice [N x 64] into a smem ring (4 x 48 KB, or 3 x 64 KB in
//              the split form; 128-byte swizzle), completing on an mbarrier.
//
// Work items are (corpus tile, query chunk of 128) pairs, so ANY number of queries is served by ONE
// launch per pass: a unit serves one chunk and every n-th tile, the chunks of a tile are visited by
// neighbouring units at the same time and share the tile through L2, i.e. HBM is read once per
// search, not once per 128 queries.
//
// Admission thresholds.  A first launch of the same kernel in SAMPLE mode scores a strided sample
// of corpus tiles; its epilogue is branch-free: it only keeps the maxima of blocks of the dots of a
// query (128 rows for large corpora; 32 or 8 rows when the target is a larger share of the corpus)
// and stores them.  The unit that finishes a query chunk's last sample tile then derives, per query,
// the 8th largest block maximum — at least 8 distinct rows reach it — lowers it to the bottom of its
// float32 score class, never below the caller's min_score, and publishes it as the admission
// threshold (expected to admit `target` rows of the corpus, see make_plan).  The MAIN launch then
// streams the whole corpus once; a finalize kernel maps the admitted dots to scores and selects the
// top k with the library's total order.
// Exactness: every row not admitted scores strictly below every admitted row, so if at least k
// rows were admitted (or the threshold is the caller's min_score itself) the result is the exact
// top-k.  For k <= 8 that always holds (the 8 block maxima are themselves admitted); otherwise a
// query for which it does not (pathological score distributions; probability ~6e-8 on well-mixed
// data) or whose buffer overflowed is flagged and redone by the exact row-scan path.
//
// Optional row mask (predicate / post-filter pushdown, reference: aitools/vectorbase.py:191-201,
// storage/sqlite/messageindex.py:296-326): one bit per corpus row; masked-out rows are dropped
// in the epilogue (and ignored by the sampler, so the threshold adapts to the mask's density).
// Per-query masks (kSampleQ / kMainQ): the same, with each query's own mask; a query whose mask allows at most
// pop_exact rows is admitted at the min_score floor, so a sparse mask does not starve it into the exact redo.
//
// Algorithmic bytes per search: N*D*2 (corpus, read once) + queries + hits.

#include <float.h>
#include <math.h>
#include <stdlib.h>

#include <algorithm>
#include <mutex>

#include "tav_common.cuh"
#include "tav_internal.h"
#include "tav_ptx.cuh"

namespace tav {

namespace {

constexpr int kBM = 128;   // queries per chunk (two warpgroups of 64)
constexpr int kBK = 64;    // 16-bit elements per K slice = one 128-byte swizzle row
constexpr int kABytes = kBM * kBK * 2;              // 16 KB
constexpr int kConsumerWarps = 8;                   // two warpgroups
constexpr int kMmaThreads = 32 * kConsumerWarps + 32;  // + the TMA producer warp
constexpr int kSampleTop = 8;                       // the threshold is the 8th largest block maximum
constexpr int kMaxChunks = 512;                     // query chunks per launch (tav_search slabs larger batches)
constexpr int kFinalizeFast = 8192;                 // finalize sorts up to this many candidates in one go
constexpr int kSegPerUnit = 4;                      // candidate segments per query per unit (the 4 threads of a quad)
constexpr int kMaxSegments = kSegPerUnit * 160;     // candidate segments per query
constexpr int kTileRows = 256;                      // corpus rows per tile (128 in the split form)
constexpr int kTileRowsSplit = 128;
constexpr size_t kTileSmem = 192 * 1024;            // the stage ring: 4 x (16 + 32) KB, or 3 x 2 x (16 + 16) KB
constexpr size_t kScratchBytes = 2 * kBM * kSampleTop * sizeof(float);  // the sampler tail's exchange of partial top-8 lists
constexpr size_t kSmemBytes = 1024 + kTileSmem + 256 + kScratchBytes;

// kSampleQ / kMainQ: kSample / kMain with per-query masks (KernelArgs::qmask)
enum Mode { kSample = 0, kMain = 1, kDump = 2, kSampleQ = 3, kMainQ = 4 };

struct KernelArgs {
    int64_t n_rows;
    int n_tiles_work;      // tiles visited by this launch
    int64_t tile_mul;      // visited tile t -> corpus tile (t * tile_mul) / tile_div
    int64_t tile_div;
    int kb_count;          // ceil(dim / 64)
    int nq;                // valid queries (all chunks)
    int nqc;               // query chunks of 128 queries
    int nq_pad;            // nqc * 128
    int n_seg;             // MAIN: candidate segments per query = 4 * (units per chunk)
    float* thr;            // [nq_pad] admission threshold (raw dot) per query: SAMPLE writes, MAIN reads
    float* floor_x;        // SAMPLE: [nq_pad] the caller's min_score as a dot floor
    float* sample_max;     // SAMPLE: [n_tiles_work * blocks per tile, nq_pad] block maxima
    int sample_gph;        // SAMPLE: blocks per 128 rows: 1 (128 rows each), 4 (32 rows) or 16 (8 rows)
    int sample_use;        // SAMPLE: blocks the threshold is derived from ...
    int sample_stride;     //         ... every sample_stride-th of the stored ones
    uint32_t* sample_done; // SAMPLE: [nqc] finished-unit counters (self-resetting)
    int32_t* retry;        // SAMPLE: [nq] per-query "redo exactly" flags, cleared here
    float floor_score;     // SAMPLE: (float)min_score
    uint64_t* cand;        // MAIN: [nq_pad, n_seg, cap_seg]  (dot bits << 32 | row)
    uint32_t* cand_count;  // MAIN: [nq_pad, n_seg] rows each epilogue thread admitted (may exceed cap_seg: overflow)
    uint32_t cap_seg;
    const uint32_t* row_mask;  // optional: bit r set = row r may be returned
    float* dump;           // DUMP: [nq, n_rows] raw dots
    QueryMasks qmask;      // kSampleQ / kMainQ: per-query masks (bits padded to whole tiles)
    uint32_t pop_exact;    // kSampleQ: a query whose mask allows at most this many rows is admitted at the floor
};

__device__ __forceinline__ void insert_top(float (&top)[kSampleTop], float x) {
    // top[] sorted descending; branch-free insertion (x below top[last] falls out)
#pragma unroll
    for (int i = 0; i < kSampleTop; ++i) {
        const float hi = fmaxf(top[i], x);
        x = fminf(top[i], x);
        top[i] = hi;
    }
}

// accumulator d[4j + 2h + e] of a thread: query row h (0: r, 1: r + 8), corpus column 8j + 2 (lane % 4) + e
__device__ __forceinline__ int acc_index(int j, int h, int e) { return 4 * j + 2 * h + e; }

// MAIN epilogue of one group of 32 corpus rows for ONE query of this thread (h): its 8 dots of those rows
// (columns 32g + 8jj + 2 (lane % 4) + e) against the query's admission threshold.  The maximum of the 8 is
// tested first; only a group that holds an admitted row runs the 8 predicated compare-and-store steps,
// appending (dot, row) keys to the thread's PRIVATE candidate segment (one writer, a register counter).
// `amask`: bit i set = row rbase + i exists and passes the row mask (warp-uniform).
template <int NACC>
__device__ __forceinline__ void admit_group(const float (&d)[NACC], int g, int h, int t4, float tau, uint32_t rbase,
                                            uint32_t amask, uint64_t* my_cand, uint32_t& n_admitted,
                                            uint32_t cap_seg) {
    float m = -INFINITY;
#pragma unroll
    for (int jj = 0; jj < 4; ++jj)
        m = fmaxf(m, fmaxf(d[acc_index(4 * g + jj, h, 0)], d[acc_index(4 * g + jj, h, 1)]));
    if (m >= tau) {
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const float x = d[acc_index(4 * g + jj, h, e)];
                const int i = 8 * jj + 2 * t4 + e;
                if (x >= tau && ((amask >> i) & 1u)) {
                    if (n_admitted < cap_seg)
#if TAV_SCALE_MUTANT == 1
                        my_cand[n_admitted] = (static_cast<uint64_t>(__float_as_uint(x)) << 32) | ((rbase + i) & 0xFFFFFFu);
#else
                        my_cand[n_admitted] = (static_cast<uint64_t>(__float_as_uint(x)) << 32) | (rbase + i);
#endif
                    ++n_admitted;
                }
            }
        }
    }
}

// maximum over the 4 threads of a quad (which together hold every column of a query's 8-row group)
__device__ __forceinline__ float quad_max(float x) {
    x = fmaxf(x, __shfl_xor_sync(0xFFFFFFFFu, x, 1));
    return fmaxf(x, __shfl_xor_sync(0xFFFFFFFFu, x, 2));
}

// SAMPLE epilogue of one tile for one query of this thread (h): maxima of blocks of JPB * 8 rows, the
// masked-out rows ignored, stored to dst[block * nq_pad] by one thread of the quad.
template <int JPB, int NACC>
__device__ __forceinline__ void sample_blocks(const float (&d)[NACC], int h, int t4, const uint32_t* row_mask,
                                              int64_t row0, float* dst, int nq_pad) {
    constexpr int kJ = NACC / 4;  // 8-row groups in the tile
#pragma unroll
    for (int b = 0; b < kJ / JPB; ++b) {
        float m = -INFINITY;
#pragma unroll
        for (int jj = 0; jj < JPB; ++jj) {
            const int j = b * JPB + jj;
            const uint32_t bits = row_mask ? row_mask[(row0 >> 5) + (j >> 2)] : 0xFFFFFFFFu;
            const int i = 8 * (j & 3) + 2 * t4;
            m = fmaxf(m, ((bits >> i) & 1u) ? d[acc_index(j, h, 0)] : -INFINITY);
            m = fmaxf(m, ((bits >> (i + 1)) & 1u) ? d[acc_index(j, h, 1)] : -INFINITY);
        }
        m = quad_max(m);
        if (t4 == (b & 3)) dst[static_cast<size_t>(b) * nq_pad] = m;
    }
}

// Work distribution: unit u (a CTA) serves ONE query chunk, c = u % nqc, and every (n_units / nqc)-th
// tile of the launch, starting at u / nqc — so the nqc units that share a tile run side by side (the tile
// is fetched from HBM once and served to the others by L2) and an epilogue thread keeps the same queries
// for the whole launch (its candidate counters live in registers).
// Item i of unit `unit` -> (visited tile t, query chunk c); false when the unit has no such item.
__device__ __forceinline__ bool get_item(const KernelArgs& a, int unit, int n_units, int i, int& t, int& c) {
    const int upc = n_units / a.nqc;  // units per chunk (the launcher makes n_units a multiple of nqc)
    c = unit % a.nqc;
    t = unit / a.nqc + i * upc;
    return t < a.n_tiles_work;
}

// ---- float <-> order-preserving uint32 ------------------------------------------------------
__device__ __forceinline__ uint32_t float_to_ord(float f) {
    const uint32_t b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float ord_to_float(uint32_t o) {
    return __uint_as_float((o & 0x80000000u) ? (o ^ 0x80000000u) : ~o);
}
// smallest dot x whose score clip((x+1)/2,0,1) is >= s: -inf when every x qualifies, +inf when
// none does (s > 1, or NaN: `score >= NaN` is false for every row, as in the reference)
__device__ float dot_floor_for_score(float s) {
    if (s != s) return INFINITY;
    if (!(s > 0.0f)) return -INFINITY;
    if (s > 1.0f) return INFINITY;
    uint32_t lo = float_to_ord(-FLT_MAX), hi = float_to_ord(FLT_MAX);
    while (lo < hi) {
        const uint32_t mid = lo + ((hi - lo) >> 1);
        if (score_from_dot(ord_to_float(mid)) >= s) hi = mid;
        else lo = mid + 1;
    }
    return ord_to_float(lo);
}

template <int N, bool BF16>
__device__ __forceinline__ void wgmma_step(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
    if constexpr (N == 256) {
        if constexpr (BF16) ptx::wgmma_m64n256_bf16(d, da, db, scale_d);
        else ptx::wgmma_m64n256_f16(d, da, db, scale_d);
    } else {
        static_assert(N == 128 && !BF16, "the split form is fp16, N = 128");
        ptx::wgmma_m64n128_f16(d, da, db, scale_d);
    }
}

// BF16: operand format (bf16 or fp16).
// SPLIT: float32 data carried as two fp16 planes, x = hi + lo / 2048 (22 significant bits; products of
//        fp16 values are exact in the fp32 accumulator).  Three MMAs per K step: hi.hi' into the MAIN
//        accumulator, hi.lo' + lo.hi' into the CROSS accumulator; the epilogue combines main + cross /
//        2048 (the lo.lo' term, <= 2^-22 relative, is dropped).  Two accumulators of 64 x 128 take the
//        registers one of 64 x 256 does, so tiles are 128 corpus rows in this form.
template <int MODE, bool BF16, bool SPLIT>
__global__ void __launch_bounds__(kMmaThreads, 1)
mma_topk_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_c,
                const __grid_constant__ CUtensorMap map_q_lo, const __grid_constant__ CUtensorMap map_c_lo,
                const KernelArgs a) {
    constexpr bool kQM = MODE == kSampleQ || MODE == kMainQ;   // per-query masks
    constexpr bool kIsSample = MODE == kSample || MODE == kSampleQ;
    constexpr bool kIsMain = MODE == kMain || MODE == kMainQ;
    constexpr int kTileN = SPLIT ? kTileRowsSplit : kTileRows;  // corpus rows per tile
    constexpr int kNacc = kTileN / 2;                          // accumulator registers per thread
    constexpr int kBBytes = kTileN * kBK * 2;
    constexpr int kPlanes = SPLIT ? 2 : 1;
    constexpr int kStageBytes = kPlanes * (kABytes + kBBytes);  // [A | B | A_lo | B_lo]
    constexpr int kNumStages = static_cast<int>(kTileSmem / kStageBytes);
    static_assert(kNumStages * kStageBytes == static_cast<int>(kTileSmem), "stage ring");
    extern __shared__ uint8_t smem_dyn[];
    // SWIZZLE_128B tiles need 1024-byte alignment
    uint8_t* tiles = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(tiles + kTileSmem);
    uint64_t* full = bars;                    // [stages] TMA -> MMA
    uint64_t* empty = bars + kNumStages;      // [stages] MMA -> TMA (one arrive per consumer warp)
    float* scratch = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(bars) + 256);  // sampler tail
    __shared__ int s_last;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int unit = blockIdx.x, n_units = gridDim.x;

    if (threadIdx.x == 0) {
        for (int s = 0; s < kNumStages; ++s) {
            ptx::mbar_init(&full[s], 1);  // the producer arrives once with the stage's bytes
            ptx::mbar_init(&empty[s], kConsumerWarps);
        }
        ptx::fence_mbar_init();
    }
    if (warp == kConsumerWarps && lane == 0) {
        ptx::prefetch_tensormap(&map_q);
        ptx::prefetch_tensormap(&map_c);
        if (SPLIT) {
            ptx::prefetch_tensormap(&map_q_lo);
            ptx::prefetch_tensormap(&map_c_lo);
        }
    }
    // per-query masks: the mask row of each query of this unit's chunk, in the sampler tail's scratch (unused
    // until the tail), so that the epilogue keeps no register for it (padding queries: nullptr, nothing read)
    const uint32_t** s_qrow = reinterpret_cast<const uint32_t**>(scratch);
    if constexpr (kQM) {
        if (threadIdx.x < kBM) {
            const int q = (unit % a.nqc) * kBM + threadIdx.x;
            s_qrow[threadIdx.x] =
                q < a.nq ? a.qmask.bits + static_cast<int64_t>(a.qmask.map ? a.qmask.map[q] : q) * a.qmask.stride : nullptr;
        }
    }
    __syncthreads();

    if (warp == kConsumerWarps) {
        // ================= TMA producer =================
        if (lane == 0) {
            uint32_t stage = 0, phase = 0;
            int t, c;
            for (int i = 0; get_item(a, unit, n_units, i, t, c); ++i) {
                const int64_t tile = (static_cast<int64_t>(t) * a.tile_mul) / a.tile_div;
                const int32_t row0 = static_cast<int32_t>(tile * kTileN);
                const int32_t qrow = c * kBM;
                for (int kb = 0; kb < a.kb_count; ++kb) {
                    ptx::mbar_wait(&empty[stage], phase ^ 1);
                    uint8_t* sa = tiles + static_cast<size_t>(stage) * kStageBytes;
                    ptx::mbar_expect_tx(&full[stage], kStageBytes);
                    ptx::tma_load_2d(sa, &map_q, &full[stage], kb * kBK, qrow, ptx::kEvictLast);
                    ptx::tma_load_2d(sa + kABytes, &map_c, &full[stage], kb * kBK, row0, ptx::kEvictFirst);
                    if (SPLIT) {
                        uint8_t* sl = sa + kABytes + kBBytes;
                        ptx::tma_load_2d(sl, &map_q_lo, &full[stage], kb * kBK, qrow, ptx::kEvictLast);
                        ptx::tma_load_2d(sl + kABytes, &map_c_lo, &full[stage], kb * kBK, row0, ptx::kEvictFirst);
                    }
                    if (++stage == kNumStages) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
            }
        }
    } else {
        // ================= consumer warpgroups: MMAs, then the epilogue on the accumulators =====
        const int wg = warp >> 2;                    // which 64 queries of the chunk
        const int t4 = lane & 3;                     // column pair inside every 8-row group
        const int c_unit = unit % a.nqc;
        const int q_local = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // + 8 for the second query (h = 1)
        const int my_q[2] = {c_unit * kBM + q_local, c_unit * kBM + q_local + 8};
        // MAIN: this thread's private candidate segments (no atomics: one writer per segment)
        const int seg = (unit / a.nqc) * kSegPerUnit + t4;
        uint64_t* my_cand[2];
        uint32_t n_admitted[2] = {0u, 0u};
        float tau[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            my_cand[h] = a.cand + (static_cast<size_t>(my_q[h]) * a.n_seg + seg) * a.cap_seg;
            tau[h] = (kIsMain && my_q[h] < a.nq) ? a.thr[my_q[h]] : INFINITY;
        }
        // A: this warpgroup's 64 query rows (8 swizzle groups of 1024 B in); B: the corpus slice
        const uint32_t a_off = static_cast<uint32_t>(wg) * 64 * 128;
        float acc[kNacc];
        float accx[SPLIT ? kNacc : 1];
#pragma unroll
        for (int i = 0; i < kNacc; ++i) acc[i] = 0.0f;
#pragma unroll
        for (int i = 0; i < (SPLIT ? kNacc : 1); ++i) accx[i] = 0.0f;
        uint32_t stage = 0, phase = 0;
        int t, c;
        for (int i = 0; get_item(a, unit, n_units, i, t, c); ++i) {
            const int64_t tile = (static_cast<int64_t>(t) * a.tile_mul) / a.tile_div;
            const int64_t row0 = tile * kTileN;
            uint32_t prev = 0;
            for (int kb = 0; kb < a.kb_count; ++kb) {
                ptx::mbar_wait(&full[stage], phase);
                const uint32_t sa = ptx::smem_u32(tiles + static_cast<size_t>(stage) * kStageBytes);
                const uint64_t da = ptx::make_kmajor_sw128_desc(sa + a_off);
                const uint64_t db = ptx::make_kmajor_sw128_desc(sa + kABytes);
                ptx::wgmma_fence();
#pragma unroll
                for (int k = 0; k < kBK / 16; ++k) {
                    const uint32_t accumulate = (kb | k) != 0 ? 1u : 0u;
                    wgmma_step<kTileN, BF16>(acc, da + 2 * k, db + 2 * k, accumulate);
                    if constexpr (SPLIT) {
                        const uint64_t da_lo = ptx::make_kmajor_sw128_desc(sa + kABytes + kBBytes + a_off) + 2 * k;
                        const uint64_t db_lo = ptx::make_kmajor_sw128_desc(sa + 2 * kABytes + kBBytes) + 2 * k;
                        wgmma_step<kTileN, false>(accx, da + 2 * k, db_lo, accumulate);  // hi . lo'
                        wgmma_step<kTileN, false>(accx, da_lo, db + 2 * k, 1u);          // lo . hi'
                    }
                }
                ptx::wgmma_commit();
                // the previous slice's MMAs have retired: its slot may be refilled
                if (kb > 0) {
                    ptx::wgmma_wait<1>();
                    if (lane == 0) ptx::mbar_arrive(&empty[prev]);
                }
                prev = stage;
                if (++stage == static_cast<uint32_t>(kNumStages)) {
                    stage = 0;
                    phase ^= 1;
                }
            }
            ptx::wgmma_wait<0>();
            if (lane == 0) ptx::mbar_arrive(&empty[prev]);
            if constexpr (SPLIT) {
                // x = main + cross / 2048
#pragma unroll
                for (int r = 0; r < kNacc; ++r) acc[r] = fmaf(accx[r], 1.0f / 2048.0f, acc[r]);
            }

            // columns of the tile that are real corpus rows (uniform)
            const int ncols = static_cast<int>(max(static_cast<int64_t>(0),
                                                   min(static_cast<int64_t>(kTileN), a.n_rows - row0)));
            if (MODE == kDump) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    if (my_q[h] >= a.nq) continue;
                    float* out = a.dump + static_cast<size_t>(my_q[h]) * a.n_rows + row0;
#pragma unroll
                    for (int j = 0; j < kNacc / 4; ++j)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int col = 8 * j + 2 * t4 + e;
                            if (col < ncols) out[col] = acc[acc_index(j, h, e)];
                        }
                }
            } else if (kIsSample) {
                // branch-free: sample tiles are full tiles, every column is a real row
                const int bpt = (kTileN / 128) * a.sample_gph;  // blocks per tile
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float* dst = a.sample_max + static_cast<size_t>(t) * bpt * a.nq_pad + my_q[h];
                    const uint32_t* mask = a.row_mask;
                    if constexpr (kQM)  // each query's own rows: its threshold adapts to its mask
                        mask = s_qrow[q_local + 8 * h];
                    if (a.sample_gph == 16) sample_blocks<1>(acc, h, t4, mask, row0, dst, a.nq_pad);
                    else if (a.sample_gph == 4) sample_blocks<4>(acc, h, t4, mask, row0, dst, a.nq_pad);
                    else sample_blocks<16>(acc, h, t4, mask, row0, dst, a.nq_pad);
                }
            } else {
                // MAIN: group-wise screen and private-segment append (admit_group)
#pragma unroll
                for (int g = 0; g < kTileN / 32; ++g) {
                    const int nvalid = min(32, ncols - 32 * g);
                    if (nvalid <= 0) break;
                    const uint32_t rbase = static_cast<uint32_t>(row0 + 32 * g);
                    uint32_t amask = nvalid >= 32 ? 0xFFFFFFFFu : ((1u << nvalid) - 1u);
                    if (!kQM && a.row_mask) amask &= a.row_mask[rbase >> 5];
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        uint32_t am = amask;
                        if constexpr (kQM) {  // the query's own mask word of these 32 rows
                            const uint32_t* qr = s_qrow[q_local + 8 * (TAV_QUERY_MASK_MUTANT == 1 ? h ^ 1 : h)];
                            am = qr ? am & qr[rbase >> 5] : 0u;
                        }
                        admit_group(acc, g, h, t4, tau[h], rbase, am, my_cand[h], n_admitted[h], a.cap_seg);
                    }
                }
            }
        }
        if (kIsSample) __threadfence();  // block maxima visible device-wide before the unit signs off
        if (kIsMain && unit / a.nqc < n_units / a.nqc) {
#pragma unroll
            for (int h = 0; h < 2; ++h) a.cand_count[static_cast<size_t>(my_q[h]) * a.n_seg + seg] = n_admitted[h];
        }
    }

    if (kIsSample) {
        // ---- sampler tail: the last unit of a query chunk turns block maxima into thresholds ----
        __syncthreads();
        const int upc = n_units / a.nqc;
        const int c = unit % a.nqc;
        const bool has_items = unit / a.nqc < min(upc, a.n_tiles_work);
        const int n_signing = min(upc, a.n_tiles_work);  // units of this chunk that visited a tile
        if (threadIdx.x == 0) {
            int last = 0;
            if (has_items) {
                __threadfence();
                const uint32_t done = atomicAdd(&a.sample_done[c], 1u);
                last = done == static_cast<uint32_t>(n_signing - 1);
                if (last) a.sample_done[c] = 0;  // ready for the next search
            }
            s_last = last;
        }
        __syncthreads();
        if (s_last && warp < kConsumerWarps) {
            __threadfence();
            const int te = threadIdx.x;  // 0..255
            const int ql = te & (kBM - 1), part = te >> 7;
            const int q = c * kBM + ql;
            const int n_blocks = a.sample_use;  // blocks j * sample_stride of the stored ones, j < sample_use
            float top[kSampleTop];
#pragma unroll
            for (int i = 0; i < kSampleTop; ++i) top[i] = -INFINITY;
            // 8 independent loads in flight per thread (a rolled loop pays one L2 latency per block)
            for (int b0 = part; b0 < n_blocks; b0 += 16) {
                float x[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    const int b = b0 + 2 * u;
                    x[u] = b < n_blocks ? __ldcg(&a.sample_max[static_cast<size_t>(b) * a.sample_stride * a.nq_pad + q])
                                        : -INFINITY;
                }
#pragma unroll
                for (int u = 0; u < 8; ++u) insert_top(top, x[u]);
            }
            if (part == 1) {
#pragma unroll
                for (int i = 0; i < kSampleTop; ++i) scratch[(i * kBM) + ql] = top[i];
            }
            asm volatile("bar.sync 1, 256;" ::: "memory");  // the consumer warps
            if (part == 0) {
#pragma unroll
                for (int i = 0; i < kSampleTop; ++i) insert_top(top, scratch[(i * kBM) + ql]);
                if (q < a.nq) {
                    const float floor_x = dot_floor_for_score(a.floor_score);
                    float thr = floor_x;
                    const float sampled = top[kSampleTop - 1];
                    if (sampled > -INFINITY) {
                        // bottom of the float32 score class of the sampled dot: rows below it score strictly less
                        thr = fmaxf(dot_floor_for_score(score_from_dot(sampled)), floor_x);
                    }
                    if constexpr (kQM) {
                        // a sparse mask: every allowed row fits the segments (or fewer than k are allowed), so the
                        // exact floor admits them all instead of a sampled threshold that could starve the query
                        if (a.qmask.pop && a.qmask.pop[a.qmask.map ? a.qmask.map[q] : q] <= a.pop_exact) thr = floor_x;
                    }
                    a.thr[q] = thr;
                    a.floor_x[q] = floor_x;
                    a.retry[q] = 0;
                }
            }
        }
    }
}

// ---- small kernels around the tensor-core passes ---------------------------------------------
__device__ __forceinline__ void store_rn(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }
__device__ __forceinline__ void store_rn(__half* p, float v) { *p = __float2half_rn(v); }

// per-query state of a search that runs WITHOUT a sample pass (small corpora): the admission
// threshold is the caller's min_score itself; counters and flags cleared
__device__ __forceinline__ void init_query_state(int q, int nq, float floor_score, float* thr, float* floor_out,
                                                 int32_t* retry) {
    if (q >= nq) return;
    const float floor_x = dot_floor_for_score(floor_score);
    thr[q] = floor_x;
    floor_out[q] = floor_x;
    retry[q] = 0;
}

// queries float32 [nq, dim] -> storage dtype [nq_pad, dim], rows >= nq zeroed; with `init_state`
// also the per-query search state (see init_query_state) — one launch instead of two
template <typename T>
__global__ void query_prep_kernel(const float* q, T* out, int nq, int nq_pad, int dim, int init_state,
                                  float floor_score, float* thr, float* floor_out, int32_t* retry) {
    const int64_t total = static_cast<int64_t>(nq_pad) * dim;
    const int64_t tid = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    for (int64_t i = tid; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int row = static_cast<int>(i / dim);
        const float v = row < nq ? q[i] : 0.0f;
        store_rn(out + i, v);
    }
    if (init_state && tid < nq) init_query_state(static_cast<int>(tid), nq, floor_score, thr, floor_out, retry);
}

// float32 x -> fp16 planes hi = fp16(x), lo = fp16((x - hi) * 2048): x ~= hi + lo / 2048 to 2^-22.
// Rows >= n_valid are zero-filled (query padding).  |x| must be below the fp16 range; a value
// that is not sets *overflow and the caller redoes the search with the exact row scan.
__global__ void split_rows_kernel(const float* src, __half* hi, __half* lo, int64_t n_valid, int64_t n_total,
                                  int dim, int* overflow, int* overflow_host, int init_state, float floor_score,
                                  float* thr, float* floor_out, int32_t* retry) {
    const int64_t total = n_total * dim;
    const int64_t tid = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    bool bad = false;
    for (int64_t i = tid; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const float x = (i / dim) < n_valid ? src[i] : 0.0f;
        const __half h = __float2half_rn(x);
        const float rest = __fmul_rn(__fsub_rn(x, __half2float(h)), 2048.0f);
        hi[i] = h;
        lo[i] = __float2half_rn(rest);
        bad |= fabsf(x) > 60000.0f;
    }
    if (bad) {
        atomicOr(overflow, 1);
        if (overflow_host) atomicOr(overflow_host, 1);
    }
    if (init_state && tid < n_valid)
        init_query_state(static_cast<int>(tid), static_cast<int>(n_valid), floor_score, thr, floor_out, retry);
}

// one CTA per query: admitted (dot,row) pairs -> scores -> top-k, or flag the query for the row scan.
// The candidates of a query lie in n_seg private segments (one per epilogue thread that served it).
// Shared memory: [fast_cap keys | kSelOut survivor keys | kSelBuckets histogram words].
constexpr int kSelOut = 1024;
__global__ void __launch_bounds__(kSelectThreads)
finalize_kernel(const uint64_t* cand, const uint32_t* cand_count, int n_seg, uint32_t cap_seg, int fast_cap,
                const float* thr, const float* floor_x, int k, int64_t item_offset, int64_t* out_items,
                float* out_scores, int32_t* out_counts, int32_t* retry, int32_t* retry_total,
                int32_t* retry_total_host) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint64_t* keys = reinterpret_cast<uint64_t*>(smem_raw);
    uint64_t* sel_out = keys + fast_cap;
    uint32_t* hist = reinterpret_cast<uint32_t*>(sel_out + kSelOut);
    __shared__ uint32_t s_prefix[kMaxSegments + 1];
    __shared__ int s_cnt, s_overflow;
    __shared__ uint64_t s_admit;
    const int q = blockIdx.x, tid = threadIdx.x;
    const uint32_t* counts = cand_count + static_cast<size_t>(q) * n_seg;
    if (tid == 0) s_overflow = 0;
    __syncthreads();
    for (int sgm = tid; sgm < n_seg; sgm += kSelectThreads) {
        const uint32_t c = __ldcg(&counts[sgm]);
        s_prefix[sgm + 1] = c;
        if (c > cap_seg) s_overflow = 1;
    }
    __syncthreads();
    if (tid < 32) {  // inclusive scan of the segment counts by one warp
        uint32_t carry = 0;
        for (int base = 0; base < n_seg; base += 32) {
            const int i = base + tid;
            uint32_t v = i < n_seg ? s_prefix[i + 1] : 0u;
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) {
                const uint32_t o = __shfl_up_sync(0xFFFFFFFFu, v, off);
                if (tid >= off) v += o;
            }
            if (i < n_seg) s_prefix[i + 1] = v + carry;
            carry += __shfl_sync(0xFFFFFFFFu, v, 31);
        }
        if (tid == 0) s_prefix[0] = 0;
    }
    __syncthreads();
    const uint32_t total = s_prefix[n_seg];
    const bool overflow = s_overflow != 0;
    const bool starved = total < static_cast<uint32_t>(k) && thr[q] > floor_x[q];
    int64_t* items = out_items + static_cast<size_t>(q) * k;
    float* scores = out_scores + static_cast<size_t>(q) * k;
    if (overflow || starved) {  // CTA-uniform
        for (int j = tid; j < k; j += kSelectThreads) {
            items[j] = -1;
            scores[j] = 0.0f;
        }
        if (tid == 0) {
            out_counts[q] = 0;
            retry[q] = 1;
            atomicAdd(retry_total, 1);
            if (retry_total_host) atomicAdd(retry_total_host, 1);  // mapped pinned copy: the host reads it without a D2H
        }
        return;
    }
    const uint64_t* in = cand + static_cast<size_t>(q) * n_seg * cap_seg;
    auto to_key = [](uint64_t e) {
        return make_key(score_from_dot(__uint_as_float(static_cast<uint32_t>(e >> 32))), static_cast<uint32_t>(e));
    };
    int n;
    const uint64_t* result = keys;
    if (total <= static_cast<uint32_t>(fast_cap)) {
        // the usual case (~`target` admitted rows): everything into shared memory — a thread per segment,
        // four independent loads in flight each — then the k best by histogram selection
        for (int sgm = tid; sgm < n_seg; sgm += kSelectThreads) {
            const uint32_t base = s_prefix[sgm], cnt = s_prefix[sgm + 1] - base;
            const uint64_t* src = in + static_cast<size_t>(sgm) * cap_seg;
            for (uint32_t i = 0; i < cnt; i += 4) {
                uint64_t e[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) e[u] = i + u < cnt ? __ldcs(&src[i + u]) : 0;
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    if (i + u < cnt) keys[base + i + u] = to_key(e[u]);
            }
        }
        __syncthreads();
        n = -1;
        if (k <= kSelOut / 2 && total > 256) {
            const int got = select_topk_smem<kSelectThreads>(keys, static_cast<int>(total), k, hist, sel_out, kSelOut);
            if (got >= 0) {
                n = min(got, k);
                result = sel_out;
            }
        }
        if (n < 0) {  // few keys, large k, or massive ties: one bitonic sort of everything
            int cap = 32;
            while (cap < static_cast<int>(total)) cap <<= 1;
            for (int i = static_cast<int>(total) + tid; i < cap; i += kSelectThreads) keys[i] = 0;
            bitonic_sort_desc<kSelectThreads>(keys, cap);
            n = min(static_cast<int>(total), k);
        }
    } else {
        // many candidates (large k): stream them through a k-best list with periodic compaction
        const int cap = 1 << (32 - __clz(k + kSelectThreads - 1));
        if (tid == 0) {
            s_cnt = 0;
            s_admit = 0;
        }
        CandList l{keys, &s_cnt, &s_admit};
        int need = 0;
        for (uint32_t base = 0; base < total; base += kSelectThreads) {
            if (__syncthreads_or(need)) {
                need = 0;
                list_compact<kSelectThreads>(l, cap, k, 0);
            }
            const uint32_t e = base + tid;
            uint64_t key = 0;
            if (e < total) {
                int lo = 0, hi = n_seg - 1;  // segment holding flat element e: last sgm with prefix[sgm] <= e
                while (lo < hi) {
                    const int mid = (lo + hi + 1) >> 1;
                    if (s_prefix[mid] <= e) lo = mid;
                    else hi = mid - 1;
                }
                key = to_key(__ldcs(&in[static_cast<size_t>(lo) * cap_seg + (e - s_prefix[lo])]));
            }
            need |= list_push_warp(l, key, e < total && key >= s_admit, cap - kSelectThreads);
        }
        __syncthreads();
        list_compact<kSelectThreads>(l, cap, k, 0);
        n = s_cnt;
    }
    for (int j = tid; j < k; j += kSelectThreads) {
        if (j < n) {
            items[j] = static_cast<int64_t>(key_pos(result[j])) + item_offset;
            scores[j] = key_score(result[j]);
        } else {
            items[j] = -1;
            scores[j] = 0.0f;
        }
    }
    if (tid == 0) out_counts[q] = n;
}

// ---- threshold search (collect plan): per-query totals, then the keys of every segment in CSR order ------
// one warp per query: total admitted rows and the fullest segment (> cap_seg: the query overflowed)
__global__ void collect_count_kernel(const uint32_t* cand_count, int n_seg, int nq, uint32_t* totals, uint32_t* maxseg) {
    const int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (q >= nq) return;
    uint32_t sum = 0, mx = 0;
    for (int sgm = lane; sgm < n_seg; sgm += 32) {
        const uint32_t c = cand_count[static_cast<size_t>(q) * n_seg + sgm];
        sum += c;
        mx = max(mx, c);
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
        sum += __shfl_xor_sync(0xFFFFFFFFu, sum, off);
        mx = max(mx, __shfl_xor_sync(0xFFFFFFFFu, mx, off));
    }
    if (lane == 0) {
        totals[q] = sum;
        maxseg[q] = mx;
    }
}

// one CTA per query with dst_off[q] >= 0: its (dot bits << 32 | row) candidates -> library keys
// (score bits << 32 | row, ~row with ties_low) at dst + dst_off[q], segment after segment
__global__ void __launch_bounds__(kSelectThreads)
collect_gather_kernel(const uint64_t* cand, const uint32_t* cand_count, int n_seg, uint32_t cap_seg,
                      const int64_t* dst_off, uint64_t* dst, int ties_low) {
    __shared__ uint32_t s_prefix[kMaxSegments + 1];
    const int q = blockIdx.x, tid = threadIdx.x;
    const int64_t base = dst_off[q];
    if (base < 0) return;
    const uint32_t* counts = cand_count + static_cast<size_t>(q) * n_seg;
    if (tid < 32) {  // exclusive scan of the segment counts by one warp
        uint32_t carry = 0;
        for (int b0 = 0; b0 < n_seg; b0 += 32) {
            const int i = b0 + tid;
            const uint32_t c = i < n_seg ? min(counts[i], cap_seg) : 0u;
            uint32_t v = c;
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) {
                const uint32_t o = __shfl_up_sync(0xFFFFFFFFu, v, off);
                if (tid >= off) v += o;
            }
            if (i < n_seg) s_prefix[i] = carry + v - c;
            carry += __shfl_sync(0xFFFFFFFFu, v, 31);
        }
        if (tid == 0) s_prefix[n_seg] = carry;
    }
    __syncthreads();
    const uint64_t* in = cand + static_cast<size_t>(q) * n_seg * cap_seg;
    const int warp = tid >> 5, lane = tid & 31;
    for (int sgm = warp; sgm < n_seg; sgm += kSelectThreads / 32) {  // a warp per segment, coalesced
        const uint32_t n = s_prefix[sgm + 1] - s_prefix[sgm];
        const uint64_t* src = in + static_cast<size_t>(sgm) * cap_seg;
        uint64_t* out = dst + base + s_prefix[sgm];
        for (uint32_t i = lane; i < n; i += 32) {
            const uint64_t e = src[i];
            const uint32_t row = static_cast<uint32_t>(e);
            out[i] = make_key(score_from_dot(__uint_as_float(static_cast<uint32_t>(e >> 32))), ties_low ? ~row : row);
        }
    }
}

// ---- host side --------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (fn) return fn;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess)
        return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(p);
    return fn;
}

// row-major [rows, dim] 16-bit matrix; box = 64 elements x box_rows, 128-byte swizzle, zero OOB fill
bool encode_map(CUtensorMap* map, int dtype, const void* base, int64_t rows, int dim, int box_rows) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) return false;
    const cuuint64_t dims[2] = {static_cast<cuuint64_t>(dim), static_cast<cuuint64_t>(rows)};
    const cuuint64_t strides[1] = {static_cast<cuuint64_t>(dim) * 2};
    const cuuint32_t box[2] = {kBK, static_cast<cuuint32_t>(box_rows)};
    const cuuint32_t estr[2] = {1, 1};
    const CUtensorMapDataType dt =
        dtype == TAV_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    return fn(map, dt, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
              CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

struct Plan {
    int sms;
    int nqc;           // query chunks of 128
    int nq_pad;        // nqc * 128
    int tile_n;        // corpus rows per tile: 256, or 128 in the split form
    int n_tiles;
    int n_full_tiles;
    int kb_count;
    int n_sample;      // tiles in the sample pass (0 = no sampling)
    int sample_gph;    // blocks per 128 rows in the sample pass (block = 128 / sample_gph rows)
    int sample_use;    // blocks the threshold uses, every sample_stride-th of the stored ones
    int sample_stride;
    int sample_units;  // a multiple of nqc
    int main_units;    // a multiple of nqc
    int n_seg;         // candidate segments per query = 4 * main_units / nqc
    uint32_t cap_seg;  // rows a segment holds
    // workspace offsets
    size_t off_q, off_q_lo, off_sample, off_thr, off_floor, off_count, off_done, off_cand, total;
};

// collect_cap >= 0: the threshold search's collect plan (tav_range_search): no sample pass, segments of
// collect_cap keys (at most what a segment can see), `force_per_chunk` units per query chunk when > 0 (a
// re-pass must split the rows into the same segments as its first pass), candidates of padded queries not
// stored (they admit nothing)
Plan make_plan(int device, int64_t n_rows, int dim, int nq, int k, bool split, int force_per_chunk = 0,
               int64_t collect_cap = -1) {
    Plan p{};
    p.sms = 132;
    cudaDeviceGetAttribute(&p.sms, cudaDevAttrMultiProcessorCount, device);
    p.nqc = std::max(1, (nq + kBM - 1) / kBM);
    p.nq_pad = p.nqc * kBM;
    p.tile_n = split ? kTileRowsSplit : kTileRows;
    p.n_tiles = static_cast<int>((n_rows + p.tile_n - 1) / p.tile_n);
    p.n_full_tiles = static_cast<int>(n_rows / p.tile_n);
    p.kb_count = (dim + kBK - 1) / kBK;
    const int max_units = p.sms;
    // Rows we aim to admit per query (`target`).  The threshold is the m-th largest (m = kSampleTop = 8)
    // block maximum of a uniform sample of L blocks of 128 rows; with p = target / N the chance that a
    // block's maximum clears the p-quantile is q_b = 1 - (1-p)^128, so L = m / q_b blocks put the m-th
    // largest block maximum at that quantile.  The number of corpus rows above it is then ~target *
    // Gamma(m)/m, so a query starves (< k admitted) with probability P(Gamma(8) < 8k/target): 6e-8 at
    // target = 16k — and never for k <= 8, because the 8 block maxima are 8 distinct admitted rows.
    // Overflow (> 8*target admitted) is rarer still.  Either way the query is merely redone by the exact
    // row scan.  Large corpora aim at 2048 rows, small ones at 128; never fewer than 16k.
    // For k <= 8 nothing can starve, so small corpora aim much lower (32 rows: a quarter of the corpus is
    // sampled, with the branch-free epilogue, and MAIN's epilogue then rarely has anything to append).
    static const int64_t small_k_floor = [] {
        const char* e = getenv("TAV_SMALLK_TARGET");  // tuning knob of the small-k admission target
        const int64_t v = e ? atoll(e) : 0;
        return v >= 8 ? v : int64_t(32);
    }();
    const int64_t target = k <= kSampleTop
                               ? std::min<int64_t>(2048, std::max<int64_t>(small_k_floor, n_rows / 4096))
                               : std::max<int64_t>(16ll * k, std::min<int64_t>(2048, std::max<int64_t>(128, n_rows / 4096)));
    int64_t admitted = n_rows;  // rows a query is expected to admit
    const int64_t per_tile = static_cast<int64_t>(p.tile_n / 128);  // 128-row spans per tile (x sample_gph blocks)
    if (collect_cap >= 0 || n_rows <= 16384 || 8 * target >= n_rows || p.n_full_tiles < 8) {
        p.n_sample = 0;
    } else {
        // Block size: the m-th largest of L block maxima sits at the row quantile p when 1 - (1-p)^b = m / L;
        // for p * b well above 1 every block clears the quantile and the maxima say nothing about it (the
        // threshold would come out too high and queries starve).  So mid-size corpora — where the target is a
        // larger fraction of the rows — use blocks of 32 or 8 rows instead of 128.
        const double prob = static_cast<double>(target) / static_cast<double>(n_rows);
        const int block_rows = prob * 128 <= 0.7 ? 128 : (prob * 32 <= 0.7 ? 32 : 8);
        p.sample_gph = 128 / block_rows;
        const double q_b = 1.0 - pow(1.0 - prob, static_cast<double>(block_rows));
        const int64_t blocks = static_cast<int64_t>(ceil(kSampleTop / q_b));
        const int64_t blocks_per_tile = per_tile * p.sample_gph;
        p.n_sample = static_cast<int>(std::min<int64_t>(
            p.n_full_tiles, std::max<int64_t>(4, (blocks + blocks_per_tile - 1) / blocks_per_tile)));
        const int64_t stored = static_cast<int64_t>(p.n_sample) * blocks_per_tile;
        p.sample_use = static_cast<int>(std::min<int64_t>(blocks, stored));
        p.sample_stride = static_cast<int>(std::max<int64_t>(1, stored / p.sample_use));
        admitted = target;
    }
    // sample units: chunk-bound (unit u serves chunk u % nqc), so a multiple of nqc
    {
        const int per_chunk = std::max(1, std::min(std::max(1, max_units / p.nqc), std::max(1, p.n_sample)));
        p.sample_units = per_chunk * p.nqc;  // may exceed max_units when nqc > max_units: extra units queue
    }
    {
        // every unit of a chunk owns four candidate segments per query (one per thread of the quad that
        // holds the query): room for 16x the expected share of a segment (at least half a tile's share),
        // and for every row it can see when nothing is cut
        const int per_chunk = force_per_chunk > 0 ? force_per_chunk : std::max(
            1, std::min(std::min(std::max(1, max_units / p.nqc), p.n_tiles), kMaxSegments / kSegPerUnit));
        p.main_units = per_chunk * p.nqc;
        p.n_seg = kSegPerUnit * per_chunk;
        const int64_t tiles_per_unit = (p.n_tiles + per_chunk - 1) / per_chunk;
        const int64_t seen = tiles_per_unit * (p.tile_n / kSegPerUnit);
        const int64_t want = p.n_sample == 0 ? seen : std::max<int64_t>(p.tile_n / (2 * kSegPerUnit), (16 * admitted + p.n_seg - 1) / p.n_seg);
        p.cap_seg = static_cast<uint32_t>(std::min<int64_t>(want, seen));
        if (collect_cap >= 0) p.cap_seg = static_cast<uint32_t>(std::max<int64_t>(1, std::min<int64_t>(collect_cap, seen)));
    }
    auto align = [](size_t v) { return (v + 255) & ~size_t(255); };
    // the sampler's self-resetting unit counters live at a FIXED place (offset 0), whatever the shape of
    // the search: they must read zero at the start of every search and only the kernels ever write them
    size_t off = 0;
    p.off_done = off;
    off = align(off + static_cast<size_t>(kMaxChunks) * sizeof(uint32_t));
    p.off_q = off;
    off = align(off + static_cast<size_t>(p.nq_pad) * dim * 2);
    p.off_q_lo = off;  // lo plane of the queries (split form only; reserved always)
    off = align(off + static_cast<size_t>(p.nq_pad) * dim * 2);
    p.off_sample = off;  // block maxima [n_sample * blocks per tile, nq_pad]
    off = align(off + static_cast<size_t>(std::max(1, p.n_sample)) * per_tile * std::max(1, p.sample_gph) * p.nq_pad *
                          sizeof(float));
    p.off_thr = off;
    off = align(off + static_cast<size_t>(p.nq_pad) * sizeof(float));
    p.off_floor = off;
    off = align(off + static_cast<size_t>(p.nq_pad) * sizeof(float));
    p.off_count = off;
    off = align(off + static_cast<size_t>(p.nq_pad) * p.n_seg * sizeof(uint32_t));
    p.off_cand = off;
    off = align(off + static_cast<size_t>(collect_cap >= 0 ? nq : p.nq_pad) * p.n_seg * p.cap_seg * sizeof(uint64_t));
    p.total = off;
    return p;
}

struct Maps {
    CUtensorMap q, q_lo;  // queries, 128-row boxes (hi plane / lo plane when split)
    CUtensorMap c, c_lo;  // corpus, one tile of rows per box
};

template <int MODE, bool BF16, bool SPLIT>
cudaError_t launch_kernel_t(const Maps& m, const KernelArgs& ka, int units, cudaStream_t s) {
    auto kern = mma_topk_kernel<MODE, BF16, SPLIT>;
    static int granted[16] = {};
    cudaError_t e = ensure_dynamic_smem(kern, kSmemBytes, granted);
    if (e != cudaSuccess) return e;
    kern<<<units, kMmaThreads, kSmemBytes, s>>>(m.q, m.c, m.q_lo, m.c_lo, ka);
    return cudaGetLastError();
}

// split: two-plane fp16 (float32 data)
template <int MODE>
cudaError_t launch_kernel(const Maps& m, const KernelArgs& ka, int dtype, bool split, int units, cudaStream_t s) {
    if (split) return launch_kernel_t<MODE, false, true>(m, ka, units, s);
    if (dtype == TAV_BF16) return launch_kernel_t<MODE, true, false>(m, ka, units, s);
    return launch_kernel_t<MODE, false, false>(m, ka, units, s);
}

cudaError_t prep_queries(const MmaArgs& a, void* dst, void* dst_lo, int nq_pad, int init_state, float* thr,
                         float* floor_out, cudaStream_t s) {
    const int64_t total = static_cast<int64_t>(nq_pad) * a.dim;
    const int grid = static_cast<int>(std::max<int64_t>(
        std::min<int64_t>((total + 255) / 256, 132 * 8),
        init_state ? (a.nq + 255) / 256 : 1));
    if (a.split) {
        split_rows_kernel<<<grid, 256, 0, s>>>(a.queries, static_cast<__half*>(dst), static_cast<__half*>(dst_lo),
                                               a.nq, nq_pad, a.dim, a.split_overflow, a.split_overflow_host, init_state,
                                               a.floor_score, thr, floor_out, a.retry_flags);
        return cudaGetLastError();
    }
    if (a.dtype == TAV_BF16)
        query_prep_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(a.queries, static_cast<__nv_bfloat16*>(dst), a.nq, nq_pad,
                                                              a.dim, init_state, a.floor_score, thr, floor_out,
                                                              a.retry_flags);
    else
        query_prep_kernel<__half><<<grid, 256, 0, s>>>(a.queries, static_cast<__half*>(dst), a.nq, nq_pad, a.dim,
                                                       init_state, a.floor_score, thr, floor_out, a.retry_flags);
    return cudaGetLastError();
}

}  // namespace

bool mma_supported(int dtype, int dim) {
    return (dtype == TAV_BF16 || dtype == TAV_F16) && dim >= 8 && dim % 8 == 0;
}
bool mma_split_supported(int dim) { return dim >= 8 && dim % 8 == 0; }

cudaError_t launch_split_rows(const float* src, void* hi, void* lo, int64_t n, int dim, int* overflow,
                              cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    const int64_t total = n * dim;
    const int grid = static_cast<int>(std::min<int64_t>((total + 255) / 256, 132 * 16));
    split_rows_kernel<<<grid, 256, 0, s>>>(src, static_cast<__half*>(hi), static_cast<__half*>(lo), n, n, dim, overflow,
                                           nullptr, 0, 0.0f, nullptr, nullptr, nullptr);
    return cudaGetLastError();
}

namespace {
// storage dtype the tensor-core kernel sees: fp16 planes for split float32 data
inline int mma_dtype(const MmaArgs& a) { return a.split ? TAV_F16 : a.dtype; }

bool build_maps_uncached(const MmaArgs& a, const void* d_q, const void* d_q_lo, int nq_pad, Maps& m);

// cuTensorMapEncodeTiled costs 1-2 us a piece and a search needs four: remember, per device, the maps of
// the last search (serving loops repeat the same corpus / workspace pointers and shapes)
struct MapCacheEntry {
    const void *corpus = nullptr, *corpus_lo = nullptr, *q = nullptr, *q_lo = nullptr;
    int64_t n = -1;
    int dim = 0, dt = -1, nq_pad = 0;
    Maps maps;
    bool valid = false;
};
std::mutex g_map_mu;
MapCacheEntry g_map_cache[16];

bool build_maps(const MmaArgs& a, const void* d_q, const void* d_q_lo, int nq_pad, Maps& m) {
    const int dt = mma_dtype(a);
    std::lock_guard<std::mutex> lock(g_map_mu);
    MapCacheEntry& e = g_map_cache[a.device >= 0 && a.device < 16 ? a.device : 0];
    const void* lo = a.split ? a.corpus_lo : nullptr;
    if (!(e.valid && e.corpus == a.corpus && e.corpus_lo == lo && e.q == d_q && e.q_lo == d_q_lo && e.n == a.n_corpus &&
          e.dim == a.dim && e.dt == dt && e.nq_pad == nq_pad)) {
        e.valid = false;
        if (!build_maps_uncached(a, d_q, d_q_lo, nq_pad, e.maps)) return false;
        e.corpus = a.corpus, e.corpus_lo = lo, e.q = d_q, e.q_lo = d_q_lo, e.n = a.n_corpus;
        e.dim = a.dim, e.dt = dt, e.nq_pad = nq_pad;
        e.valid = true;
    }
    m = e.maps;
    return true;
}

bool build_maps_uncached(const MmaArgs& a, const void* d_q, const void* d_q_lo, int nq_pad, Maps& m) {
    const int dt = mma_dtype(a);
    const int tile_n = a.split ? kTileRowsSplit : kTileRows;
    if (!encode_map(&m.c, dt, a.corpus, a.n_corpus, a.dim, tile_n)) return false;
    const void* lo = a.split ? a.corpus_lo : a.corpus;  // unused maps still need a valid encoding
    if (!encode_map(&m.c_lo, dt, lo, a.n_corpus, a.dim, tile_n)) return false;
    if (!encode_map(&m.q, dt, d_q, nq_pad, a.dim, kBM)) return false;
    return encode_map(&m.q_lo, dt, a.split ? d_q_lo : d_q, nq_pad, a.dim, kBM);
}
bool args_ok(const MmaArgs& a) {
    if (a.n_corpus >= (1ll << 31) || reinterpret_cast<uintptr_t>(a.corpus) % 16 != 0) return false;
    if (a.split) return a.dtype == TAV_F32 && mma_split_supported(a.dim) && a.corpus_lo && a.split_overflow;
    return mma_supported(a.dtype, a.dim);
}
}  // namespace

size_t mma_workspace_bytes(const MmaArgs& a) {
    return make_plan(a.device, a.n_corpus, a.dim, a.nq, a.k, a.split != 0).total;
}

cudaError_t launch_mma_search(const MmaArgs& a, void* workspace, size_t workspace_bytes, cudaStream_t s,
                              int* launches) {
    if (!args_ok(a) || a.k > kPassK || a.nq < 1 || a.nq > kMmaMaxQueries) return cudaErrorInvalidValue;
    const Plan p = make_plan(a.device, a.n_corpus, a.dim, a.nq, a.k, a.split != 0);
    if (workspace_bytes < p.total) return cudaErrorInvalidValue;
    char* ws = static_cast<char*>(workspace);
    void* d_q = ws + p.off_q;
    void* d_q_lo = ws + p.off_q_lo;
    float* d_sample = reinterpret_cast<float*>(ws + p.off_sample);
    float* d_thr = reinterpret_cast<float*>(ws + p.off_thr);
    float* d_floor = reinterpret_cast<float*>(ws + p.off_floor);
    uint32_t* d_count = reinterpret_cast<uint32_t*>(ws + p.off_count);
    uint32_t* d_done = reinterpret_cast<uint32_t*>(ws + p.off_done);
    uint64_t* d_cand = reinterpret_cast<uint64_t*>(ws + p.off_cand);
    int n_launch = 0, ev_used = 0;
    cudaError_t e;
    // event pairs around the kernels: all of them, or (ev_main_only) only around the dominant kernel — two
    // event records per kernel boundary are a measurable share of a 0.1-0.4 ms search
    bool ev_open = false;
    auto ev_begin_kind = [&](int kind) -> cudaError_t {
        ev_open = a.ev && ev_used < a.ev_max && (!a.ev_main_only || kind == 0);
        return ev_open ? cudaEventRecord(a.ev[ev_used][0], s) : cudaSuccess;
    };
    auto ev_end = [&](int kind) -> cudaError_t {
        if (!ev_open) return cudaSuccess;
        ev_open = false;
        if (a.ev_kind) a.ev_kind[ev_used] = kind;
        return cudaEventRecord(a.ev[ev_used++][1], s);
    };

    // tensor maps first (host work only), so that the launches below go out back to back
    Maps maps;
    if (!build_maps(a, d_q, d_q_lo, p.nq_pad, maps)) return cudaErrorUnknown;

    // queries -> storage dtype; without a sample pass this launch also initialises thresholds / counters
    if ((e = ev_begin_kind(2)) != cudaSuccess) return e;
    e = prep_queries(a, d_q, d_q_lo, p.nq_pad, p.n_sample == 0 ? 1 : 0, d_thr, d_floor, s);
    if (e != cudaSuccess) return e;
    if ((e = ev_end(2)) != cudaSuccess) return e;
    ++n_launch;
    const int kdt = mma_dtype(a);
    const bool split = a.split != 0;

    KernelArgs ka{};
    ka.n_rows = a.n_corpus;
    ka.kb_count = p.kb_count;
    ka.nq = a.nq;
    ka.nqc = p.nqc;
    ka.nq_pad = p.nq_pad;
    ka.thr = d_thr;
    ka.floor_x = d_floor;
    ka.sample_max = d_sample;
    ka.sample_gph = std::max(1, p.sample_gph);
    ka.sample_use = p.sample_use;
    ka.sample_stride = std::max(1, p.sample_stride);
    ka.sample_done = d_done;
    ka.retry = a.retry_flags;
    ka.floor_score = a.floor_score;
    ka.cand = d_cand;
    ka.cand_count = d_count;
    ka.cap_seg = p.cap_seg;
    ka.n_seg = p.n_seg;
    ka.row_mask = a.row_mask;
    ka.qmask = a.qmask;
    ka.pop_exact = std::max<uint32_t>(p.cap_seg, static_cast<uint32_t>(a.k));

    if (p.n_sample > 0) {
        // strided sample of FULL tiles; the last unit of every query chunk publishes the thresholds
        ka.n_tiles_work = p.n_sample;
        ka.tile_mul = p.n_full_tiles;
        ka.tile_div = p.n_sample;
        if ((e = ev_begin_kind(1)) != cudaSuccess) return e;
        e = ka.qmask.bits ? launch_kernel<kSampleQ>(maps, ka, kdt, split, p.sample_units, s)
                          : launch_kernel<kSample>(maps, ka, kdt, split, p.sample_units, s);
        if (e != cudaSuccess) return e;
        if ((e = ev_end(1)) != cudaSuccess) return e;
        ++n_launch;
    }

    ka.n_tiles_work = p.n_tiles;
    ka.tile_mul = 1;
    ka.tile_div = 1;
    if ((e = ev_begin_kind(0)) != cudaSuccess) return e;
    e = ka.qmask.bits ? launch_kernel<kMainQ>(maps, ka, kdt, split, p.main_units, s)
                      : launch_kernel<kMain>(maps, ka, kdt, split, p.main_units, s);
    if (e != cudaSuccess) return e;
    if ((e = ev_end(0)) != cudaSuccess) return e;
    ++n_launch;

    // shared memory sized to what this search can need: all candidates of a query (bounded by the segments'
    // capacity and kFinalizeFast) or the streaming list for large k, + the selection's survivors and histogram
    const int64_t most = static_cast<int64_t>(p.n_seg) * p.cap_seg;
    const int fast_cap = std::max(next_pow2(a.k + kSelectThreads),
                                  static_cast<int>(std::min<int64_t>(kFinalizeFast, next_pow2(static_cast<int>(std::min<int64_t>(most, kFinalizeFast))))));
    const size_t sel_smem = static_cast<size_t>(fast_cap) * sizeof(uint64_t) + kSelOut * sizeof(uint64_t) +
                            kSelBuckets * sizeof(uint32_t);
    static int finalize_granted[16] = {};
    e = ensure_dynamic_smem(finalize_kernel, sel_smem, finalize_granted);
    if (e != cudaSuccess) return e;
    if ((e = ev_begin_kind(2)) != cudaSuccess) return e;
    finalize_kernel<<<a.nq, kSelectThreads, sel_smem, s>>>(d_cand, d_count, p.n_seg, p.cap_seg, fast_cap, d_thr, d_floor,
                                                           a.k, a.item_offset, a.out_items, a.out_scores,
                                                           a.out_counts, a.retry_flags, a.retry_total, a.retry_total_host);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    if ((e = ev_end(2)) != cudaSuccess) return e;
    ++n_launch;

    if (launches) *launches = n_launch;
    if (a.ev_used) *a.ev_used = ev_used;
    return cudaSuccess;
}

MmaCollect mma_collect_plan(const MmaArgs& a, int per_chunk, int64_t cap_seg) {
    const Plan p = make_plan(a.device, a.n_corpus, a.dim, a.nq, 1, a.split != 0, per_chunk, std::max<int64_t>(cap_seg, 1));
    MmaCollect c;
    c.per_chunk = p.n_seg / kSegPerUnit;
    c.n_seg = p.n_seg;
    c.cap_seg = p.cap_seg;
    c.ws_bytes = p.total;
    return c;
}

cudaError_t launch_mma_collect(const MmaArgs& a, const MmaCollect& c, void* workspace, uint32_t* totals,
                               uint32_t* maxseg, cudaStream_t s, int* launches) {
    if (!args_ok(a) || a.nq < 1 || a.nq > kMmaMaxQueries || !a.retry_flags) return cudaErrorInvalidValue;
    const Plan p = make_plan(a.device, a.n_corpus, a.dim, a.nq, 1, a.split != 0, c.per_chunk, c.cap_seg);
    if (p.n_seg != c.n_seg || p.cap_seg != c.cap_seg) return cudaErrorInvalidValue;
    char* ws = static_cast<char*>(workspace);
    void* d_q = ws + p.off_q;
    void* d_q_lo = ws + p.off_q_lo;
    float* d_thr = reinterpret_cast<float*>(ws + p.off_thr);
    float* d_floor = reinterpret_cast<float*>(ws + p.off_floor);
    uint32_t* d_count = reinterpret_cast<uint32_t*>(ws + p.off_count);
    Maps maps;
    if (!build_maps(a, d_q, d_q_lo, p.nq_pad, maps)) return cudaErrorUnknown;
    // queries -> storage dtype, thresholds = the exact dot floor of min_score (no sample pass)
    cudaError_t e = prep_queries(a, d_q, d_q_lo, p.nq_pad, 1, d_thr, d_floor, s);
    if (e != cudaSuccess) return e;
    KernelArgs ka{};
    ka.n_rows = a.n_corpus;
    ka.kb_count = p.kb_count;
    ka.nq = a.nq;
    ka.nqc = p.nqc;
    ka.nq_pad = p.nq_pad;
    ka.thr = d_thr;
    ka.floor_x = d_floor;
    ka.cand = reinterpret_cast<uint64_t*>(ws + p.off_cand);
    ka.cand_count = d_count;
    ka.cap_seg = p.cap_seg;
    ka.n_seg = p.n_seg;
    ka.row_mask = a.row_mask;
    ka.qmask = a.qmask;
    ka.n_tiles_work = p.n_tiles;
    ka.tile_mul = 1;
    ka.tile_div = 1;
    const bool timed = a.ev && a.ev_used && *a.ev_used < a.ev_max;
    if (timed && (e = cudaEventRecord(a.ev[*a.ev_used][0], s)) != cudaSuccess) return e;
    e = ka.qmask.bits ? launch_kernel<kMainQ>(maps, ka, mma_dtype(a), a.split != 0, p.main_units, s)
                      : launch_kernel<kMain>(maps, ka, mma_dtype(a), a.split != 0, p.main_units, s);
    if (e != cudaSuccess) return e;
    if (timed) {
        if (a.ev_kind) a.ev_kind[*a.ev_used] = 0;
        if ((e = cudaEventRecord(a.ev[(*a.ev_used)++][1], s)) != cudaSuccess) return e;
    }
    collect_count_kernel<<<(a.nq + 7) / 8, 256, 0, s>>>(d_count, p.n_seg, a.nq, totals, maxseg);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    if (launches) *launches += 3;
    return cudaSuccess;
}

cudaError_t launch_mma_gather(const MmaArgs& a, const MmaCollect& c, void* workspace, const int64_t* dst_off,
                              uint64_t* dst, int ties_low, cudaStream_t s) {
    const Plan p = make_plan(a.device, a.n_corpus, a.dim, a.nq, 1, a.split != 0, c.per_chunk, c.cap_seg);
    char* ws = static_cast<char*>(workspace);
    collect_gather_kernel<<<a.nq, kSelectThreads, 0, s>>>(reinterpret_cast<const uint64_t*>(ws + p.off_cand),
                                                          reinterpret_cast<const uint32_t*>(ws + p.off_count), p.n_seg,
                                                          p.cap_seg, dst_off, dst, ties_low);
    return cudaGetLastError();
}

// Debug / verification entry: all raw dot products of the tensor-core path, out[nq, n_rows] (device).
cudaError_t launch_mma_dump(const MmaArgs& a, void* workspace, size_t workspace_bytes, float* out, cudaStream_t s) {
    if (!args_ok(a) || a.nq < 1 || a.nq > kMmaMaxQueries) return cudaErrorInvalidValue;
    Plan p = make_plan(a.device, a.n_corpus, a.dim, a.nq, 1, a.split != 0);
    if (workspace_bytes < p.total) return cudaErrorInvalidValue;
    char* ws = static_cast<char*>(workspace);
    void* d_q = ws + p.off_q;
    void* d_q_lo = ws + p.off_q_lo;
    cudaError_t e = prep_queries(a, d_q, d_q_lo, p.nq_pad, 0, nullptr, nullptr, s);
    if (e != cudaSuccess) return e;
    Maps maps;
    if (!build_maps(a, d_q, d_q_lo, p.nq_pad, maps)) return cudaErrorUnknown;
    KernelArgs ka{};
    ka.n_rows = a.n_corpus;
    ka.kb_count = p.kb_count;
    ka.nq = a.nq;
    ka.nqc = p.nqc;
    ka.nq_pad = p.nq_pad;
    ka.n_tiles_work = p.n_tiles;
    ka.tile_mul = 1;
    ka.tile_div = 1;
    ka.dump = out;
    return launch_kernel<kDump>(maps, ka, mma_dtype(a), a.split != 0, p.main_units, s);
}

}  // namespace tav
