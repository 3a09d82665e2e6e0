// tav_api.cu — the C ABI of libtavec (include/tavec.h): index lifecycle, append / adopt,
// the search dispatcher (row-scan path or wgmma tensor-core path) and the shard-merge entry point.
//
// Reference surface this stands in for (src/typeagent/aitools/vectorbase.py):
//   add_embedding(s) :115-148 -> tav_append          clear :253-256        -> tav_clear
//   deserialize      :273-287 -> tav_append (bulk)   fuzzy_lookup_embedding :163-201 and
//   fuzzy_lookup_embedding_in_subset :203-230        -> tav_search
// There is no CPU path in this library: every entry point that computes needs a CUDA device.

#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include <algorithm>
#include <atomic>
#include <mutex>
#include <new>
#include <string>
#include <vector>

#include "tav_common.cuh"
#include "tav_internal.h"

namespace tav {

static thread_local char g_error[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_error, sizeof(g_error), fmt, ap);
    va_end(ap);
}

static inline size_t dtype_size(int dt) { return dt == TAV_F32 ? 4 : 2; }
static inline bool dtype_ok(int dt) { return dt == TAV_F32 || dt == TAV_BF16 || dt == TAV_F16; }

#define TAV_CUDA(expr)                                                                     \
    do {                                                                                   \
        cudaError_t _e = (expr);                                                           \
        if (_e != cudaSuccess) {                                                           \
            set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return _e == cudaErrorMemoryAllocation ? TAV_ERR_OOM : TAV_ERR_CUDA;           \
        }                                                                                  \
    } while (0)

// a grow-only buffer from one alloc / free pair; it owns its memory: freed when it is destroyed, moved, never copied
template <cudaError_t (*Alloc)(void**, size_t), cudaError_t (*Free)(void*)>
struct GrowBuf {
    void* p = nullptr;
    size_t bytes = 0;
    GrowBuf() = default;
    GrowBuf(GrowBuf&& o) noexcept : p(o.p), bytes(o.bytes) {
        o.p = nullptr;
        o.bytes = 0;
    }
    GrowBuf& operator=(GrowBuf&& o) noexcept {
        if (this != &o) {
            release();
            p = o.p;
            bytes = o.bytes;
            o.p = nullptr;
            o.bytes = 0;
        }
        return *this;
    }
    ~GrowBuf() { release(); }
    cudaError_t ensure(size_t need) {
        if (need <= bytes) return cudaSuccess;
        release();
        size_t want = std::max(need, size_t(1) << 16);
        cudaError_t e = Alloc(&p, want);
        if (e == cudaSuccess) bytes = want;
        return e;
    }
    void release() {
        if (p) Free(p);
        p = nullptr;
        bytes = 0;
    }
};
using DevBuf = GrowBuf<cudaMalloc, cudaFree>;
// pinned host memory: staging for truly asynchronous H2D / D2H of small payloads
using PinBuf = GrowBuf<cudaMallocHost, cudaFreeHost>;

constexpr int kMaxTimedKernels = 12;   // event pairs per search (more kernels than that go untimed)
constexpr int kHistory = 64;           // timed searches remembered (tav_timing_history)
constexpr int kMaxPending = 64;        // deferred searches that may await one tav_finish_search
constexpr size_t kPinnedStageLimit = size_t(8) << 20;  // payloads above this go straight from user memory
constexpr size_t kZeroCopyOutLimit = size_t(16) << 10; // results up to this size are written to host memory by the kernels
constexpr size_t kAppendStageBytes = size_t(32) << 20; // pinned double buffer of the bulk-load path
// the single-launch row scan runs one wave of CTAs (its last CTA merges): a latency form for corpora that
// fit L2; bigger scans want 4 CTAs per SM in flight and take the two-kernel form
constexpr size_t kFusedScanMaxBytes = size_t(32) << 20;
// single-launch form, k up to this: the host watches the mapped result slots instead of a completion word
constexpr int kWatchSlotsMaxK = 64;
constexpr int64_t kNoItemYet = INT64_MIN;        // no hit has this ordinal ...
constexpr uint32_t kNoScoreYet = 0xFFFFFFFFu;    // ... or this score (a NaN pattern; scores are clipped to [0, 1])

// CUDA events around one search (created lazily, when timing is first enabled)
struct TimedSearch {
    cudaEvent_t total[2] = {nullptr, nullptr};
    cudaEvent_t ev[kMaxTimedKernels][2] = {};
    int kind[kMaxTimedKernels];  // 0 dominant kernel, 1 sample pass, 2 auxiliary
    int used = 0;
    int launches = 0;
    int path = 0;
    bool valid = false;
};

// a TAV_DEFER_RETRY search whose "redo exactly" flags have not been looked at yet
struct Pending {
    const float* queries;  // device: the caller's, or normalised ones in tav_index::held_queries
    int nq, k;
    float floor;
    int64_t item_offset;
    int64_t* items;
    float* scores;
    int32_t* counts;
    int slot;
    bool split;
    const uint32_t* mask;  // the row mask, or query 0's per-query mask (query q's: mask + q * mask_stride)
    int64_t mask_stride;   // 0 for the row mask
    // a threshold search into the caller's buffers (tav_range_search_into; k == 0): `items` / `scores` hold
    // its first `cap` hits, `offsets` its CSR offsets
    int64_t* offsets = nullptr;
    int64_t cap = 0;
    const int64_t* subset = nullptr;  // device ordinals (held, like normalised queries), or nullptr
    int64_t n_scan = 0;
    int ties_low = 0;
    int64_t expected_hits = 0;
    QueryMasks qm{};                  // per-query masks of the whole search (nq > 1)
    int per_chunk = 0, n_seg = 0;     // the tensor-core collection plan a re-pass repeats (0: the row scan)
    // per-query subsets from device memory (tav_search_subsets_into / _range_): the search's status word (device),
    // read at the finish; nothing is redone
    const int* subsets_status = nullptr;
};

}  // namespace tav

using namespace tav;

struct tav_index {
    int device = 0;
    int dim = 0;
    int dtype = TAV_F32;
    int flags = 0;
    int64_t size = 0;
    int64_t capacity = 0;
    void* rows = nullptr;  // [capacity, dim] storage dtype
    bool adopted = false;
    std::mutex mu;         // one call at a time per index (ctypes releases the GIL)

    // search workspace
    DevBuf queries;     // float32 [n_queries, dim]
    DevBuf subset;      // int64 [subset_len]
    DevBuf cand_keys;   // [qb, cand_stride] uint64
    DevBuf cand_count;  // [8] uint64 bounds | [8] uint32 counters | fused ticket
    DevBuf out_pack;    // device result staging for host outputs: [items | scores | counts]
    PinBuf pin_in;      // pinned staging: queries (+ subset) on the way in
    PinBuf pin_out;     // pinned staging: packed results on the way out (+ the completion word)
    PinBuf pin_append[2];             // bulk load: pinned double buffer
    cudaEvent_t ev_append[2] = {nullptr, nullptr};
    bool append_busy[2] = {false, false};  // an H2D copy recorded under ev_append[b] may still read pin_append[b]
    cudaEvent_t ev_pin_in = nullptr;  // completion of the last H2D that read pin_in
    bool pin_in_busy = false;
    uint32_t done_seq = 0;            // completion word sequence of the single-launch form
    DevBuf staging;     // append: source rows before conversion
    DevBuf mma_ws;      // tensor-core path workspace
    // "redo exactly" bookkeeping of the tensor-core path, one slot per outstanding search:
    // [kMaxPending][2] int32 {flagged queries, a query value left the fp16 range} | [kMaxPending][retry_cap] flags
    DevBuf retry;
    PinBuf retry_host;  // mapped pinned twin of the [kMaxPending][2] totals: tav_finish_search reads it without a D2H copy
    int retry_cap = 0;
    std::vector<Pending> pending;
    int next_slot = 0;
    // normalised queries of deferred searches (TAV_NORMALIZE): each pending search owns a region here that
    // later searches do not touch, until tav_finish_search has redone its flagged queries
    DevBuf held_queries;
    size_t held_used = 0;        // bytes of held_queries used by pending searches
    std::vector<DevBuf> held_retired;  // outgrown held_queries buffers that pending searches still read
    int last_first_slot = -1, last_n_slots = 0;   // bookkeeping slots of the most recent search (-1: row scan)
    bool last_split = false;     // the most recent search ran the split form (finish redoes it all on split_flag[0])
    // float32 indexes: the rows as two fp16 planes for the tensor-core path (built lazily,
    // extended on append); split_flag[0] = a corpus value left the fp16 range
    DevBuf split_hi, split_lo, split_flag;
    int64_t split_rows = 0;      // rows [0, split_rows) of the planes are current
    int64_t split_cap = 0;
    // rows were removed or overwritten since the planes were built: the overflow flag may stand for rows that
    // are gone, so the next build looks at it and rebuilds from row 0 (which resets it) when it is set
    bool split_recheck = false;
    // removal (tav_remove_rows): the device copy of the removed-row keys, the compaction policy and what the
    // last removal did (tav_internal_compact_policy / _stats)
    DevBuf compact_keys;
    int compact_mode = 0;            // 0 the default (in place), 1 out of place, 2 in place
    int64_t compact_scratch = 0;     // bytes of the in-place window buffer (0: kCompactScratchBytes)
    int compact_path = 0;            // 0 nothing moved, 1 out of place, 2 in place
    int64_t compact_windows = 0;
    // rebalance (tav_rows_stage / tav_rows_commit): the staged new block and the cap on its allocation
    void* staged = nullptr;
    int64_t staged_rows = 0;
    size_t rows_bytes = 0;           // bytes of the library-owned allocation behind `rows` (0 when adopted)
    size_t staged_bytes = 0;
    int64_t stage_cap = -1;          // bytes, -1 = no cap (tav_internal_stage_cap)
    int64_t qmask_cap = -1;          // bytes of per-query masks, -1 = no cap (tav_internal_qmask_cap)
    bool alloc_fail = false;         // tensor-core searches ask cudaMalloc for too much (tav_internal_search_alloc_fail)
    // predicate pushdown: one bit per row (tav_set_row_mask)
    DevBuf row_mask;
    int64_t row_mask_rows = 0;   // 0 = no mask set
    // per-query masks (tav_set_query_masks): qmask_n rows of qmask_stride words, and their popcounts
    DevBuf qmask, qmask_pop;
    int qmask_n = 0;             // 0 = no masks set
    int64_t qmask_rows = 0;
    int64_t qmask_stride = 0;
    // threshold search (tav_range_search): collect regions, re-pass regions, sort scratch, CSR result
    DevBuf range_keys, range_keys2, range_counts, range_qgather, range_qmap, range_tmp, range_sortws;
    DevBuf range_mmaws, range_mmaws2, range_mmaaux;  // tensor-core collection: workspaces, scratch
    DevBuf range_items, range_scores;
    int64_t range_total = 0;     // hits of the last range search held in range_items / range_scores
    bool range_grouped = false;  // ... and they are the leaders of a tav_range_search_groups (tav_range_fetch_groups)
    // grouped lookups (tav_set_row_groups): the group of every row (group_stage holds an upload until it is checked),
    // and the runs of equal consecutive values, which size the top-k prefix of tav_search_groups
    DevBuf group_map, group_stage, group_stat;
    int64_t group_rows = 0;      // 0 = no map
    int64_t group_runs = 0;
    // leader reduction: segments, open-addressing tables, leader counters; the top-k prefix and its keys
    DevBuf group_segs, group_table, group_counts, group_topk, group_keys, group_csr;
    DevBuf range_groups;         // the groups of the leaders in range_items (tav_range_search_groups)
    DevBuf group_res;            // tav_search_groups with host outputs: [groups | rows | scores | counts]
    bool range_replaced = false; // a tav_range_search_into ran after it: tav_range_fetch has nothing to copy
    // per-query subsets: device [offsets | work-item starts | CSR offsets of the hits], each n_queries + 1
    DevBuf subsets_meta;
    // per-query subsets from device memory: the status words, [kMaxPending] of deferred searches by bookkeeping slot
    // and one of the synchronous form; the first refusal a finish met, reported by tav_finish_search
    DevBuf subsets_status;
    int deferred_rc = TAV_OK;
    std::string deferred_msg;

    // call order on the device (join_stream / mark_queued / wait_queued): ev_last marks the end of the work
    // of the calls so far while `outstanding`; last_stream is ordered after it
    cudaEvent_t ev_last = nullptr;
    cudaStream_t last_stream = nullptr;
    bool outstanding = false;

    // timing
    TimedSearch* hist = nullptr; // [kHistory], created by tav_set_timing(1)
    int64_t search_seq = 0;      // searches timed so far
    TimedSearch untimed;         // path / launch count of the last search when timing is off
    bool timing_on = false;
    bool timing_light = false;  // events only around the dominant kernel and the whole search
};

// Bytes held in row blocks (the library-owned rows of every index of the process, and their staged blocks): every
// such allocation and free goes through these two, so tav_internal_row_bytes can show that a replaced block was freed.
static std::atomic<int64_t> g_row_bytes{0};
static cudaError_t rows_malloc(void** p, size_t bytes) {
    cudaError_t e = cudaMalloc(p, bytes);
    if (e == cudaSuccess) g_row_bytes += static_cast<int64_t>(bytes);
    return e;
}
static void rows_free(void* p, size_t bytes) {
    if (!p) return;
    cudaFree(p);
    g_row_bytes -= static_cast<int64_t>(bytes);
}

static TimedSearch* cur_timed(tav_index* ix) {
    return ix->timing_on && ix->hist ? &ix->hist[(ix->search_seq) % kHistory] : nullptr;
}
static TimedSearch* last_timed(tav_index* ix) {
    if (ix->timing_on && ix->hist && ix->search_seq > 0) return &ix->hist[(ix->search_seq - 1) % kHistory];
    return &ix->untimed;
}

// The pinned input staging may still be the source of an in-flight H2D copy when the previous
// search returned without synchronising (device outputs): wait for that copy before reuse.
static cudaError_t pin_in_acquire(tav_index* ix, size_t bytes) {
    if (ix->pin_in_busy) {
        cudaError_t e = cudaEventSynchronize(ix->ev_pin_in);
        if (e != cudaSuccess) return e;
        ix->pin_in_busy = false;
    }
    return ix->pin_in.ensure(bytes);
}

static int set_device(const tav_index* ix) {
    TAV_CUDA(cudaSetDevice(ix->device));
    return TAV_OK;
}

// The device work of the calls on one index runs in the order of the calls, whatever stream each names.
// A call that may return with work still queued records ev_last behind it (mark_queued); a call that
// synchronises its stream after joining it leaves nothing queued (mark_done).  On entry a call on another
// stream makes that stream wait for ev_last (an event, not the earlier stream: that one may be gone by now);
// consecutive calls on one stream issue no CUDA call for this.
static int join_stream(tav_index* ix, cudaStream_t s) {
    if (ix->outstanding && s != ix->last_stream) TAV_CUDA(cudaStreamWaitEvent(s, ix->ev_last, 0));
    ix->last_stream = s;  // whatever is enqueued on s from here on runs after ev_last
    return TAV_OK;
}

static int mark_queued(tav_index* ix, cudaStream_t s) {
    TAV_CUDA(cudaEventRecord(ix->ev_last, s));
    ix->last_stream = s;
    ix->outstanding = true;
    return TAV_OK;
}

// entry of the calls that name a stream: the index's device, and s ordered after the earlier calls' work
static int enter_stream(tav_index* ix, cudaStream_t s) {
    if (int rc = set_device(ix)) return rc;
    return join_stream(ix, s);
}

static void mark_done(tav_index* ix) { ix->outstanding = false; }

// the entry points without a stream (clear, adopt, reserve): the host waits for the earlier calls' work
static int wait_queued(tav_index* ix) {
    if (ix->outstanding) TAV_CUDA(cudaEventSynchronize(ix->ev_last));
    ix->outstanding = false;
    return TAV_OK;
}

static int finish_pending(tav_index* ix, cudaStream_t s, int* redone);

// bitmask words of n_rows rows padded to whole 256-row tiles (the tensor-core epilogue reads one word per 32 rows
// of a tile)
static inline int64_t mask_words(int64_t n_rows) { return (n_rows + 255) / 256 * 8; }

// numpy's IndexError for ordinals outside [-size, size)
static int check_subset_ordinals(const tav_index* ix, const int64_t* ordinals, int64_t n) {
    for (int64_t i = 0; i < n; ++i)
        if (ordinals[i] < -ix->size || ordinals[i] >= ix->size) {
            set_error("index %lld is out of bounds for axis 0 with size %lld", (long long)ordinals[i],
                      (long long)ix->size);
            return TAV_ERR_RANGE;
        }
    return TAV_OK;
}

// The error of a per-query subset search from device memory that its status word `st` (non-zero) refused, with its
// message; `size` is the index's row count when the search was issued.
static int subsets_status_error(int st, int64_t size) {
    if (st & kSubsetBadOffsets) {
        set_error("per-query subsets: offsets must be n_queries + 1 values from 0 to n_ordinals, never decreasing");
        return TAV_ERR_INVALID;
    }
    set_error("per-query subsets: an ordinal is out of bounds for axis 0 with size %lld", (long long)size);
    return TAV_ERR_RANGE;
}

static void destroy_history(tav_index* ix) {
    if (!ix->hist) return;
    for (int h = 0; h < kHistory; ++h) {
        for (auto& ev : ix->hist[h].total)
            if (ev) cudaEventDestroy(ev);
        for (auto& pr : ix->hist[h].ev)
            for (auto& ev : pr)
                if (ev) cudaEventDestroy(ev);
    }
    delete[] ix->hist;
    ix->hist = nullptr;
}

// Rows [first, first + n) of the index <- n rows of src_dtype from host or device memory, converted to the
// storage dtype as appends convert them (RNE, TAV_NORMALIZE); queued on s, which the caller has joined.
static int store_rows(tav_index* ix, int64_t first, const void* rows, int64_t n, int src_dtype, int src_on_device,
                      cudaStream_t s) {
    const size_t dst_row = static_cast<size_t>(ix->dim) * dtype_size(ix->dtype);
    const size_t src_row = static_cast<size_t>(ix->dim) * dtype_size(src_dtype);
    char* dst = static_cast<char*>(ix->rows) + static_cast<size_t>(first) * dst_row;
    const bool plain = (src_dtype == ix->dtype) && !(ix->flags & TAV_NORMALIZE);
    const int norm = (ix->flags & TAV_NORMALIZE) ? 1 : 0;
    if (src_on_device) {
        if (plain)
            TAV_CUDA(cudaMemcpyAsync(dst, rows, static_cast<size_t>(n) * src_row, cudaMemcpyDeviceToDevice, s));
        else
            TAV_CUDA(launch_convert(rows, src_dtype, dst, ix->dtype, n, ix->dim, norm, s));
    } else {
        // Host source (bulk load at open, storage/sqlite/messageindex.py:33-45; incremental appends):
        // through a pinned double buffer, so that the H2D copies are truly asynchronous and the host
        // memcpy of chunk i+1 overlaps the DMA (+ conversion kernel) of chunk i.
        const int64_t chunk_rows = std::max<int64_t>(1, static_cast<int64_t>(kAppendStageBytes / src_row));
        const size_t stage_bytes = static_cast<size_t>(std::min(n, chunk_rows)) * src_row;
        if (!plain) TAV_CUDA(ix->staging.ensure(2 * stage_bytes));
        int b = 0;
        for (int64_t done = 0; done < n; done += chunk_rows, b ^= 1) {
            const int64_t m = std::min(chunk_rows, n - done);
            const size_t bytes = static_cast<size_t>(m) * src_row;
            if (ix->append_busy[b]) {  // also across calls: the previous append may still be queued on its stream
                TAV_CUDA(cudaEventSynchronize(ix->ev_append[b]));
                ix->append_busy[b] = false;
            }
            TAV_CUDA(ix->pin_append[b].ensure(stage_bytes));
            memcpy(ix->pin_append[b].p, static_cast<const char*>(rows) + done * src_row, bytes);
            if (plain) {
                TAV_CUDA(cudaMemcpyAsync(dst + done * dst_row, ix->pin_append[b].p, bytes, cudaMemcpyHostToDevice, s));
            } else {
                char* stage = static_cast<char*>(ix->staging.p) + static_cast<size_t>(b) * stage_bytes;
                TAV_CUDA(cudaMemcpyAsync(stage, ix->pin_append[b].p, bytes, cudaMemcpyHostToDevice, s));
                TAV_CUDA(launch_convert(stage, src_dtype, dst + done * dst_row, ix->dtype, m, ix->dim, norm, s));
            }
            TAV_CUDA(cudaEventRecord(ix->ev_append[b], s));
            ix->append_busy[b] = true;
        }
        // the caller's buffer was fully consumed by the memcpys above; the pinned buffers are
        // re-acquired through their events, so no synchronisation is needed here
    }
    return TAV_OK;
}

extern "C" {

int tav_abi_version(void) { return TAV_ABI_VERSION; }

const char* tav_last_error(void) { return g_error; }

int tav_device_count(int* out_count) {
    if (!out_count) return TAV_ERR_INVALID;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) {
        cudaGetLastError();
        n = 0;
    }
    *out_count = n;
    return TAV_OK;
}

int tav_create(int device, int dim, int store_dtype, int index_flags, int64_t reserve_rows,
               tav_index** out) {
    if (!out || dim < 0 || !dtype_ok(store_dtype) || reserve_rows < 0) {
        set_error("tav_create: invalid argument");
        return TAV_ERR_INVALID;
    }
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        cudaGetLastError();
        set_error("tav_create: no CUDA device available (%s); libtavec has no CPU fallback",
                  e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
        return TAV_ERR_CUDA;
    }
    if (device < 0 || device >= n) {
        set_error("tav_create: device %d out of range (have %d)", device, n);
        return TAV_ERR_INVALID;
    }
    TAV_CUDA(cudaSetDevice(device));
    tav_index* ix = new (std::nothrow) tav_index();
    if (!ix) return TAV_ERR_OOM;
    ix->device = device;
    ix->dim = dim;
    ix->dtype = store_dtype;
    ix->flags = index_flags;
    cudaError_t ce = cudaEventCreateWithFlags(&ix->ev_pin_in, cudaEventDisableTiming);
    if (ce == cudaSuccess) ce = cudaEventCreateWithFlags(&ix->ev_last, cudaEventDisableTiming);
    for (int i = 0; ce == cudaSuccess && i < 2; ++i)
        ce = cudaEventCreateWithFlags(&ix->ev_append[i], cudaEventDisableTiming);
    if (ce != cudaSuccess) {
        set_error("tav_create: event creation failed: %s", cudaGetErrorString(ce));
        tav_destroy(ix);
        return TAV_ERR_CUDA;
    }
    *out = ix;
    if (reserve_rows > 0 && dim > 0) {
        int rc = tav_reserve(ix, reserve_rows);
        if (rc != TAV_OK) {
            tav_destroy(ix);
            *out = nullptr;
            return rc;
        }
    }
    return TAV_OK;
}

int tav_destroy(tav_index* ix) {
    if (!ix) return TAV_OK;
    cudaSetDevice(ix->device);
    cudaDeviceSynchronize();  // searches may still be in flight on the caller's streams
    if (!ix->adopted) rows_free(ix->rows, ix->rows_bytes);
    rows_free(ix->staged, ix->staged_bytes);
    if (ix->ev_last) cudaEventDestroy(ix->ev_last);
    if (ix->ev_pin_in) cudaEventDestroy(ix->ev_pin_in);
    for (auto& ev : ix->ev_append)
        if (ev) cudaEventDestroy(ev);
    destroy_history(ix);
    delete ix;  // (its buffers free themselves)
    return TAV_OK;
}

int tav_clear(tav_index* ix) {
    if (!ix) return TAV_ERR_INVALID;
    std::lock_guard<std::mutex> lock(ix->mu);
    // queued searches read the rows (or the adopted memory) that later appends overwrite
    if (int rc = set_device(ix)) return rc;
    if (int rc = wait_queued(ix)) return rc;
    if (ix->adopted) {
        ix->rows = nullptr;
        ix->adopted = false;
        ix->capacity = 0;
    }
    ix->size = 0;
    // (the "a corpus value left the fp16 range" flag is reset where the planes are rebuilt from row 0)
    ix->split_rows = 0;
    ix->row_mask_rows = 0;
    ix->qmask_n = 0;
    ix->group_rows = 0;
    return TAV_OK;
}

// the caller has joined `s` (or waited for the earlier calls' work): the copy reads complete rows
static int reserve_locked(tav_index* ix, int64_t rows, cudaStream_t s) {
    if (ix->adopted) {
        set_error("tav_reserve: index uses adopted device memory");
        return TAV_ERR_STATE;
    }
    if (rows <= ix->capacity) return TAV_OK;
    if (ix->dim <= 0) {
        set_error("tav_reserve: embedding size not known yet");
        return TAV_ERR_STATE;
    }
    if (int rc = set_device(ix)) return rc;
    const size_t row_bytes = static_cast<size_t>(ix->dim) * dtype_size(ix->dtype);
    void* fresh = nullptr;
    const size_t fresh_bytes = std::max<size_t>(static_cast<size_t>(rows) * row_bytes, 256);
    TAV_CUDA(rows_malloc(&fresh, fresh_bytes));
    if (ix->size > 0) {
        cudaError_t e = cudaMemcpyAsync(fresh, ix->rows, static_cast<size_t>(ix->size) * row_bytes,
                                        cudaMemcpyDeviceToDevice, s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (e != cudaSuccess) {
            rows_free(fresh, fresh_bytes);
            set_error("tav_reserve: copy failed: %s", cudaGetErrorString(e));
            return TAV_ERR_CUDA;
        }
    }
    if (ix->rows) {
        cudaDeviceSynchronize();
        rows_free(ix->rows, ix->rows_bytes);
    }
    ix->rows = fresh;
    ix->rows_bytes = fresh_bytes;
    ix->capacity = rows;
    return TAV_OK;
}

int tav_reserve(tav_index* ix, int64_t rows) {
    if (!ix || rows < 0) return TAV_ERR_INVALID;
    std::lock_guard<std::mutex> lock(ix->mu);
    if (rows > ix->capacity && !ix->adopted) {  // the copy must see every queued append
        if (int rc = set_device(ix)) return rc;
        if (int rc = wait_queued(ix)) return rc;
    }
    return reserve_locked(ix, rows, nullptr);
}

int tav_append(tav_index* ix, const void* rows, int64_t n, int dim, int src_dtype,
               int src_on_device, void* stream) {
    if (!ix || n < 0 || dim <= 0 || !dtype_ok(src_dtype) || (n > 0 && !rows)) {
        set_error("tav_append: invalid argument");
        return TAV_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lock(ix->mu);
    if (ix->adopted) {
        set_error("tav_append: index uses adopted device memory");
        return TAV_ERR_STATE;
    }
    if (ix->dim == 0) ix->dim = dim;  // first append fixes the width (vectorbase.py:119-121)
    if (dim != ix->dim) {
        set_error("Embedding size mismatch: expected %d, got %d", ix->dim, dim);
        return TAV_ERR_INVALID;
    }
    if (n == 0) return TAV_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (int rc = enter_stream(ix, s)) return rc;
    if (ix->size + n > ix->capacity) {
        int64_t want = std::max<int64_t>(ix->size + n, ix->capacity * 2);
        want = std::max<int64_t>(want, 1024);
        TAV_CUDA(cudaStreamSynchronize(s));
        mark_done(ix);
        if (int rc = reserve_locked(ix, want, s)) return rc;
    }
    if (int rc = store_rows(ix, ix->size, rows, n, src_dtype, src_on_device, s)) return rc;
    ix->size += n;
    return mark_queued(ix, s);
}

int tav_adopt_device(tav_index* ix, void* device_rows, int64_t n, int dim) {
    if (!ix || n < 0 || dim <= 0 || (n > 0 && !device_rows)) return TAV_ERR_INVALID;
    std::lock_guard<std::mutex> lock(ix->mu);
    if (ix->flags & TAV_NORMALIZE) {
        set_error("tav_adopt_device: not available on a TAV_NORMALIZE index (rows are used as is)");
        return TAV_ERR_STATE;
    }
    if (ix->dim != 0 && ix->dim != dim) {
        set_error("Embedding size mismatch: expected %d, got %d", ix->dim, dim);
        return TAV_ERR_INVALID;
    }
    if (reinterpret_cast<uintptr_t>(device_rows) % 16 != 0) {
        set_error("tav_adopt_device: pointer must be 16-byte aligned");
        return TAV_ERR_INVALID;
    }
    if (int rc = set_device(ix)) return rc;
    if (int rc = wait_queued(ix)) return rc;  // queued searches read the rows replaced here
    if (ix->rows && !ix->adopted) {
        cudaDeviceSynchronize();
        rows_free(ix->rows, ix->rows_bytes);
    }
    ix->rows_bytes = 0;
    ix->dim = dim;
    ix->rows = device_rows;
    ix->split_rows = 0;  // (the planes' overflow flag is reset where they are rebuilt from row 0)
    ix->row_mask_rows = 0;
    ix->qmask_n = 0;
    ix->group_rows = 0;
    ix->adopted = true;
    ix->size = n;
    ix->capacity = n;
    return TAV_OK;
}

int64_t tav_size(const tav_index* ix) { return ix ? ix->size : 0; }
int tav_dim(const tav_index* ix) { return ix ? ix->dim : 0; }
int tav_store_dtype(const tav_index* ix) { return ix ? ix->dtype : -1; }
int tav_device(const tav_index* ix) { return ix ? ix->device : -1; }

int tav_read_rows(tav_index* ix, int64_t first, int64_t n, float* out_host, void* stream) {
    if (!ix || n < 0 || (n > 0 && !out_host)) return TAV_ERR_INVALID;
    std::lock_guard<std::mutex> lock(ix->mu);
    if (first < 0 || first + n > ix->size) {
        set_error("tav_read_rows: rows [%lld, %lld) out of range (size %lld)", (long long)first,
                  (long long)(first + n), (long long)ix->size);
        return TAV_ERR_RANGE;
    }
    if (n == 0) return TAV_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (int rc = enter_stream(ix, s)) return rc;
    const size_t row = static_cast<size_t>(ix->dim) * dtype_size(ix->dtype);
    const char* src = static_cast<const char*>(ix->rows) + static_cast<size_t>(first) * row;
    if (ix->dtype == TAV_F32) {
        TAV_CUDA(cudaMemcpyAsync(out_host, src, static_cast<size_t>(n) * row, cudaMemcpyDeviceToHost, s));
    } else {
        const size_t bytes = static_cast<size_t>(n) * ix->dim * sizeof(float);
        TAV_CUDA(ix->staging.ensure(bytes));
        TAV_CUDA(launch_convert(src, ix->dtype, ix->staging.p, TAV_F32, n, ix->dim, 0, s));
        TAV_CUDA(cudaMemcpyAsync(out_host, ix->staging.p, bytes, cudaMemcpyDeviceToHost, s));
    }
    TAV_CUDA(cudaStreamSynchronize(s));
    mark_done(ix);
    return TAV_OK;
}

int tav_set_row_mask(tav_index* ix, const uint32_t* bits, int64_t n_rows, int on_device, void* stream) {
    if (!ix || n_rows < 0 || (n_rows > 0 && !bits)) return TAV_ERR_INVALID;
    std::lock_guard<std::mutex> lock(ix->mu);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (int rc = enter_stream(ix, s)) return rc;  // queued searches read the old mask
    // an outstanding search may still need the old mask for its exact redo
    if (int rc = finish_pending(ix, s, nullptr)) return rc;
    if (n_rows == 0) {
        ix->row_mask_rows = 0;
        return TAV_OK;
    }
    if (n_rows != ix->size) {
        set_error("tav_set_row_mask: %lld bits for an index of %lld rows", (long long)n_rows, (long long)ix->size);
        return TAV_ERR_INVALID;
    }
    const size_t words = static_cast<size_t>(mask_words(n_rows));
    const size_t src_words = static_cast<size_t>((n_rows + 31) / 32);
    TAV_CUDA(ix->row_mask.ensure(words * sizeof(uint32_t)));
    TAV_CUDA(cudaMemsetAsync(ix->row_mask.p, 0, words * sizeof(uint32_t), s));
    TAV_CUDA(cudaMemcpyAsync(ix->row_mask.p, bits, src_words * sizeof(uint32_t),
                             on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, s));
    ix->row_mask_rows = n_rows;
    if (on_device) return mark_queued(ix, s);
    TAV_CUDA(cudaStreamSynchronize(s));
    mark_done(ix);
    return TAV_OK;
}

int tav_set_query_masks(tav_index* ix, const uint32_t* bits, int n_queries, int64_t n_rows, int64_t stride_words,
                        int on_device, void* stream) {
    if (!ix || n_queries < 0 || n_rows < 0 || (n_queries > 0 && !bits)) return TAV_ERR_INVALID;
    std::lock_guard<std::mutex> lock(ix->mu);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (int rc = enter_stream(ix, s)) return rc;  // queued searches read the old masks
    // an outstanding search may still need the old masks for its exact redo
    if (int rc = finish_pending(ix, s, nullptr)) return rc;
    if (n_queries == 0) {
        ix->qmask_n = 0;
        return TAV_OK;
    }
    const int64_t src_words = (n_rows + 31) / 32;
    if (n_rows != ix->size || n_rows == 0) {
        set_error("tav_set_query_masks: %lld bits per mask for an index of %lld rows", (long long)n_rows,
                  (long long)ix->size);
        return TAV_ERR_INVALID;
    }
    if (stride_words < src_words) {
        set_error("tav_set_query_masks: stride of %lld words is below the %lld words of a mask", (long long)stride_words,
                  (long long)src_words);
        return TAV_ERR_INVALID;
    }
    const int64_t words = mask_words(n_rows);
    const size_t bytes = static_cast<size_t>(n_queries) * words * sizeof(uint32_t);
    ix->qmask_n = 0;
    cudaError_t e = ix->qmask_cap >= 0 && bytes > static_cast<size_t>(ix->qmask_cap) ? cudaErrorMemoryAllocation
                                                                                      : ix->qmask.ensure(bytes);
    if (e == cudaSuccess) e = ix->qmask_pop.ensure(static_cast<size_t>(n_queries) * sizeof(uint32_t));
    if (e != cudaSuccess) {
        cudaGetLastError();  // no sticky error: the index stays usable
        ix->qmask.release();
        ix->qmask_pop.release();
        set_error("tav_set_query_masks: cannot allocate %zu bytes for %d masks: %s", bytes, n_queries, cudaGetErrorString(e));
        return e == cudaErrorMemoryAllocation ? TAV_ERR_OOM : TAV_ERR_CUDA;
    }
    TAV_CUDA(cudaMemsetAsync(ix->qmask.p, 0, bytes, s));
    TAV_CUDA(cudaMemcpy2DAsync(ix->qmask.p, static_cast<size_t>(words) * sizeof(uint32_t), bits,
                               static_cast<size_t>(stride_words) * sizeof(uint32_t),
                               static_cast<size_t>(src_words) * sizeof(uint32_t), static_cast<size_t>(n_queries),
                               on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, s));
    // (bits beyond n_rows are never tested: the kernels test rows < n_rows only, and the popcount ignores them)
    TAV_CUDA(launch_mask_popcount(static_cast<const uint32_t*>(ix->qmask.p), n_queries, n_rows, words,
                                  static_cast<uint32_t*>(ix->qmask_pop.p), s));
    ix->qmask_n = n_queries;
    ix->qmask_rows = n_rows;
    ix->qmask_stride = words;
    if (on_device) return mark_queued(ix, s);
    TAV_CUDA(cudaStreamSynchronize(s));
    mark_done(ix);
    return TAV_OK;
}

}  // extern "C"

static inline cudaError_t ev_record(cudaEvent_t& ev, cudaStream_t s) {
    if (!ev) {
        cudaError_t e = cudaEventCreate(&ev);
        if (e != cudaSuccess) return e;
    }
    return cudaEventRecord(ev, s);
}

// the timing record of a search that starts now: the next history entry when timing is on, else ix->untimed
static TimedSearch* begin_search(tav_index* ix, int path) {
    ix->last_first_slot = -1;
    ix->last_n_slots = 0;
    ix->last_split = false;
    TimedSearch* ts = cur_timed(ix);
    if (!ts) ts = &ix->untimed;
    ts->used = 0;
    ts->launches = 0;
    ts->path = path;
    ts->valid = false;
    return ts;
}

// the search's work is queued: its closing event, and the record counts
static int end_search(tav_index* ix, TimedSearch* ts, cudaStream_t s) {
    if (ts != &ix->untimed) {
        TAV_CUDA(ev_record(ts->total[1], s));
        ++ix->search_seq;
    }
    ts->valid = true;
    return TAV_OK;
}

// One kernel launch of a search, with an event pair of `kind` around it when the search is timed and a pair is
// free; light timing (tav_set_timing(2)) times only the dominant kernels (kind 0).  ts may be nullptr.
template <class Launch>
static cudaError_t timed_launch(const tav_index* ix, TimedSearch* ts, bool timing, int kind, cudaStream_t s,
                                Launch&& launch) {
    const bool timed = timing && ts && ts->used < kMaxTimedKernels && (kind == 0 || !ix->timing_light);
    cudaError_t e;
    if (timed && (e = ev_record(ts->ev[ts->used][0], s)) != cudaSuccess) return e;
    if ((e = launch()) != cudaSuccess || !timed) return e;
    ts->kind[ts->used] = kind;
    return ev_record(ts->ev[ts->used++][1], s);
}

// the tensor-core launchers record into existing events: every pair of a timed search is created first
static int create_events(TimedSearch* ts) {
    for (auto& pr : ts->ev)
        for (auto& ev : pr)
            if (!ev) TAV_CUDA(cudaEventCreate(&ev));
    return TAV_OK;
}

// the corpus fields of a row-scan launch
static ScanArgs scan_args(const tav_index* ix) {
    ScanArgs a{};
    a.corpus = ix->rows;
    a.dtype = ix->dtype;
    a.n_corpus = ix->size;
    a.dim = ix->dim;
    return a;
}

// the corpus fields of a tensor-core launch: the rows, or (split) the float32 index's two fp16 planes
static MmaArgs mma_args(const tav_index* ix, bool split) {
    MmaArgs m{};
    m.device = ix->device;
    m.corpus = split ? ix->split_hi.p : ix->rows;
    m.corpus_lo = split ? ix->split_lo.p : nullptr;
    m.split = split ? 1 : 0;
    m.dtype = ix->dtype;
    m.n_corpus = ix->size;
    m.dim = ix->dim;
    return m;
}

// the tensor-core search workspace, at least `bytes`: earlier searches may still use the old one, and the
// sampler's unit counters (its first 64 KB) must read zero
static int ensure_mma_ws(tav_index* ix, size_t bytes, cudaStream_t s) {
    if (bytes <= ix->mma_ws.bytes) return TAV_OK;
    TAV_CUDA(cudaStreamSynchronize(s));
    TAV_CUDA(ix->mma_ws.ensure(bytes));
    TAV_CUDA(cudaMemsetAsync(ix->mma_ws.p, 0, std::min<size_t>(ix->mma_ws.bytes, 65536), s));
    return TAV_OK;
}

// Host outputs of a top-k search of n_queries x k, packed [items | scores | counts | done word] in one buffer
// so that a single D2H copy (into pinned staging) brings them back.
struct ResultPack {
    size_t nk, n;  // hits, counts
    size_t off_scores, off_counts, off_done;
    ResultPack(int n_queries, int k)
        : nk(static_cast<size_t>(n_queries) * k), n(static_cast<size_t>(n_queries)), off_scores(nk * sizeof(int64_t)),
          off_counts(off_scores + ((nk * sizeof(float) + 7) & ~size_t(7))),
          off_done(off_counts + ((n * sizeof(int32_t) + 7) & ~size_t(7))) {}
    size_t bytes() const { return off_done + 8; }
    size_t counts_end() const { return off_counts + n * sizeof(int32_t); }  // the pack without the done word
    // the three arrays in a pack at `base`
    void place(void* base, int64_t** items, float** scores, int32_t** counts) const {
        char* b = static_cast<char*>(base);
        *items = reinterpret_cast<int64_t*>(b);
        *scores = reinterpret_cast<float*>(b + off_scores);
        *counts = reinterpret_cast<int32_t*>(b + off_counts);
    }
    // a pack in host memory -> the caller's arrays
    void unpack(const void* h, int64_t* items, float* scores, int32_t* counts) const {
        const char* b = static_cast<const char*>(h);
        memcpy(items, b, nk * sizeof(int64_t));
        memcpy(scores, b + off_scores, nk * sizeof(float));
        memcpy(counts, b + off_counts, n * sizeof(int32_t));
    }
};

// a pack in device memory -> the caller's host arrays, each array copied on its own; synchronises s
static int copy_pack_out(const ResultPack& p, const void* d, int64_t* items, float* scores, int32_t* counts,
                         cudaStream_t s) {
    const char* b = static_cast<const char*>(d);
    TAV_CUDA(cudaMemcpyAsync(items, b, p.nk * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    TAV_CUDA(cudaMemcpyAsync(scores, b + p.off_scores, p.nk * sizeof(float), cudaMemcpyDeviceToHost, s));
    TAV_CUDA(cudaMemcpyAsync(counts, b + p.off_counts, p.n * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    TAV_CUDA(cudaStreamSynchronize(s));
    return TAV_OK;
}

// CSR offsets of a threshold search -> the caller (host or device); the sort after the last synchronisation
// may still run
static int deliver_offsets(tav_index* ix, const std::vector<int64_t>& offsets, int64_t* out, bool o_dev, cudaStream_t s) {
    const size_t bytes = offsets.size() * sizeof(int64_t);
    if (o_dev) {  // from pageable memory: consumed when the call returns
        TAV_CUDA(cudaMemcpyAsync(out, offsets.data(), bytes, cudaMemcpyHostToDevice, s));
    } else {
        memcpy(out, offsets.data(), bytes);
    }
    return mark_queued(ix, s);
}

// workspace of the row-scan kernels: [8] u64 bounds | [8] u32 counters | [1] u32 fused ticket, zeroed once
static int ensure_scan_counters(tav_index* ix, cudaStream_t s) {
    const size_t need = 8 * (sizeof(uint32_t) + sizeof(uint64_t)) + 64;
    if (ix->cand_count.bytes < need) {
        TAV_CUDA(ix->cand_count.ensure(need));
        TAV_CUDA(cudaMemsetAsync(ix->cand_count.p, 0, ix->cand_count.bytes, s));
    }
    return TAV_OK;
}

// Row-scan search of nq_total queries (device float32), any k: passes of <= kPassK hits.
static int scan_search(tav_index* ix, TimedSearch* ts, bool timing, const float* d_queries, int nq_total, int k, float floor_score,
                       const int64_t* d_subset, int64_t n_scan, int64_t item_offset, int64_t* d_items,
                       float* d_scores, int32_t* d_counts, const uint32_t* d_mask, int ties_low, cudaStream_t s,
                       bool allow_fuse = true, int positions = 0, QueryMasks qm = QueryMasks{}) {
    const int pass_k = std::min(k, kPassK);
    int qb = scan_max_queries(ix->dim, pass_k);
    if (qb < 1) {
        set_error("tav_search: embedding size %d too large for the row-scan kernel", ix->dim);
        return TAV_ERR_INVALID;
    }
    qb = std::min(qb, nq_total);
    // round qb down to a power of two (kernel instantiations 1/2/4/8)
    while (qb & (qb - 1)) qb &= qb - 1;
    int grid = scan_grid(ix->device, ix->dtype, ix->dim, qb, pass_k, n_scan);
    const int n_pass = (k + pass_k - 1) / pass_k;
    // L2-sized scans with a small k end in the scan kernel itself: its last CTA merges the survivors of all
    // CTAs and writes the hits (no select launch) — the device-query twin of the single-launch latency form
    const bool fuse = allow_fuse && n_pass == 1 && pass_k <= 64 &&
                      static_cast<size_t>(n_scan) * ix->dim * dtype_size(ix->dtype) <= kFusedScanMaxBytes &&
                      static_cast<int64_t>(std::min(grid, 132)) * std::max(pass_k, 32) <= kFusedSelectMax;
    if (fuse) grid = std::min(grid, kFusedSelectMax / std::max(pass_k, 32));
    const int cand_stride = grid * (fuse ? std::max(pass_k, 32) : pass_k);
    TAV_CUDA(ix->cand_keys.ensure(static_cast<size_t>(qb) * cand_stride * sizeof(uint64_t)));
    if (int rc = ensure_scan_counters(ix, s)) return rc;
    uint64_t* d_bound = static_cast<uint64_t*>(ix->cand_count.p);
    uint32_t* d_count = reinterpret_cast<uint32_t*>(d_bound + 8);

    for (int q0 = 0; q0 < nq_total; q0 += qb) {
        const int nq = std::min(qb, nq_total - q0);
        for (int pass = 0; pass < n_pass; ++pass) {
            const int kk = std::min(pass_k, k - pass * pass_k);
            ScanArgs a = scan_args(ix);
            a.subset = d_subset;
            a.n_scan = n_scan;
            a.queries = d_queries + static_cast<size_t>(q0) * ix->dim;
            a.nq = nq;
            a.floor_score = floor_score;
            a.bound = pass > 0 ? d_bound : nullptr;
            a.k = kk;
            a.cand_keys = static_cast<uint64_t*>(ix->cand_keys.p);
            a.cand_stride = cand_stride;
            a.cand_count = d_count;
            a.grid = grid;
            a.row_mask = d_mask;
            if (qm.bits && nq == 1 && !qm.map) a.row_mask = qm.bits + static_cast<int64_t>(q0) * qm.stride;  // the row-mask form
            else if (qm.bits) a.qmask = qmask_from(qm, q0);
            a.ties_low = ties_low;
            a.items_as_positions = positions;
            if (fuse) {
                a.fused = 1;
                a.fused_ticket = d_count + 8;
                a.item_offset = item_offset;
                a.out_items = d_items + static_cast<size_t>(q0) * k;
                a.out_scores = d_scores + static_cast<size_t>(q0) * k;
                a.out_counts = d_counts + q0;
            }
            TAV_CUDA(timed_launch(ix, ts, timing, 0, s, [&] { return launch_scan(a, s); }));
            if (fuse) {
                if (ts) ts->launches += 1;
                continue;
            }
            SelectArgs sel{};
            sel.cand_keys = a.cand_keys;
            sel.cand_stride = cand_stride;
            sel.cand_count = d_count;
            sel.cand_count_reset = d_count;
            sel.nq = nq;
            sel.k = kk;
            sel.out_stride = k;
            sel.out_offset = pass * pass_k;
            sel.subset = positions ? nullptr : d_subset;  // items = the position itself
            sel.item_offset = item_offset;
            sel.out_items = d_items + static_cast<size_t>(q0) * k;
            sel.out_scores = d_scores + static_cast<size_t>(q0) * k;
            sel.out_counts = d_counts + q0;
            sel.bound_out = n_pass > 1 ? d_bound : nullptr;
            sel.accumulate = pass > 0;
            sel.ties_low = ties_low;
            TAV_CUDA(launch_select(sel, s));
            if (ts) ts->launches += 2;
        }
    }
    return TAV_OK;
}

// float32 index -> fp16 hi/lo planes covering rows [0, size); returns TAV_ERR_OOM when they do not fit
static int ensure_split_planes(tav_index* ix, TimedSearch* ts, cudaStream_t s) {
    const size_t plane_row = static_cast<size_t>(ix->dim) * 2;
    if (ix->split_flag.bytes == 0) {
        TAV_CUDA(ix->split_flag.ensure(2 * sizeof(int)));
        TAV_CUDA(cudaMemsetAsync(ix->split_flag.p, 0, 2 * sizeof(int), s));
    }
    if (ix->size > ix->split_cap) {
        const int64_t cap = std::max<int64_t>(ix->size, ix->capacity);
        ix->split_hi.release();
        ix->split_lo.release();
        ix->split_cap = 0;
        ix->split_rows = 0;
        cudaError_t e1 = ix->split_hi.ensure(static_cast<size_t>(cap) * plane_row);
        cudaError_t e2 = e1 == cudaSuccess ? ix->split_lo.ensure(static_cast<size_t>(cap) * plane_row) : e1;
        if (e2 != cudaSuccess) {
            cudaGetLastError();
            ix->split_hi.release();
            ix->split_lo.release();
            set_error("not enough device memory for the fp16 planes of the float32 index");
            return TAV_ERR_OOM;
        }
        ix->split_cap = cap;
    }
    if (ix->split_recheck) {  // the flag may stand for rows that were removed or overwritten since
        ix->split_recheck = false;
        if (ix->split_rows > 0) {
            int flag = 0;
            TAV_CUDA(cudaMemcpyAsync(&flag, ix->split_flag.p, sizeof(int), cudaMemcpyDeviceToHost, s));
            TAV_CUDA(cudaStreamSynchronize(s));
            if (flag) ix->split_rows = 0;  // rebuilt from row 0, which resets it
        }
    }
    if (ix->split_rows < ix->size) {
        if (ix->split_rows == 0) TAV_CUDA(cudaMemsetAsync(ix->split_flag.p, 0, sizeof(int), s));  // planes rebuilt from row 0
        const int64_t first = ix->split_rows, n = ix->size - first;
        TAV_CUDA(launch_split_rows(static_cast<const float*>(ix->rows) + first * ix->dim,
                                   static_cast<char*>(ix->split_hi.p) + static_cast<size_t>(first) * plane_row,
                                   static_cast<char*>(ix->split_lo.p) + static_cast<size_t>(first) * plane_row, n,
                                   ix->dim, static_cast<int*>(ix->split_flag.p), s));
        ix->split_rows = ix->size;
        if (ts) ts->launches += 1;
    }
    return TAV_OK;
}

static int range_into_redo(tav_index* ix, const Pending& p, bool redo_all, int* n_redone, cudaStream_t s);

static inline int32_t* retry_totals(tav_index* ix, int slot) { return static_cast<int32_t*>(ix->retry.p) + 2 * slot; }
static inline int32_t* retry_flags(tav_index* ix, int slot) {
    return static_cast<int32_t*>(ix->retry.p) + 2 * kMaxPending + static_cast<size_t>(slot) * ix->retry_cap;
}

// Synchronising tail of the tensor-core searches: look at the "redo exactly" bookkeeping of every
// outstanding search and redo flagged queries with the row scan, into that search's own outputs.
static int finish_pending(tav_index* ix, cudaStream_t s, int* redone) {
    if (redone) *redone = 0;
    if (ix->pending.empty()) return TAV_OK;
    if (int rc = join_stream(ix, s)) return rc;  // the searches may have been issued on other streams
    int32_t totals[2 * kMaxPending];
    int corpus_overflow = 0;
    bool any_split = false, any_subsets = false;
    for (const Pending& p : ix->pending) {
        any_split |= p.split;
        any_subsets |= p.subsets_status != nullptr;
    }
    if (any_split)
        TAV_CUDA(cudaMemcpyAsync(&corpus_overflow, ix->split_flag.p, sizeof(int), cudaMemcpyDeviceToHost, s));
    int status[kMaxPending];
    if (any_subsets)
        TAV_CUDA(cudaMemcpyAsync(status, ix->subsets_status.p, sizeof(status), cudaMemcpyDeviceToHost, s));
    TAV_CUDA(cudaStreamSynchronize(s));
    memcpy(totals, ix->retry_host.p, sizeof(totals));  // written by the kernels through the mapping; current after the sync
    std::vector<Pending> todo;
    todo.swap(ix->pending);
    ix->next_slot = 0;
    bool dirty = false;
    int n_redone = 0;
    std::vector<int32_t> host;
    for (const Pending& p : todo) {
        if (p.subsets_status && TAV_SUBSETS_DEVICE_MUTANT != 2) {  // refused on the device: its outputs say no hits
            const int st = status[p.slot];
            if (st && ix->deferred_rc == TAV_OK) {
                ix->deferred_rc = subsets_status_error(st, p.n_scan);
                ix->deferred_msg = tav_last_error();
            }
        }
        const int flagged = totals[2 * p.slot], q_overflow = totals[2 * p.slot + 1];
        const bool redo_all = p.split && (corpus_overflow != 0 || q_overflow != 0);
        dirty |= flagged != 0 || q_overflow != 0;
        if (flagged == 0 && !redo_all) continue;
        if (p.k == 0) {  // a threshold search into the caller's buffers
            if (int rc = range_into_redo(ix, p, redo_all, &n_redone, s)) return rc;
            continue;
        }
        host.assign(static_cast<size_t>(p.nq), 1);
        if (!redo_all) {
            TAV_CUDA(cudaMemcpyAsync(host.data(), retry_flags(ix, p.slot), static_cast<size_t>(p.nq) * sizeof(int32_t),
                                     cudaMemcpyDeviceToHost, s));
            TAV_CUDA(cudaStreamSynchronize(s));
        }
        for (int q = 0; q < p.nq; ++q) {
            if (!host[q]) continue;
            ++n_redone;
            // the query's own mask (the row mask: stride 0), as the row-mask form of the scan
            const uint32_t* mask = p.mask ? p.mask + static_cast<int64_t>(TAV_QUERY_MASK_MUTANT == 2 ? 0 : q) * p.mask_stride
                                          : nullptr;
            int rc = scan_search(ix, nullptr, false, p.queries + static_cast<size_t>(q) * ix->dim, 1, p.k, p.floor, nullptr,
                                 ix->size, p.item_offset, p.items + static_cast<size_t>(q) * p.k,
                                 p.scores + static_cast<size_t>(q) * p.k, p.counts + q, mask, 0, s);
            if (rc != TAV_OK) return rc;
        }
    }
    if (dirty) TAV_CUDA(cudaMemsetAsync(ix->retry.p, 0, sizeof(totals), s));
    if (dirty || n_redone > 0) TAV_CUDA(cudaStreamSynchronize(s));
    if (dirty) memset(ix->retry_host.p, 0, sizeof(totals));
    mark_done(ix);
    // No queued work reads a held query region now, whatever stream a later search uses: the searches ended
    // at the first synchronisation above (s joined the stream of the last call first), their redo scans at the
    // last.  So the regions can be reused and the outgrown buffers freed.
    ix->held_used = 0;
    ix->held_retired.clear();
    if (redone) *redone = n_redone;
    return TAV_OK;
}

// The subset arguments of tav_search / tav_range_search (`fn`), checked before the index is looked at; a
// threshold search also refuses TAV_DEFER_RETRY.
static int check_subset_args(const char* fn, int flags, const int64_t* subset, int64_t subset_len, bool threshold) {
    if ((subset && subset_len < 0) || (!subset && subset_len != 0)) {
        set_error("%s: subset / subset_len mismatch", fn);
        return TAV_ERR_INVALID;
    }
    if (threshold && (flags & TAV_DEFER_RETRY)) {
        set_error("%s: TAV_DEFER_RETRY is not available for threshold searches", fn);
        return TAV_ERR_INVALID;
    }
    if ((flags & TAV_ITEMS_AS_POSITIONS) && !subset) {
        set_error("%s: TAV_ITEMS_AS_POSITIONS needs a subset", fn);
        return TAV_ERR_INVALID;
    }
    return TAV_OK;
}

// The filter of a search of n_queries (`fn` names the entry point in the messages), or the error:
// TAV_USE_ROW_MASK -> the row mask in *d_mask; TAV_USE_QUERY_MASKS -> the index's per-query masks in *qm, except
// that one query takes the row-mask form (its mask in *d_mask, *qm empty).
static int resolve_masks(tav_index* ix, const char* fn, int n_queries, int flags, bool has_subset,
                         const uint32_t** d_mask, QueryMasks* qm) {
    *d_mask = nullptr;
    *qm = QueryMasks{};
    if (flags & TAV_USE_QUERY_MASKS) {
        if (flags & TAV_USE_ROW_MASK) {
            set_error("%s: TAV_USE_QUERY_MASKS and TAV_USE_ROW_MASK cannot be combined", fn);
            return TAV_ERR_INVALID;
        }
        if (has_subset) {
            set_error("%s: per-query masks and a subset cannot be combined", fn);
            return TAV_ERR_INVALID;
        }
        if (ix->qmask_n == 0 || ix->qmask_rows != ix->size || ix->size == 0) {
            set_error("%s: TAV_USE_QUERY_MASKS without current per-query masks (tav_set_query_masks)", fn);
            return TAV_ERR_STATE;
        }
        if (n_queries != ix->qmask_n) {
            set_error("%s: %d queries for %d per-query masks", fn, n_queries, ix->qmask_n);
            return TAV_ERR_INVALID;
        }
        if (n_queries == 1) {
            *d_mask = static_cast<const uint32_t*>(ix->qmask.p);
            return TAV_OK;
        }
        qm->bits = static_cast<const uint32_t*>(ix->qmask.p);
        qm->stride = ix->qmask_stride;
        qm->pop = static_cast<const uint32_t*>(ix->qmask_pop.p);
    } else if (flags & TAV_USE_ROW_MASK) {
        if (ix->row_mask_rows != ix->size || ix->size == 0) {
            set_error("%s: TAV_USE_ROW_MASK without a current row mask (tav_set_row_mask)", fn);
            return TAV_ERR_STATE;
        }
        if (has_subset) {
            set_error("%s: a row mask and a subset cannot be combined", fn);
            return TAV_ERR_INVALID;
        }
        *d_mask = static_cast<const uint32_t*>(ix->row_mask.p);
    }
    return TAV_OK;
}

// ---- threshold search (tav_range_search; tav_search with k >= rows) ------------------------------------
constexpr int64_t kRangeDefaultPerQuery = 16384;  // collect region per query when the caller gives no hint

// an allocation of the threshold search: a failure leaves no sticky error behind and the index usable
static int range_alloc(DevBuf& b, size_t bytes, const char* what) {
    cudaError_t e = b.ensure(bytes);
    if (e == cudaSuccess) return TAV_OK;
    cudaGetLastError();
    set_error("threshold search: cannot allocate %s (%zu bytes): %s", what, bytes, cudaGetErrorString(e));
    return e == cudaErrorMemoryAllocation ? TAV_ERR_OOM : TAV_ERR_CUDA;
}

// host queries / subset -> device, shared by tav_search and the threshold search: subset ordinals through
// pinned staging, queries float32 (normalised when the index is TAV_NORMALIZE).  `o_dev`: the call returns
// without synchronising, so the pinned staging stays busy until the copies are done.  `held`: where normalised
// queries go instead of ix->queries (a deferred search's own region).
static int stage_inputs(tav_index* ix, TimedSearch* ts, bool timing, const float* queries, int n_queries, bool q_dev,
                        bool o_dev, const int64_t* subset, int64_t subset_len, const float** out_queries,
                        const int64_t** out_subset, cudaStream_t s, float* held = nullptr) {
    const int64_t* d_subset = nullptr;
    // subset ordinals -> device
    if (subset) {
        const size_t sub_bytes = static_cast<size_t>(subset_len) * sizeof(int64_t);
        TAV_CUDA(ix->subset.ensure(sub_bytes));
        const void* src = subset;
        if (sub_bytes <= kPinnedStageLimit) {
            TAV_CUDA(pin_in_acquire(ix, ((sub_bytes + 15) & ~size_t(15)) +
                                            static_cast<size_t>(n_queries) * ix->dim * sizeof(float)));
            memcpy(ix->pin_in.p, subset, sub_bytes);
            src = ix->pin_in.p;
        }
        TAV_CUDA(cudaMemcpyAsync(ix->subset.p, src, sub_bytes, cudaMemcpyHostToDevice, s));
        d_subset = static_cast<const int64_t*>(ix->subset.p);
    }

    if (timing) TAV_CUDA(ev_record(ts->total[0], s));

    // queries -> device float32 (normalised in place when the index is TAV_NORMALIZE)
    const float* d_queries = queries;
    const size_t q_bytes = static_cast<size_t>(n_queries) * ix->dim * sizeof(float);
    if (!q_dev || (ix->flags & TAV_NORMALIZE)) {
        if (!held) TAV_CUDA(ix->queries.ensure(q_bytes));
        float* dst = held ? held : static_cast<float*>(ix->queries.p);
        if (ix->flags & TAV_NORMALIZE) {
            const void* src = queries;
            if (!q_dev) {
                TAV_CUDA(ix->staging.ensure(q_bytes));
                TAV_CUDA(cudaMemcpyAsync(ix->staging.p, queries, q_bytes, cudaMemcpyHostToDevice, s));
                src = ix->staging.p;
            }
            TAV_CUDA(launch_convert(src, TAV_F32, dst, TAV_F32, n_queries, ix->dim, 1, s));
            ts->launches += 1;
        } else {
            const void* src = queries;
            cudaPointerAttributes qa{};
            const bool q_pinned = !o_dev &&  // (device outputs: the call returns before the copy ends, staging protects the caller's buffer)
                                  cudaPointerGetAttributes(&qa, queries) == cudaSuccess && qa.type == cudaMemoryTypeHost;
            if (!q_pinned) cudaGetLastError();
            if (q_bytes <= kPinnedStageLimit && !q_pinned) {
                // via pinned staging: a pageable source would make the copy synchronous (a caller that
                // already passes pinned memory is copied from directly)
                const size_t sub_bytes = subset ? static_cast<size_t>(subset_len) * sizeof(int64_t) : 0;
                const size_t sub_off = sub_bytes <= kPinnedStageLimit ? ((sub_bytes + 15) & ~size_t(15)) : 0;
                TAV_CUDA(pin_in_acquire(ix, sub_off + q_bytes));
                memcpy(static_cast<char*>(ix->pin_in.p) + sub_off, queries, q_bytes);
                src = static_cast<char*>(ix->pin_in.p) + sub_off;
            }
            TAV_CUDA(cudaMemcpyAsync(dst, src, q_bytes, cudaMemcpyHostToDevice, s));
        }
        d_queries = dst;
    }

    if (o_dev && (!q_dev || subset)) {  // no synchronisation at the end of this call
        TAV_CUDA(cudaEventRecord(ix->ev_pin_in, s));
        ix->pin_in_busy = true;
    }

    *out_queries = d_queries;
    *out_subset = d_subset;
    return TAV_OK;
}

// collect-mode row scans of nq queries (device, contiguous): query q's keys -> keys + q * stride, counts[q]
static int collect_scans(tav_index* ix, TimedSearch* ts, bool timing, const float* d_queries, int nq, float floor,
                         const int64_t* d_subset, int64_t n_scan, const uint32_t* d_mask, int ties_low,
                         uint64_t* keys, int64_t stride, uint32_t* counts, cudaStream_t s, QueryMasks qm = QueryMasks{}) {
    const int qb = scan_collect_max_queries(ix->dim);  // a smaller last block takes a smaller instantiation
    if (qb < 1) {
        set_error("threshold search: embedding size %d too large for the row-scan kernel", ix->dim);
        return TAV_ERR_INVALID;
    }
    const int grid = scan_collect_grid(ix->device, ix->dim, qb, n_scan);
    for (int q0 = 0; q0 < nq; q0 += qb) {
        ScanArgs a = scan_args(ix);
        a.subset = d_subset;
        a.n_scan = n_scan;
        a.queries = d_queries + static_cast<size_t>(q0) * ix->dim;
        a.nq = std::min(qb, nq - q0);
        a.floor_score = floor;
        a.cand_keys = keys + static_cast<size_t>(q0) * stride;
        a.collect_stride = stride;
        a.cand_count = counts + q0;
        a.grid = grid;
        a.row_mask = d_mask;
        if (qm.bits) a.qmask = qmask_from(qm, q0);
        a.ties_low = ties_low;
        TAV_CUDA(timed_launch(ix, ts, timing, 0, s, [&] { return launch_scan_collect(a, s); }));
        ts->launches += 1;
    }
    return TAV_OK;
}

// collect region per query: the caller's hint with headroom for queries above the average, at most every row
static int64_t range_per_query(int64_t expected_hits, int nq, int64_t n_scan) {
    int64_t per = kRangeDefaultPerQuery;
    if (expected_hits > 0) {
        const int64_t m = (expected_hits + nq - 1) / nq;
        per = m + m / 2 + 32;
    }
    return std::max<int64_t>(1, std::min(per, n_scan));
}

// The segmented sort of the collected keys (segs[q].keys / .n / .out set) into ix->range_items / range_scores.
static int range_sort(tav_index* ix, TimedSearch* ts, bool timing, std::vector<SortSeg>& segs, int64_t total,
                      const int64_t* d_subset, int64_t item_offset, int ties_low, cudaStream_t s) {
    const int nq = static_cast<int>(segs.size());
    std::vector<int> large, tile_seg;
    int64_t tmp_keys = 0;
    for (int q = 0; q < nq; ++q) {
        SortSeg& g = segs[q];
        g.tmp = nullptr;
        g.tile0 = 0;
        if (g.n > kSmallSortMax) {
            g.tmp = reinterpret_cast<uint64_t*>(static_cast<uintptr_t>(tmp_keys));  // offset for now
            g.tile0 = static_cast<int64_t>(tile_seg.size());
            const int64_t nt = (g.n + kRadixTile - 1) / kRadixTile;
            for (int64_t t = 0; t < nt; ++t) tile_seg.push_back(static_cast<int>(large.size()));
            large.push_back(q);
            tmp_keys += g.n;
        }
    }
    if (int rc = range_alloc(ix->range_items, static_cast<size_t>(total) * sizeof(int64_t), "the hits")) return rc;
    if (int rc = range_alloc(ix->range_scores, static_cast<size_t>(total) * sizeof(float), "the hit scores")) return rc;
    if (total == 0) return TAV_OK;
    if (int rc = range_alloc(ix->range_tmp, static_cast<size_t>(tmp_keys) * sizeof(uint64_t), "the sort scratch")) return rc;
    for (SortSeg& g : segs)
        if (g.n > kSmallSortMax)
            g.tmp = static_cast<uint64_t*>(ix->range_tmp.p) + reinterpret_cast<uintptr_t>(g.tmp);
    // sort workspace: segs | large | tile_seg | minmax | hist | offs
    const size_t n_tiles = tile_seg.size();
    const size_t b_segs = segs.size() * sizeof(SortSeg);
    const size_t o_large = (b_segs + 15) & ~size_t(15);
    const size_t o_tiles = (o_large + large.size() * sizeof(int) + 15) & ~size_t(15);
    const size_t o_minmax = (o_tiles + n_tiles * sizeof(int) + 15) & ~size_t(15);
    const size_t o_hist = o_minmax + large.size() * 2 * sizeof(uint64_t);
    const size_t o_offs = o_hist + n_tiles * 256 * sizeof(uint32_t);
    const size_t ws_bytes = o_offs + n_tiles * 256 * sizeof(uint32_t);
    if (int rc = range_alloc(ix->range_sortws, ws_bytes, "the sort workspace")) return rc;
    std::vector<char> head(o_minmax, 0);
    memcpy(head.data(), segs.data(), b_segs);
    if (!large.empty()) memcpy(head.data() + o_large, large.data(), large.size() * sizeof(int));
    if (n_tiles) memcpy(head.data() + o_tiles, tile_seg.data(), n_tiles * sizeof(int));
    char* ws = static_cast<char*>(ix->range_sortws.p);
    // from pageable memory: the copy has consumed `head` when the call returns
    TAV_CUDA(cudaMemcpyAsync(ws, head.data(), head.size(), cudaMemcpyHostToDevice, s));

    SortArgs sa{};
    sa.segs = reinterpret_cast<const SortSeg*>(ws);
    sa.n_segs = nq;
    sa.large = reinterpret_cast<const int*>(ws + o_large);
    sa.n_large = static_cast<int>(large.size());
    sa.tile_seg = reinterpret_cast<const int*>(ws + o_tiles);
    sa.n_tiles = static_cast<int64_t>(n_tiles);
    sa.minmax = reinterpret_cast<uint64_t*>(ws + o_minmax);
    sa.hist = reinterpret_cast<uint32_t*>(ws + o_hist);
    sa.offs = reinterpret_cast<uint32_t*>(ws + o_offs);
    sa.subset = d_subset;
    sa.item_offset = item_offset;
    sa.ties_low = ties_low;
    sa.out_items = static_cast<int64_t*>(ix->range_items.p);
    sa.out_scores = static_cast<float*>(ix->range_scores.p);
    TAV_CUDA(timed_launch(ix, ts, timing, 2, s, [&] { return launch_segmented_sort(sa, s, &ts->launches); }));
    return TAV_OK;
}

// Grouped lookups: every segment's keys -> the keys of its groups' leaders (tav_leaders.cu), compacted in place;
// segs[q].n, segs[q].out and offsets become the leaders' counts and CSR offsets.  One synchronisation, to learn the
// counts.  Scratch: 12 bytes per table slot, a power of two >= twice the segment's keys.
static int reduce_leaders(tav_index* ix, TimedSearch* ts, bool timing, std::vector<SortSeg>& segs,
                          std::vector<int64_t>& offsets, int ties_low, cudaStream_t s) {
    const int nq = static_cast<int>(segs.size());
    std::vector<LeaderSeg> ls(static_cast<size_t>(nq));
    int64_t slots = 0, key_tiles = 0, slot_tiles = 0;
    for (int q = 0; q < nq; ++q) {
        const int64_t n = segs[q].n;
        if (n > (int64_t(1) << 31)) {
            set_error("grouped search: %lld hits of one query are more than the leader reduction takes", (long long)n);
            return TAV_ERR_INVALID;
        }
        int64_t t = n ? 2 : 0;
        while (t && t < 2 * n) t <<= 1;
        ls[q] = LeaderSeg{segs[q].keys, n, slots, static_cast<uint32_t>(t - 1), key_tiles, slot_tiles};
        slots += t;
        key_tiles += (n + kLeaderTileKeys - 1) / kLeaderTileKeys;
        slot_tiles += (t + kLeaderTileKeys - 1) / kLeaderTileKeys;
    }
    if (int rc = range_alloc(ix->group_segs, ls.size() * sizeof(LeaderSeg), "the leader segments")) return rc;
    if (int rc = range_alloc(ix->group_table, static_cast<size_t>(slots) * 12, "the leader tables")) return rc;
    if (int rc = range_alloc(ix->group_counts, static_cast<size_t>(nq) * sizeof(uint32_t), "the leader counters"))
        return rc;
    uint64_t* tkey = static_cast<uint64_t*>(ix->group_table.p);
    int32_t* tgroup = reinterpret_cast<int32_t*>(tkey + slots);
    uint32_t* d_cnt = static_cast<uint32_t*>(ix->group_counts.p);
    // from pageable memory: consumed when the call returns
    TAV_CUDA(cudaMemcpyAsync(ix->group_segs.p, ls.data(), ls.size() * sizeof(LeaderSeg), cudaMemcpyHostToDevice, s));
    TAV_CUDA(cudaMemsetAsync(tkey, 0, static_cast<size_t>(slots) * sizeof(uint64_t), s));
    TAV_CUDA(cudaMemsetAsync(tgroup, 0xFF, static_cast<size_t>(slots) * sizeof(int32_t), s));
    TAV_CUDA(cudaMemsetAsync(d_cnt, 0, static_cast<size_t>(nq) * sizeof(uint32_t), s));
    TAV_CUDA(timed_launch(ix, ts, timing, 2, s, [&] {
        return launch_leaders(static_cast<const LeaderSeg*>(ix->group_segs.p), nq, key_tiles, slot_tiles,
                              static_cast<const int32_t*>(ix->group_map.p), ties_low, tgroup, tkey, d_cnt, s);
    }));
    ts->launches += 2;
    std::vector<uint32_t> cnt(static_cast<size_t>(nq));
    TAV_CUDA(cudaMemcpyAsync(cnt.data(), d_cnt, cnt.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    TAV_CUDA(cudaStreamSynchronize(s));
    offsets.assign(static_cast<size_t>(nq) + 1, 0);
    for (int q = 0; q < nq; ++q) {
        offsets[q + 1] = offsets[q] + cnt[q];
        segs[q].n = cnt[q];
        segs[q].out = offsets[q];
    }
    return TAV_OK;
}

// the masks of a re-pass over the gathered queries `over` (indexes into the search whose masks are qm)
static int gather_mask_map(tav_index* ix, const std::vector<int>& over, const QueryMasks& qm, QueryMasks& out,
                           cudaStream_t s) {
    if (int rc = range_alloc(ix->range_qmap, over.size() * sizeof(int32_t), "the re-pass mask map")) return rc;
    std::vector<int32_t> map(over.begin(), over.end());
    // from pageable memory: consumed when the call returns
    TAV_CUDA(cudaMemcpyAsync(ix->range_qmap.p, map.data(), map.size() * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    out = qm;
    out.map = TAV_QUERY_MASK_MUTANT == 3 ? nullptr : static_cast<const int32_t*>(ix->range_qmap.p);
    return TAV_OK;
}

// the queries `over` of d_queries, contiguous in ix->range_qgather for a re-pass (one copy per query)
static int gather_repass_queries(tav_index* ix, const float* d_queries, const std::vector<int>& over, cudaStream_t s) {
    const size_t qrow = static_cast<size_t>(ix->dim) * sizeof(float);
    if (int rc = range_alloc(ix->range_qgather, over.size() * qrow, "the re-pass queries")) return rc;
    char* qg = static_cast<char*>(ix->range_qgather.p);
    for (size_t i = 0; i < over.size(); ++i)
        TAV_CUDA(cudaMemcpyAsync(qg + i * qrow, reinterpret_cast<const char*>(d_queries) + over[i] * qrow, qrow,
                                 cudaMemcpyDeviceToDevice, s));
    return TAV_OK;
}

// Row-scan collection: one collect scan per block of queries into regions sized from `expected_hits`; the
// counters keep counting past a region, so after the one synchronisation the totals are exact and the
// overflowed queries get exactly one more scan into regions of that size.
static int range_collect_scan(tav_index* ix, TimedSearch* ts, bool timing, const float* d_queries, int nq, float floor,
                              const int64_t* d_subset, int64_t n_scan, int64_t item_offset, const uint32_t* d_mask,
                              int ties_low, int64_t expected_hits, std::vector<int64_t>& offsets, cudaStream_t s,
                              int positions = 0, QueryMasks qm = QueryMasks{}, bool leaders = false) {
    const int64_t per = range_per_query(expected_hits, nq, n_scan);
    if (int rc = range_alloc(ix->range_keys, static_cast<size_t>(nq) * per * sizeof(uint64_t), "the hit regions")) return rc;
    if (int rc = range_alloc(ix->range_counts, static_cast<size_t>(nq) * sizeof(uint32_t), "the hit counters")) return rc;
    uint32_t* d_counts = static_cast<uint32_t*>(ix->range_counts.p);
    uint64_t* keys = static_cast<uint64_t*>(ix->range_keys.p);
    TAV_CUDA(cudaMemsetAsync(d_counts, 0, static_cast<size_t>(nq) * sizeof(uint32_t), s));
    if (int rc = collect_scans(ix, ts, timing, d_queries, nq, floor, d_subset, n_scan, d_mask, ties_low, keys, per,
                               d_counts, s, qm))
        return rc;

    std::vector<uint32_t> cnt(static_cast<size_t>(nq));
    TAV_CUDA(cudaMemcpyAsync(cnt.data(), d_counts, cnt.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    TAV_CUDA(cudaStreamSynchronize(s));
    offsets.assign(static_cast<size_t>(nq) + 1, 0);
    std::vector<int> over;
    int64_t over_max = 0;
    for (int q = 0; q < nq; ++q) {
        offsets[q + 1] = offsets[q] + cnt[q];
        if (cnt[q] > per) {
            over.push_back(q);
            over_max = std::max<int64_t>(over_max, cnt[q]);
        }
    }
    // overflowed queries: one more scan, gathered, into regions of their now known size
    uint64_t* keys2 = nullptr;
    const int no = static_cast<int>(over.size());
    if (no > 0) {
        if (int rc = range_alloc(ix->range_keys2, static_cast<size_t>(no) * over_max * sizeof(uint64_t), "the re-pass regions"))
            return rc;
        if (int rc = gather_repass_queries(ix, d_queries, over, s)) return rc;
        keys2 = static_cast<uint64_t*>(ix->range_keys2.p);
        TAV_CUDA(cudaMemsetAsync(d_counts, 0, static_cast<size_t>(no) * sizeof(uint32_t), s));
        QueryMasks qm2{};
        if (qm.bits) {  // each gathered query keeps its own mask
            if (int rc = gather_mask_map(ix, over, qm, qm2, s)) return rc;
        }
        if (int rc = collect_scans(ix, ts, timing, static_cast<const float*>(ix->range_qgather.p), no, floor, d_subset,
                                   n_scan, d_mask, ties_low, keys2, over_max, d_counts, s, qm2))
            return rc;
    }
    std::vector<SortSeg> segs(static_cast<size_t>(nq));
    size_t oi = 0;
    for (int q = 0; q < nq; ++q) {
        const bool o = oi < over.size() && over[oi] == q;
        segs[q].keys = o ? keys2 + static_cast<size_t>(oi++) * over_max : keys + static_cast<size_t>(q) * per;
        segs[q].out = offsets[q];
        segs[q].n = cnt[q];
    }
    if (leaders)
        if (int rc = reduce_leaders(ix, ts, timing, segs, offsets, ties_low, s)) return rc;
    return range_sort(ix, ts, timing, segs, offsets[nq], positions ? nullptr : d_subset, item_offset, ties_low, s);
}

constexpr int kRangeUseScan = 1;  // range_collect_mma: the tensor-core form cannot serve this search

// Tensor-core collection: the MAIN kernel without a sample pass and with the exact dot floor of min_score
// as threshold, segments sized from `expected_hits`, a count kernel; after the one synchronisation the
// overflowed queries get one more MAIN pass (only they, same rows per segment, segments of the counted size)
// and every query's keys are gathered in CSR order.  Returns kRangeUseScan when the float32 split form met
// a value beyond the fp16 range (the exact row scan then serves the search, as it does for top-k searches).
static int range_collect_mma(tav_index* ix, TimedSearch* ts, bool timing, const float* d_queries, int nq, float floor,
                             int64_t item_offset, const uint32_t* d_mask, int ties_low, int64_t expected_hits,
                             std::vector<int64_t>& offsets, cudaStream_t s, QueryMasks qm, bool leaders) {
    const bool split = ix->dtype == TAV_F32;
    if (split) {
        const int rc = ensure_split_planes(ix, ts, s);
        if (rc == TAV_ERR_OOM) return kRangeUseScan;  // a speed choice, not a correctness one
        if (rc != TAV_OK) return rc;
    }
    // scratch: [nq] retry flags (query prep clears them) | [2] split overflow flags | [nq] gather offsets
    const size_t o_flags = (static_cast<size_t>(nq) * sizeof(int32_t) + 15) & ~size_t(15);
    const size_t o_dst = o_flags + 16;
    if (int rc = range_alloc(ix->range_mmaaux, o_dst + static_cast<size_t>(nq) * sizeof(int64_t), "the tensor-core scratch"))
        return rc;
    char* aux = static_cast<char*>(ix->range_mmaaux.p);
    int* d_qflag = reinterpret_cast<int*>(aux + o_flags);
    int64_t* d_dst = reinterpret_cast<int64_t*>(aux + o_dst);
    TAV_CUDA(cudaMemsetAsync(d_qflag, 0, 16, s));
    if (int rc = range_alloc(ix->range_counts, static_cast<size_t>(nq) * 2 * sizeof(uint32_t), "the hit counters")) return rc;
    uint32_t* d_tot = static_cast<uint32_t*>(ix->range_counts.p);
    uint32_t* d_max = d_tot + nq;
    if (timing)
        if (int rc = create_events(ts)) return rc;
    MmaArgs m = mma_args(ix, split);
    m.split_overflow = split ? d_qflag : nullptr;
    m.queries = d_queries;
    m.nq = nq;
    m.floor_score = floor;
    m.k = 1;
    m.item_offset = item_offset;
    m.retry_flags = reinterpret_cast<int32_t*>(aux);
    m.row_mask = d_mask;
    m.qmask = qm;
    int ev_used = ts->used;
    m.ev = timing ? ts->ev : nullptr;
    m.ev_kind = ts->kind;
    m.ev_max = kMaxTimedKernels;
    m.ev_used = &ev_used;
    const int64_t per = range_per_query(expected_hits, nq, ix->size);
    const MmaCollect shape = mma_collect_plan(m, 0, 1);
    // segments: twice a query's even share of its region (rows reach segments unevenly), a little more
    const MmaCollect c = mma_collect_plan(m, shape.per_chunk, 2 * ((per + shape.n_seg - 1) / shape.n_seg) + 8);
    if (int rc = range_alloc(ix->range_mmaws, c.ws_bytes, "the tensor-core workspace")) return rc;
    TAV_CUDA(launch_mma_collect(m, c, ix->range_mmaws.p, d_tot, d_max, s, &ts->launches));
    ts->used = ev_used;

    std::vector<uint32_t> host(2 * static_cast<size_t>(nq));
    int flags[2] = {0, 0};
    TAV_CUDA(cudaMemcpyAsync(host.data(), d_tot, host.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    if (split) {
        TAV_CUDA(cudaMemcpyAsync(&flags[0], d_qflag, sizeof(int), cudaMemcpyDeviceToHost, s));
        TAV_CUDA(cudaMemcpyAsync(&flags[1], ix->split_flag.p, sizeof(int), cudaMemcpyDeviceToHost, s));
    }
    TAV_CUDA(cudaStreamSynchronize(s));
    if (flags[0] || flags[1]) return kRangeUseScan;
    offsets.assign(static_cast<size_t>(nq) + 1, 0);
    std::vector<int> over;
    std::vector<int64_t> dst(static_cast<size_t>(nq));
    uint32_t over_seg = 0;
    for (int q = 0; q < nq; ++q) {
        offsets[q + 1] = offsets[q] + host[q];
        dst[q] = offsets[q];
        if (host[nq + q] > c.cap_seg) {
            over.push_back(q);
            over_seg = std::max(over_seg, host[nq + q]);
            dst[q] = -1;
        }
    }
    const int64_t total = offsets[nq];
    if (int rc = range_alloc(ix->range_keys, static_cast<size_t>(total) * sizeof(uint64_t), "the hit keys")) return rc;
    uint64_t* keys = static_cast<uint64_t*>(ix->range_keys.p);
    TAV_CUDA(cudaMemcpyAsync(d_dst, dst.data(), dst.size() * sizeof(int64_t), cudaMemcpyHostToDevice, s));
    TAV_CUDA(launch_mma_gather(m, c, ix->range_mmaws.p, d_dst, keys, ties_low, s));
    ts->launches += 1;

    const int no = static_cast<int>(over.size());
    if (no > 0) {
        // the overflowed queries, gathered, through the same units per chunk: every segment receives the
        // rows it received before, and the counts just read size it exactly
        if (int rc = gather_repass_queries(ix, d_queries, over, s)) return rc;
        MmaArgs m2 = m;
        m2.queries = static_cast<const float*>(ix->range_qgather.p);
        m2.nq = no;
        if (qm.bits) {  // each gathered query keeps its own mask
            if (int rc = gather_mask_map(ix, over, qm, m2.qmask, s)) return rc;
        }
        const MmaCollect c2 = mma_collect_plan(m2, c.per_chunk, over_seg);
        if (c2.n_seg != c.n_seg || c2.cap_seg < over_seg) {
            set_error("threshold search: tensor-core re-pass plan mismatch");
            return TAV_ERR_CUDA;
        }
        if (int rc = range_alloc(ix->range_mmaws2, c2.ws_bytes, "the tensor-core re-pass workspace")) return rc;
        ev_used = ts->used;
        TAV_CUDA(launch_mma_collect(m2, c2, ix->range_mmaws2.p, d_tot, d_max, s, &ts->launches));
        ts->used = ev_used;
        // the re-pass must admit exactly the rows the first pass counted (a second look at its counts)
        std::vector<uint32_t> host2(2 * static_cast<size_t>(no));
        TAV_CUDA(cudaMemcpyAsync(host2.data(), d_tot, no * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        TAV_CUDA(cudaMemcpyAsync(host2.data() + no, d_max, no * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        TAV_CUDA(cudaStreamSynchronize(s));
        for (int i = 0; i < no; ++i)
            if (host2[i] != host[over[i]] || host2[no + i] > c2.cap_seg) return kRangeUseScan;
        std::vector<int64_t> dst2(static_cast<size_t>(no));
        for (int i = 0; i < no; ++i) dst2[i] = offsets[over[i]];
        TAV_CUDA(cudaMemcpyAsync(d_dst, dst2.data(), dst2.size() * sizeof(int64_t), cudaMemcpyHostToDevice, s));
        TAV_CUDA(launch_mma_gather(m2, c2, ix->range_mmaws2.p, d_dst, keys, ties_low, s));
        ts->launches += 1;
    }
    std::vector<SortSeg> segs(static_cast<size_t>(nq));
    for (int q = 0; q < nq; ++q) {
        segs[q].keys = keys + offsets[q];
        segs[q].out = offsets[q];
        segs[q].n = host[q];
    }
    if (leaders)
        if (int rc = reduce_leaders(ix, ts, timing, segs, offsets, ties_low, s)) return rc;
    return range_sort(ix, ts, timing, segs, offsets[nq], nullptr, item_offset, ties_low, s);
}

// Every row with score >= floor, for each of nq device queries -> ix->range_items / range_scores in CSR order
// (offsets[nq + 1], host): collected by the tensor cores (use_mma) or the row scan, then the segmented sort.
// `leaders` (grouped lookups): only each group's leader is sorted (reduce_leaders), offsets count the leaders.
static int range_core(tav_index* ix, TimedSearch* ts, bool timing, const float* d_queries, int nq, float floor,
                      const int64_t* d_subset, int64_t n_scan, int64_t item_offset, const uint32_t* d_mask,
                      int ties_low, int64_t expected_hits, bool use_mma, std::vector<int64_t>& offsets, cudaStream_t s,
                      int positions = 0, QueryMasks qm = QueryMasks{}, bool leaders = false) {
    if (use_mma) {
        const int rc = range_collect_mma(ix, ts, timing, d_queries, nq, floor, item_offset, d_mask, ties_low,
                                         expected_hits, offsets, s, qm, leaders);
        if (rc != kRangeUseScan) return rc;
        ts->path = 1;  // a value beyond the fp16 range: the exact row scan serves the search
    }
    return range_collect_scan(ix, ts, timing, d_queries, nq, floor, d_subset, n_scan, item_offset, d_mask, ties_low,
                              expected_hits, offsets, s, positions, qm, leaders);
}

// ---- threshold search into caller buffers (tav_range_search_into) ----------------------------------------
// The hits land in the caller's device memory: CSR offsets [nq + 1] always complete, items / scores at the CSR
// positions below cap.  No host synchronisation: the plan kernel sizes the result on the device, the sort is
// launched over upper bounds known on the host, and a query whose region overflowed is flagged for
// tav_finish_search (finish_pending -> range_into_redo) instead of being re-collected now.  Nothing here touches
// range_items / range_scores: the hits of the last tav_range_search stay as they were until the next call that
// replaces them (tav_range_search_into itself gives them up on entry).
struct RangeOut {
    int64_t* offsets;
    int64_t* items;
    float* scores;
    int64_t cap;
};

// The "redo exactly" bookkeeping for searches of up to `need` queries, sized for `cap` when it grows (which
// finishes the outstanding searches first).
static int ensure_retry(tav_index* ix, int need, int cap, cudaStream_t s) {
    if (need <= ix->retry_cap && ix->retry.p && !ix->alloc_fail) return TAV_OK;
    if (int rc = finish_pending(ix, s, nullptr)) return rc;
    cap = std::max(cap, 1024);
    const size_t bytes = (static_cast<size_t>(2) * kMaxPending + static_cast<size_t>(kMaxPending) * cap) * sizeof(int32_t);
    TAV_CUDA(ix->retry.ensure(ix->alloc_fail ? ~size_t(0) >> 4 : bytes));
    TAV_CUDA(cudaMemsetAsync(ix->retry.p, 0, 2 * kMaxPending * sizeof(int32_t), s));
    TAV_CUDA(ix->retry_host.ensure(2 * kMaxPending * sizeof(int32_t)));
    memset(ix->retry_host.p, 0, 2 * kMaxPending * sizeof(int32_t));
    ix->retry_cap = cap;
    return TAV_OK;
}

// A deferred search re-reads its queries (and subset) at tav_finish_search, after later searches on this index have
// restaged ix->queries: `bytes` of held_queries stay its own until then (*out; *end = the region's end).  When they
// do not fit, a buffer of at least twice the size takes over and the old one is kept (not freed) until the
// searches that read it are finished: no search is finished early.
static int hold_region(tav_index* ix, size_t bytes, void** out, size_t* end) {
    bytes = (bytes + 255) & ~size_t(255);
    const size_t need = ix->held_used + bytes;
    if (need > ix->held_queries.bytes) {
        const size_t want = std::max(need, 2 * ix->held_queries.bytes);
        if (ix->held_used > 0) {  // pending searches read the current buffer
            ix->held_retired.push_back(std::move(ix->held_queries));
            ix->held_used = 0;
        }
        TAV_CUDA(ix->held_queries.ensure(want));
    }
    *out = static_cast<char*>(ix->held_queries.p) + ix->held_used;
    ix->held_used += bytes;
    *end = ix->held_used;
    return TAV_OK;
}

// Where a plan's results go besides the sort setup (see RangePlanArgs): a first pass scans the counts into
// `offsets` and flags its overflowed queries; a re-pass puts query i's hits at base[i] (host, nq entries).
struct PlanDest {
    int64_t* offsets = nullptr;
    const int64_t* base = nullptr;
    int32_t* flags = nullptr;
    int32_t* n_flagged = nullptr;
    int32_t* n_flagged_host = nullptr;
    const int* abandon[2] = {nullptr, nullptr};
    // per-query subsets: query q's keys at keys + key_off[q] (device), total_keys in all (region, key_stride unused)
    const int64_t* key_off = nullptr;
    int64_t total_keys = 0;
};

// The device plan of nq queries whose counters are count / fill (see RangePlanArgs), at most `region` keys per
// query that did not overflow, then the sort setup: *sa for launch_segmented_sort_dev, *sizes its counts, and
// (packed keys) *dst_off the gather offsets.
static int range_plan(tav_index* ix, TimedSearch* ts, int nq, const uint32_t* count, const uint32_t* fill, uint32_t cap,
                      int64_t region, int64_t key_stride, uint64_t* keys, const int64_t* d_subset, int64_t item_offset,
                      int ties_low, const RangeOut& out, const PlanDest& dest, SortArgs* sa, const int** sizes,
                      int64_t** dst_off, cudaStream_t s) {
    const bool var = dest.key_off != nullptr;
    const bool any_large = (var ? dest.total_keys : region) > kSmallSortMax;
    // variable bases: at most total / (kSmallSortMax + 1) large segments, whose tiles number at most
    // total / kRadixTile + one partial tile each
    const int n_large_max =
        !any_large ? 0 : var ? static_cast<int>(std::min<int64_t>(nq, dest.total_keys / (kSmallSortMax + 1))) : nq;
    const int64_t tiles_max = !any_large ? 0
                              : var      ? dest.total_keys / kRadixTile + n_large_max
                                         : static_cast<int64_t>(nq) * ((region + kRadixTile - 1) / kRadixTile);
    uint64_t* tmp = nullptr;
    if (any_large) {
        const int64_t tmp_keys = var ? dest.total_keys : static_cast<int64_t>(nq) * region;
        if (int rc = range_alloc(ix->range_tmp, static_cast<size_t>(tmp_keys) * sizeof(uint64_t), "the sort scratch"))
            return rc;
        tmp = static_cast<uint64_t*>(ix->range_tmp.p);
    }
    // sort workspace: segs | large | tile_seg | minmax | hist | offs | sizes | dst_off | base
    auto up = [](size_t o) { return (o + 15) & ~size_t(15); };
    const size_t o_large = up(static_cast<size_t>(nq) * sizeof(SortSeg));
    const size_t o_tiles = up(o_large + static_cast<size_t>(n_large_max) * sizeof(int));
    const size_t o_minmax = up(o_tiles + static_cast<size_t>(tiles_max) * sizeof(int));
    const size_t o_hist = o_minmax + static_cast<size_t>(n_large_max) * 2 * sizeof(uint64_t);
    const size_t o_offs = o_hist + static_cast<size_t>(tiles_max) * 256 * sizeof(uint32_t);
    const size_t o_sizes = o_offs + static_cast<size_t>(tiles_max) * 256 * sizeof(uint32_t);
    const size_t o_dst = up(o_sizes + 2 * sizeof(int));
    const size_t o_base = o_dst + static_cast<size_t>(nq) * sizeof(int64_t);
    const size_t ws_bytes = o_base + (dest.base ? static_cast<size_t>(nq) * sizeof(int64_t) : 0);
    if (int rc = range_alloc(ix->range_sortws, ws_bytes, "the sort workspace")) return rc;
    char* ws = static_cast<char*>(ix->range_sortws.p);
    if (dest.base)  // from pageable memory: consumed when the call returns
        TAV_CUDA(cudaMemcpyAsync(ws + o_base, dest.base, static_cast<size_t>(nq) * sizeof(int64_t), cudaMemcpyHostToDevice, s));

    RangePlanArgs pa{};
    pa.nq = nq;
    pa.count = count;
    pa.fill = fill;
    pa.cap = cap;
    pa.key_stride = key_stride;
    pa.keys = keys;
    pa.tmp = tmp;
    pa.out_offsets = dest.offsets;
    pa.out_base = dest.base ? reinterpret_cast<const int64_t*>(ws + o_base) : nullptr;
    pa.abandon[0] = dest.abandon[0];
    pa.abandon[1] = dest.abandon[1];
    pa.dst_off = key_stride || var ? nullptr : reinterpret_cast<int64_t*>(ws + o_dst);
    pa.flags = dest.flags;
    pa.n_flagged = dest.n_flagged;
    pa.n_flagged_host = dest.n_flagged_host;
    pa.segs = reinterpret_cast<SortSeg*>(ws);
    pa.large = reinterpret_cast<int*>(ws + o_large);
    pa.tile_seg = reinterpret_cast<int*>(ws + o_tiles);
    pa.minmax = reinterpret_cast<uint64_t*>(ws + o_minmax);
    pa.sizes = reinterpret_cast<int*>(ws + o_sizes);
    TAV_CUDA(var ? launch_range_plan_subsets(pa, dest.key_off, s) : launch_range_plan(pa, s));
    ts->launches += 1;

    *sa = SortArgs{};
    sa->segs = pa.segs;
    sa->n_segs = nq;
    sa->large = pa.large;
    sa->n_large = n_large_max;
    sa->tile_seg = pa.tile_seg;
    sa->n_tiles = tiles_max;
    sa->minmax = pa.minmax;
    sa->hist = reinterpret_cast<uint32_t*>(ws + o_hist);
    sa->offs = reinterpret_cast<uint32_t*>(ws + o_offs);
    sa->subset = d_subset;
    sa->item_offset = item_offset;
    sa->ties_low = ties_low;
    sa->out_items = out.items;
    sa->out_scores = out.scores;
    *sizes = pa.sizes;
    *dst_off = pa.dst_off;
    return TAV_OK;
}

static int range_sort_dev(tav_index* ix, TimedSearch* ts, bool timing, const SortArgs& sa, const int* sizes, int64_t cap,
                          cudaStream_t s) {
    TAV_CUDA(timed_launch(ix, ts, timing, 2, s, [&] { return launch_segmented_sort_dev(sa, sizes, cap, s, &ts->launches); }));
    return TAV_OK;
}

// the tensor-core collection plan of a threshold search: segments sized from expected_hits as in range_collect_mma
static MmaCollect range_mma_plan(const MmaArgs& m, int64_t expected_hits, int nq, int64_t n_rows) {
    const int64_t per = range_per_query(expected_hits, nq, n_rows);
    const MmaCollect shape = mma_collect_plan(m, 0, 1);
    return mma_collect_plan(m, shape.per_chunk, 2 * ((per + shape.n_seg - 1) / shape.n_seg) + 8);
}

// A first pass: collection (the row scan, or the tensor cores with the split form's planes), device plan and sort
// of a threshold search into `out`, all queued on s.  The plan's flags go to bookkeeping slot `slot` (and, with
// `count_flags`, their number).  *per_chunk / *n_seg: the tensor-core plan (0 for the row scan), which a re-pass
// must repeat.  Returns kRangeUseScan when the split planes cannot be allocated (the row scan then serves the
// search, as in range_collect_mma).
static int range_into_core(tav_index* ix, TimedSearch* ts, bool timing, const float* d_queries, int nq, float floor,
                           const int64_t* d_subset, int64_t n_scan, int64_t item_offset, const uint32_t* d_mask,
                           QueryMasks qm, int ties_low, int64_t expected_hits, bool use_mma, int slot, bool count_flags,
                           const RangeOut& out, int* per_chunk, int* n_seg, cudaStream_t s) {
    SortArgs sa;
    const int* sizes = nullptr;
    int64_t* dst_off = nullptr;
    PlanDest dest;
    dest.offsets = out.offsets;
    dest.flags = retry_flags(ix, slot);
    if (count_flags) {
        dest.n_flagged = retry_totals(ix, slot);
        dest.n_flagged_host = static_cast<int32_t*>(ix->retry_host.p) + 2 * slot;
    }
    *per_chunk = *n_seg = 0;
    if (!use_mma) {
        const int64_t per = range_per_query(expected_hits, nq, n_scan);
        if (int rc = range_alloc(ix->range_keys, static_cast<size_t>(nq) * per * sizeof(uint64_t), "the hit regions")) return rc;
        if (int rc = range_alloc(ix->range_counts, static_cast<size_t>(nq) * sizeof(uint32_t), "the hit counters")) return rc;
        uint32_t* d_counts = static_cast<uint32_t*>(ix->range_counts.p);
        uint64_t* keys = static_cast<uint64_t*>(ix->range_keys.p);
        TAV_CUDA(cudaMemsetAsync(d_counts, 0, static_cast<size_t>(nq) * sizeof(uint32_t), s));
        if (int rc = collect_scans(ix, ts, timing, d_queries, nq, floor, d_subset, n_scan, d_mask, ties_low, keys, per,
                                   d_counts, s, qm))
            return rc;
        if (int rc = range_plan(ix, ts, nq, d_counts, d_counts, static_cast<uint32_t>(per), per, per, keys, d_subset,
                                item_offset, ties_low, out, dest, &sa, &sizes, &dst_off, s))
            return rc;
    } else {
        const bool split = ix->dtype == TAV_F32;
        if (split) {
            const int rc = ensure_split_planes(ix, ts, s);
            if (rc == TAV_ERR_OOM) return kRangeUseScan;
            if (rc != TAV_OK) return rc;
        }
        if (int rc = range_alloc(ix->range_counts, static_cast<size_t>(nq) * 2 * sizeof(uint32_t), "the hit counters")) return rc;
        uint32_t* d_tot = static_cast<uint32_t*>(ix->range_counts.p);
        uint32_t* d_max = d_tot + nq;
        if (timing)
            if (int rc = create_events(ts)) return rc;
        MmaArgs m = mma_args(ix, split);
        // a query value beyond the fp16 range flags the whole search (finish_pending reads the mapped twin)
        m.split_overflow = split ? retry_totals(ix, slot) + 1 : nullptr;
        m.split_overflow_host = split ? static_cast<int*>(ix->retry_host.p) + 2 * slot + 1 : nullptr;
        m.queries = d_queries;
        m.nq = nq;
        m.floor_score = floor;
        m.k = 1;
        m.item_offset = item_offset;
        m.retry_flags = retry_flags(ix, slot);  // scratch of the query prep; the plan writes the flags after it
        m.row_mask = d_mask;
        m.qmask = qm;
        int ev_used = ts->used;
        m.ev = timing ? ts->ev : nullptr;
        m.ev_kind = ts->kind;
        m.ev_max = kMaxTimedKernels;
        m.ev_used = &ev_used;
        const MmaCollect c = range_mma_plan(m, expected_hits, nq, ix->size);
        if (int rc = range_alloc(ix->range_mmaws, c.ws_bytes, "the tensor-core workspace")) return rc;
        TAV_CUDA(launch_mma_collect(m, c, ix->range_mmaws.p, d_tot, d_max, s, &ts->launches));
        ts->used = ev_used;
        // a query that did not overflow has at most every segment full of keys
        const int64_t region = static_cast<int64_t>(c.n_seg) * c.cap_seg;
        if (int rc = range_alloc(ix->range_keys, static_cast<size_t>(nq) * region * sizeof(uint64_t), "the hit keys")) return rc;
        uint64_t* keys = static_cast<uint64_t*>(ix->range_keys.p);
        if (split) {  // the split form's overflow: nothing of this pass may reach the outputs (it is redone whole)
            dest.abandon[0] = m.split_overflow;
            dest.abandon[1] = static_cast<const int*>(ix->split_flag.p);
        }
        if (int rc = range_plan(ix, ts, nq, d_tot, d_max, c.cap_seg, region, 0, keys, nullptr, item_offset, ties_low, out,
                                dest, &sa, &sizes, &dst_off, s))
            return rc;
        TAV_CUDA(launch_mma_gather(m, c, ix->range_mmaws.p, dst_off, keys, ties_low, s));
        ts->launches += 1;
        *per_chunk = c.per_chunk;
        *n_seg = c.n_seg;
    }
    return range_sort_dev(ix, ts, timing, sa, sizes, out.cap, s);
}

// The filter of a re-pass over the queries `over` of a deferred search: its row mask, or its per-query masks
// through a map (each gathered query keeps its own mask).
static int repass_masks(tav_index* ix, const Pending& p, const std::vector<int>& over, const uint32_t** d_mask,
                        QueryMasks* qm, cudaStream_t s) {
    *d_mask = p.qm.bits ? nullptr : p.mask;
    *qm = QueryMasks{};
    if (p.qm.bits) return gather_mask_map(ix, over, p.qm, *qm, s);
    return TAV_OK;
}

// Row-scan re-pass of the flagged queries `over` of a deferred search, gathered, in one collect pass with regions
// of the largest count (nothing can overflow: the same kernel counts the same rows), sorted into the search's
// outputs at their offsets `off` (host, the search's CSR offsets).
static int range_repass_scan(tav_index* ix, const Pending& p, const std::vector<int>& over, const std::vector<int64_t>& off,
                             cudaStream_t s) {
    TimedSearch ts;
    const int no = static_cast<int>(over.size());
    int64_t per = 1;
    std::vector<int64_t> base(static_cast<size_t>(no));
    for (int i = 0; i < no; ++i) {
        per = std::max(per, off[over[i] + 1] - off[over[i]]);
        base[i] = off[over[i]];
    }
    if (int rc = gather_repass_queries(ix, p.queries, over, s)) return rc;
    const uint32_t* d_mask;
    QueryMasks qm;
    if (int rc = repass_masks(ix, p, over, &d_mask, &qm, s)) return rc;
    if (int rc = range_alloc(ix->range_keys, static_cast<size_t>(no) * per * sizeof(uint64_t), "the re-pass regions")) return rc;
    if (int rc = range_alloc(ix->range_counts, static_cast<size_t>(no) * sizeof(uint32_t), "the hit counters")) return rc;
    uint32_t* d_counts = static_cast<uint32_t*>(ix->range_counts.p);
    uint64_t* keys = static_cast<uint64_t*>(ix->range_keys.p);
    TAV_CUDA(cudaMemsetAsync(d_counts, 0, static_cast<size_t>(no) * sizeof(uint32_t), s));
    if (int rc = collect_scans(ix, &ts, false, static_cast<const float*>(ix->range_qgather.p), no, p.floor, p.subset,
                               p.n_scan, d_mask, p.ties_low, keys, per, d_counts, s, qm))
        return rc;
    SortArgs sa;
    const int* sizes = nullptr;
    int64_t* dst_off = nullptr;
    PlanDest dest;
    dest.base = base.data();
    const RangeOut out{nullptr, p.items, p.scores, p.cap};
    if (int rc = range_plan(ix, &ts, no, d_counts, d_counts, static_cast<uint32_t>(per), per, per, keys, p.subset,
                            p.item_offset, p.ties_low, out, dest, &sa, &sizes, &dst_off, s))
        return rc;
    return range_sort_dev(ix, &ts, false, sa, sizes, p.cap, s);
}

// Tensor-core re-pass of the flagged queries `over` (fill = each one's fullest segment) of a deferred search, as
// range_collect_mma re-passes: gathered, through the same units per query chunk (every segment receives the rows
// it received before) with segments of the fullest size.  Its counts are checked against the first pass's (one
// synchronisation) before anything is written; on a mismatch it returns kRangeUseScan and writes nothing.
static int range_repass_mma(tav_index* ix, const Pending& p, const std::vector<int>& over, uint32_t over_seg,
                            const std::vector<int64_t>& off, cudaStream_t s) {
    TimedSearch ts;
    const int no = static_cast<int>(over.size());
    if (int rc = gather_repass_queries(ix, p.queries, over, s)) return rc;
    MmaArgs m = mma_args(ix, p.split);
    m.split_overflow = p.split ? retry_totals(ix, p.slot) + 1 : nullptr;
    m.queries = static_cast<const float*>(ix->range_qgather.p);
    m.nq = no;
    m.floor_score = p.floor;
    m.k = 1;
    m.item_offset = p.item_offset;
    m.retry_flags = retry_flags(ix, p.slot);  // scratch (the flags were read)
    if (int rc = repass_masks(ix, p, over, &m.row_mask, &m.qmask, s)) return rc;
    const MmaCollect c = mma_collect_plan(m, p.per_chunk, over_seg);
    if (c.n_seg != p.n_seg || c.cap_seg < over_seg) return kRangeUseScan;
    if (int rc = range_alloc(ix->range_mmaws2, c.ws_bytes, "the tensor-core re-pass workspace")) return rc;
    if (int rc = range_alloc(ix->range_counts, static_cast<size_t>(no) * 2 * sizeof(uint32_t), "the hit counters")) return rc;
    uint32_t* d_tot = static_cast<uint32_t*>(ix->range_counts.p);
    uint32_t* d_max = d_tot + no;
    TAV_CUDA(launch_mma_collect(m, c, ix->range_mmaws2.p, d_tot, d_max, s, &ts.launches));
    std::vector<uint32_t> host(2 * static_cast<size_t>(no));
    TAV_CUDA(cudaMemcpyAsync(host.data(), d_tot, host.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    TAV_CUDA(cudaStreamSynchronize(s));
    int64_t most = 1;
    std::vector<int64_t> base(static_cast<size_t>(no));
    for (int i = 0; i < no; ++i) {
        const int64_t n = off[over[i] + 1] - off[over[i]];
        if (host[i] != static_cast<uint64_t>(n) || host[no + i] > c.cap_seg) return kRangeUseScan;
        most = std::max(most, n);
        base[i] = off[over[i]];
    }
    if (int rc = range_alloc(ix->range_keys, static_cast<size_t>(no) * most * sizeof(uint64_t), "the hit keys")) return rc;
    uint64_t* keys = static_cast<uint64_t*>(ix->range_keys.p);
    SortArgs sa;
    const int* sizes = nullptr;
    int64_t* dst_off = nullptr;
    PlanDest dest;
    dest.base = base.data();
    const RangeOut out{nullptr, p.items, p.scores, p.cap};
    if (int rc = range_plan(ix, &ts, no, d_tot, d_max, c.cap_seg, most, 0, keys, nullptr, p.item_offset, p.ties_low, out,
                            dest, &sa, &sizes, &dst_off, s))
        return rc;
    TAV_CUDA(launch_mma_gather(m, c, ix->range_mmaws2.p, dst_off, keys, p.ties_low, s));
    return range_sort_dev(ix, &ts, false, sa, sizes, p.cap, s);
}

// What a deferred threshold search into caller buffers left for tav_finish_search (finish_pending, after its
// synchronisation).  Its flagged queries are searched again, gathered, by the collection that flagged them (a
// row-scan re-pass, or a tensor-core re-pass with the same plan) and sorted into their places.  The whole search is
// searched again by the row scan, offsets included, when the split form met a value beyond the fp16 range (its
// first pass then wrote no hits) or a tensor-core re-pass does not count what the first pass counted (a safeguard,
// as in range_collect_mma; the first pass's hits may then remain between the new total and the capacity).
static int range_into_redo(tav_index* ix, const Pending& p, bool redo_all, int* n_redone, cudaStream_t s) {
    std::vector<int64_t> off(static_cast<size_t>(p.nq) + 1);
    std::vector<int32_t> flag(static_cast<size_t>(p.nq));
    auto read_plan = [&]() -> int {
        TAV_CUDA(cudaMemcpyAsync(off.data(), p.offsets, off.size() * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
        TAV_CUDA(cudaMemcpyAsync(flag.data(), retry_flags(ix, p.slot), flag.size() * sizeof(int32_t),
                                 cudaMemcpyDeviceToHost, s));
        TAV_CUDA(cudaStreamSynchronize(s));
        return TAV_OK;
    };
    auto flagged = [&](uint32_t* most) {
        std::vector<int> over;
        *most = 0;
        for (int q = 0; q < p.nq; ++q)
            if (flag[q]) {
                over.push_back(q);
                *most = std::max(*most, static_cast<uint32_t>(flag[q]));
            }
        return over;
    };
    uint32_t over_seg = 0;
    if (!redo_all) {
        if (int rc = read_plan()) return rc;
        const std::vector<int> over = flagged(&over_seg);
        *n_redone += static_cast<int>(over.size());
        if (over.empty()) return TAV_OK;
        if (p.per_chunk == 0) return range_repass_scan(ix, p, over, off, s);
        const int rc = range_repass_mma(ix, p, over, over_seg, off, s);
        if (rc != kRangeUseScan) return rc;
        *n_redone -= static_cast<int>(over.size());  // counted below with the whole search
    }
    // the whole search by the row scan, into the same outputs; what overflows its regions gets a row-scan re-pass
    TimedSearch ts;
    int per_chunk, n_seg;
    const RangeOut out{p.offsets, p.items, p.scores, p.cap};
    if (int rc = range_into_core(ix, &ts, false, p.queries, p.nq, p.floor, p.subset, p.n_scan, p.item_offset,
                                 p.qm.bits ? nullptr : p.mask, p.qm, p.ties_low, p.expected_hits, false, p.slot, false,
                                 out, &per_chunk, &n_seg, s))
        return rc;
    *n_redone += p.nq;
    if (int rc = read_plan()) return rc;
    const std::vector<int> over = flagged(&over_seg);
    return over.empty() ? TAV_OK : range_repass_scan(ix, p, over, off, s);
}

// ---- removal and overwrite (tav_remove_rows, tav_write_rows) -----------------------------------------------
constexpr size_t kCompactScratchBytes = size_t(256) << 20;  // window buffer of the in-place compaction

// Compacts the rows after the removal of `rem` (sorted, distinct, not empty) on s and synchronises s.  Rows
// [0, rem[0]) are not written.  Out of place (tav_internal_compact_policy mode 1) — a fresh allocation of the
// capacity, the rows before rem[0] copied over unchanged, each moving row read and written once; the old
// allocation is handed back in *old_rows for the caller to free.  In place by default: ascending windows of destinations, each gathered into a scratch buffer and copied back (the
// sources of a window lie at or above its first row, and rows above it are written only by later windows).
static int compact_rows(tav_index* ix, const std::vector<int64_t>& rem, cudaStream_t s, void** old_rows,
                        size_t* old_bytes) {
    *old_rows = nullptr;
    *old_bytes = 0;
    ix->compact_path = 0;
    ix->compact_windows = 0;
    const int64_t m = static_cast<int64_t>(rem.size());
    const int64_t first = rem[0], new_size = ix->size - m;
    const int64_t moving = new_size - first;  // surviving rows after the first removed one
    if (moving == 0) return TAV_OK;           // only the last rows were removed
    const size_t row = static_cast<size_t>(ix->dim) * dtype_size(ix->dtype);
    std::vector<int64_t> keys(rem.size());
    for (int64_t i = 0; i < m; ++i) keys[i] = rem[i] - i;
    TAV_CUDA(ix->compact_keys.ensure(keys.size() * sizeof(int64_t)));
    // from pageable memory: the copy has consumed `keys` when the call returns
    TAV_CUDA(cudaMemcpyAsync(ix->compact_keys.p, keys.data(), keys.size() * sizeof(int64_t), cudaMemcpyHostToDevice, s));
    const int64_t* d_keys = static_cast<const int64_t*>(ix->compact_keys.p);

    // Bytes moved: out of place 2 * (first + moving) rows, in place 4 * moving (one scratch round trip).  The
    // in-place form is the default all the same: at 10M x 768 bf16 the cudaMalloc / cudaFree of a second copy
    // of the rows cost about what the scratch round trip costs (DESIGN.md §3.5), and it needs no second copy.
    if (ix->compact_mode == 1) {
        void* fresh = nullptr;
        const size_t fresh_bytes = std::max<size_t>(static_cast<size_t>(ix->capacity) * row, 256);
        cudaError_t e = rows_malloc(&fresh, fresh_bytes);
        if (e != cudaSuccess) {
            cudaGetLastError();
            set_error("tav_remove_rows: no device memory for an out-of-place compaction");
            return TAV_ERR_OOM;
        }
        e = first > 0 ? cudaMemcpyAsync(fresh, ix->rows, static_cast<size_t>(first) * row, cudaMemcpyDeviceToDevice, s)
                      : cudaSuccess;
        if (e == cudaSuccess) e = launch_compact_gather(ix->rows, fresh, d_keys, m, first, new_size, 0, row, s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (e != cudaSuccess) {
            rows_free(fresh, fresh_bytes);
            set_error("tav_remove_rows: compaction failed: %s", cudaGetErrorString(e));
            return TAV_ERR_CUDA;
        }
        *old_rows = ix->rows;
        *old_bytes = ix->rows_bytes;
        ix->rows = fresh;
        ix->rows_bytes = fresh_bytes;
        ix->compact_path = 1;
        ix->compact_windows = 1;
        return TAV_OK;
    }
    const size_t scratch_bytes = ix->compact_scratch > 0 ? static_cast<size_t>(ix->compact_scratch) : kCompactScratchBytes;
    int64_t win = std::min<int64_t>(moving, std::max<int64_t>(1, static_cast<int64_t>(scratch_bytes / row)));
    // the form for short memory: when the window buffer does not fit, halve it (down to one row) rather than fail
    DevBuf scratch;
    for (;;) {
        const cudaError_t ae = scratch.ensure(static_cast<size_t>(win) * row);
        if (ae == cudaSuccess) break;
        cudaGetLastError();
        if (ae != cudaErrorMemoryAllocation || win == 1) {
            set_error("tav_remove_rows: cannot allocate the compaction window (%zu bytes): %s",
                      static_cast<size_t>(win) * row, cudaGetErrorString(ae));
            return ae == cudaErrorMemoryAllocation ? TAV_ERR_OOM : TAV_ERR_CUDA;
        }
        win = std::max<int64_t>(1, win / 2);
    }
    cudaError_t e = cudaSuccess;
    int64_t windows = 0;
    for (int64_t d0 = first; d0 < new_size && e == cudaSuccess; d0 += win, ++windows) {
        const int64_t d1 = std::min(new_size, d0 + win);
        e = launch_compact_gather(ix->rows, scratch.p, d_keys, m, d0, d1, d0, row, s);
        if (e == cudaSuccess)
            e = launch_compact_copy(ix->device, scratch.p, static_cast<char*>(ix->rows) + static_cast<size_t>(d0) * row,
                                    d1 - d0, row, s);
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) {
        set_error("tav_remove_rows: compaction failed: %s", cudaGetErrorString(e));
        return TAV_ERR_CUDA;
    }
    ix->compact_path = 2;
    ix->compact_windows = windows;
    return TAV_OK;
}

extern "C" {

int tav_remove_rows(tav_index* ix, const int64_t* ordinals, int64_t n, void* stream) {
    if (!ix || n < 0 || (n > 0 && !ordinals)) {
        set_error("tav_remove_rows: invalid argument");
        return TAV_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lock(ix->mu);
    if (ix->adopted) {
        set_error("tav_remove_rows: index uses adopted device memory");
        return TAV_ERR_STATE;
    }
    // np.delete semantics: negative ordinals count from the end, duplicates remove one row, order is free
    if (int rc = check_subset_ordinals(ix, ordinals, n)) return rc;
    if (n == 0) return TAV_OK;
    std::vector<int64_t> rem(static_cast<size_t>(n));
    for (int64_t i = 0; i < n; ++i) rem[i] = ordinals[i] < 0 ? ordinals[i] + ix->size : ordinals[i];
    if (!std::is_sorted(rem.begin(), rem.end())) std::sort(rem.begin(), rem.end());
    rem.erase(std::unique(rem.begin(), rem.end()), rem.end());
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (int rc = enter_stream(ix, s)) return rc;  // queued searches read the old rows
    // the outstanding deferred searches are finished first: their exact redo reads the rows
    if (int rc = finish_pending(ix, s, nullptr)) return rc;
    void* old_rows = nullptr;
    size_t old_bytes = 0;
    if (int rc = compact_rows(ix, rem, s, &old_rows, &old_bytes)) return rc;
    if (ix->compact_path != 0) mark_done(ix);  // s was synchronised after the compaction
    rows_free(old_rows, old_bytes);
    ix->size -= static_cast<int64_t>(rem.size());
    ix->split_rows = std::min(ix->split_rows, rem[0]);
    ix->split_recheck = true;
    ix->qmask_n = 0;
    ix->row_mask_rows = 0;  // ordinals changed meaning (a later append can restore the old size)
    ix->group_rows = 0;
    return TAV_OK;
}

int tav_write_rows(tav_index* ix, int64_t first, const void* rows, int64_t n, int dim, int src_dtype,
                   int src_on_device, void* stream) {
    if (!ix || n < 0 || dim <= 0 || !dtype_ok(src_dtype) || (n > 0 && !rows)) {
        set_error("tav_write_rows: invalid argument");
        return TAV_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lock(ix->mu);
    if (ix->adopted) {
        set_error("tav_write_rows: index uses adopted device memory");
        return TAV_ERR_STATE;
    }
    if (first < 0 || n > ix->size - first) {
        set_error("tav_write_rows: rows [%lld, %lld) out of range (size %lld)", (long long)first,
                  (long long)(first + n), (long long)ix->size);
        return TAV_ERR_RANGE;
    }
    if (dim != ix->dim) {
        set_error("Embedding size mismatch: expected %d, got %d", ix->dim, dim);
        return TAV_ERR_INVALID;
    }
    if (n == 0) return TAV_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (int rc = enter_stream(ix, s)) return rc;  // queued searches read the old rows
    // the outstanding deferred searches are finished first: their exact redo reads the rows
    if (int rc = finish_pending(ix, s, nullptr)) return rc;
    if (int rc = store_rows(ix, first, rows, n, src_dtype, src_on_device, s)) return rc;
    ix->split_rows = std::min(ix->split_rows, first);
    ix->split_recheck = true;
    return mark_queued(ix, s);
}

int tav_internal_compact_policy(tav_index* ix, int mode, int64_t scratch_bytes) {
    if (!ix || mode < 0 || mode > 2 || scratch_bytes < 0) return TAV_ERR_INVALID;
    std::lock_guard<std::mutex> lock(ix->mu);
    ix->compact_mode = mode;
    ix->compact_scratch = scratch_bytes;
    return TAV_OK;
}

int tav_internal_compact_stats(tav_index* ix, int* path, int64_t* windows) {
    if (!ix) return TAV_ERR_INVALID;
    std::lock_guard<std::mutex> lock(ix->mu);
    if (path) *path = ix->compact_path;
    if (windows) *windows = ix->compact_windows;
    return TAV_OK;
}

int tav_internal_row_bytes(tav_index* ix, int64_t* index_bytes, int64_t* process_bytes) {
    if (!ix) return TAV_ERR_INVALID;
    std::lock_guard<std::mutex> lock(ix->mu);
    if (index_bytes) *index_bytes = static_cast<int64_t>((ix->adopted ? 0 : ix->rows_bytes) + ix->staged_bytes);
    if (process_bytes) *process_bytes = g_row_bytes.load();
    return TAV_OK;
}

int tav_internal_stage_cap(tav_index* ix, int64_t max_bytes) {
    if (!ix || max_bytes < -1) return TAV_ERR_INVALID;
    std::lock_guard<std::mutex> lock(ix->mu);
    ix->stage_cap = max_bytes;
    return TAV_OK;
}

int tav_internal_qmask_cap(tav_index* ix, int64_t max_bytes) {
    if (!ix || max_bytes < -1) return TAV_ERR_INVALID;
    std::lock_guard<std::mutex> lock(ix->mu);
    ix->qmask_cap = max_bytes;
    return TAV_OK;
}

int tav_internal_search_alloc_fail(tav_index* ix, int on) {
    if (!ix) return TAV_ERR_INVALID;
    std::lock_guard<std::mutex> lock(ix->mu);
    ix->alloc_fail = on != 0;
    return TAV_OK;
}

}  // extern "C"

// ---- rebalance: a rank's new block copied from the ranks' row allocations over CUDA IPC -------------------
// one rank's record, as tav_rows_export writes it and tav_rows_stage reads it
struct RowsRecord {
    cudaIpcMemHandle_t handle;
    int64_t rows;       // rows of the rank's block
    int64_t has_handle; // 0: the rank has no row allocation (no piece can come from it)
    int32_t dim;        // the row layout: a piece is read with the stager's row size, so the ranks' must match
    int32_t dtype;
};

// the peers' row allocations mapped into this process for one stage; closed when it goes out of scope
struct PeerMappings {
    std::vector<void*> base;
    explicit PeerMappings(int world) : base(static_cast<size_t>(world), nullptr) {}
    ~PeerMappings() {
        for (void* p : base)
            if (p) cudaIpcCloseMemHandle(p);
    }
};

extern "C" {

int tav_rows_handle_bytes(void) { return static_cast<int>(sizeof(RowsRecord)); }

int tav_rows_export(tav_index* ix, void* handle_out, int64_t* rows_out) {
    if (!ix || !handle_out) return TAV_ERR_INVALID;
    std::lock_guard<std::mutex> lock(ix->mu);
    if (ix->adopted) {
        set_error("tav_rows_export: index uses adopted device memory");
        return TAV_ERR_STATE;
    }
    if (int rc = set_device(ix)) return rc;
    if (int rc = wait_queued(ix)) return rc;  // the peers read the rows as the calls so far leave them
    RowsRecord rec;
    memset(&rec, 0, sizeof(rec));
    rec.rows = ix->size;
    rec.dim = ix->dim;
    rec.dtype = ix->dtype;
    if (ix->rows && ix->size > 0) {
        TAV_CUDA(cudaIpcGetMemHandle(&rec.handle, ix->rows));
        rec.has_handle = 1;
    }
    memcpy(handle_out, &rec, sizeof(rec));
    if (rows_out) *rows_out = ix->size;
    return TAV_OK;
}

int tav_rows_stage(tav_index* ix, int world, int rank, const void* handles, int n_parts, const int32_t* part_src_rank,
                   const int64_t* part_first, const int64_t* part_rows, float* mirror_out, void* stream) {
    if (!ix || world < 1 || rank < 0 || rank >= world || n_parts < 0 || (world > 1 && !handles) ||
        (n_parts > 0 && (!part_src_rank || !part_first || !part_rows))) {
        set_error("tav_rows_stage: invalid argument");
        return TAV_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lock(ix->mu);
    if (ix->adopted) {
        set_error("tav_rows_stage: index uses adopted device memory");
        return TAV_ERR_STATE;
    }
    if (ix->staged) {
        set_error("tav_rows_stage: rows are already staged (tav_rows_commit first)");
        return TAV_ERR_STATE;
    }
    if (mirror_out && (ix->dtype != TAV_F32 || (ix->flags & TAV_NORMALIZE))) {
        set_error("tav_rows_stage: the rows read back equal the appended ones only on a float32 index without "
                  "TAV_NORMALIZE");
        return TAV_ERR_INVALID;
    }
    std::vector<RowsRecord> recs(static_cast<size_t>(world));
    if (world > 1) memcpy(recs.data(), handles, recs.size() * sizeof(RowsRecord));
    int64_t total = 0;
    for (int i = 0; i < n_parts; ++i) {
        const int src = part_src_rank[i];
        if (src < 0 || src >= world) {
            set_error("tav_rows_stage: piece %d names rank %d of %d", i, src, world);
            return TAV_ERR_INVALID;
        }
        const int64_t have = src == rank ? ix->size : recs[src].rows;
        const bool mapped = src == rank || recs[src].has_handle;
        if (src != rank && part_rows[i] > 0 && (recs[src].dim != ix->dim || recs[src].dtype != ix->dtype)) {
            set_error("tav_rows_stage: rank %d holds rows of %d elements of dtype %d, this index %d of dtype %d", src,
                      recs[src].dim, recs[src].dtype, ix->dim, ix->dtype);
            return TAV_ERR_INVALID;
        }
        if (part_first[i] < 0 || part_rows[i] < 0 || part_rows[i] > have - part_first[i] ||
            (part_rows[i] > 0 && !mapped)) {
            set_error("tav_rows_stage: piece %d, rows [%lld, %lld) of rank %d, is outside its %lld rows", i,
                      (long long)part_first[i], (long long)(part_first[i] + part_rows[i]), src, (long long)have);
            return TAV_ERR_RANGE;
        }
        total += part_rows[i];
    }
    const size_t row = static_cast<size_t>(ix->dim) * dtype_size(ix->dtype);
    const size_t bytes = std::max<size_t>(static_cast<size_t>(total) * row, 256);
    if (ix->stage_cap >= 0 && bytes > static_cast<size_t>(ix->stage_cap)) {
        set_error("tav_rows_stage: %zu bytes for the new block exceed the stage cap of %lld", bytes,
                  (long long)ix->stage_cap);
        return TAV_ERR_OOM;
    }
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (int rc = enter_stream(ix, s)) return rc;
    // the rows are about to be replaced: the outstanding deferred searches' exact redo reads them
    if (int rc = finish_pending(ix, s, nullptr)) return rc;
    void* fresh = nullptr;
    cudaError_t e = rows_malloc(&fresh, bytes);
    if (e != cudaSuccess) {
        cudaGetLastError();
        set_error("tav_rows_stage: cannot allocate %zu bytes for the new block: %s", bytes, cudaGetErrorString(e));
        return e == cudaErrorMemoryAllocation ? TAV_ERR_OOM : TAV_ERR_CUDA;
    }
    // destination order; TAV_REBALANCE_MUTANT 1 lays the first two pieces out swapped (the same bytes in all)
    std::vector<int> order(static_cast<size_t>(n_parts));
    for (int i = 0; i < n_parts; ++i) order[i] = i;
    if (TAV_REBALANCE_MUTANT == 1 && n_parts >= 2) std::swap(order[0], order[1]);
    {
        PeerMappings peers(world);
        int64_t dst = 0;
        for (int j = 0; j < n_parts && e == cudaSuccess; ++j) {
            const int i = order[j];
            const int src = part_src_rank[i];
            if (part_rows[i] == 0) continue;
            const char* base = static_cast<const char*>(ix->rows);
            if (src != rank) {
                if (!peers.base[src]) {
                    e = cudaIpcOpenMemHandle(&peers.base[src], recs[src].handle, cudaIpcMemLazyEnablePeerAccess);
                    if (e != cudaSuccess) {
                        peers.base[src] = nullptr;
                        break;
                    }
                }
                base = static_cast<const char*>(peers.base[src]);
            }
            // across GPUs the copy engines move the piece over NVLink; on one GPU it is a device-to-device copy
            e = cudaMemcpyAsync(static_cast<char*>(fresh) + static_cast<size_t>(dst) * row,
                                base + static_cast<size_t>(part_first[i]) * row, static_cast<size_t>(part_rows[i]) * row,
                                cudaMemcpyDefault, s);
            dst += part_rows[i];
        }
        if (e == cudaSuccess && mirror_out && total > 0)
            e = cudaMemcpyAsync(mirror_out, fresh, static_cast<size_t>(total) * row, cudaMemcpyDeviceToHost, s);
        // before the mappings close, also after a failure: no queued copy may still read a peer's rows
        const cudaError_t se = cudaStreamSynchronize(s);
        if (e == cudaSuccess) e = se;
    }
    if (e != cudaSuccess) {
        rows_free(fresh, bytes);
        set_error("tav_rows_stage: copying the new block failed: %s", cudaGetErrorString(e));
        return TAV_ERR_CUDA;
    }
    mark_done(ix);
    ix->staged = fresh;
    ix->staged_rows = total;
    ix->staged_bytes = bytes;
    return TAV_OK;
}

int tav_rows_commit(tav_index* ix, int commit) {
    if (!ix || (commit != 0 && commit != 1)) return TAV_ERR_INVALID;
    std::lock_guard<std::mutex> lock(ix->mu);
    if (int rc = set_device(ix)) return rc;
    if (!commit) {
        rows_free(ix->staged, ix->staged_bytes);
        ix->staged = nullptr;
        ix->staged_rows = 0;
        ix->staged_bytes = 0;
        return TAV_OK;
    }
    if (!ix->staged) {
        set_error("tav_rows_commit: no rows are staged");
        return TAV_ERR_STATE;
    }
    if (int rc = wait_queued(ix)) return rc;  // queued searches read the old rows
    if (TAV_REBALANCE_MUTANT != 4) rows_free(ix->rows, ix->rows_bytes);  // mutant 4 leaks the old rows
    ix->rows = ix->staged;
    ix->rows_bytes = ix->staged_bytes;
    ix->size = ix->capacity = ix->staged_rows;
    ix->staged = nullptr;
    ix->staged_rows = 0;
    ix->staged_bytes = 0;
    // every row may have changed: the planes are rebuilt from row 0, which also resets their overflow flag
    ix->split_rows = TAV_REBALANCE_MUTANT == 2 ? std::min(ix->split_rows, ix->size) : 0;
    ix->split_recheck = false;
    if (TAV_REBALANCE_MUTANT != 3) ix->row_mask_rows = 0;  // ordinals changed meaning
    ix->group_rows = 0;
    ix->qmask_n = 0;
    return TAV_OK;
}

const int32_t* tav_internal_retry_totals(tav_index* ix, int* count) {
    if (count) *count = 0;
    if (!ix || ix->last_first_slot < 0 || !ix->retry.p) return nullptr;
    if (count) *count = ix->last_n_slots;
    return retry_totals(ix, ix->last_first_slot);
}

const int* tav_internal_split_flag(tav_index* ix) {
    if (!ix || ix->last_first_slot < 0 || !ix->last_split) return nullptr;
    return static_cast<const int*>(ix->split_flag.p);
}

int tav_finish_search(tav_index* ix, void* stream, int* redone) {
    if (!ix) return TAV_ERR_INVALID;
    std::lock_guard<std::mutex> lock(ix->mu);
    if (redone) *redone = 0;
    if (!ix->pending.empty()) {  // (else nothing deferred: row-scan path, or already finished)
        if (int rc = set_device(ix)) return rc;
        if (int rc = finish_pending(ix, static_cast<cudaStream_t>(stream), redone)) return rc;
    }
    // a deferred subset search refused on the device, here or in an earlier finish the library ran itself
    const int rc = ix->deferred_rc;
    if (rc != TAV_OK) set_error("%s", ix->deferred_msg.c_str());
    ix->deferred_rc = TAV_OK;
    return rc;
}

// tav_search with the index's mutex held (tav_search_groups runs it as its first step)
static int search_locked(tav_index* ix, const float* queries, int n_queries, int k, float min_score, int flags,
                         const int64_t* subset, int64_t subset_len, int64_t item_offset, int64_t* out_items,
                         float* out_scores, int32_t* out_counts, void* stream);

int tav_search(tav_index* ix, const float* queries, int n_queries, int k, float min_score,
               int flags, const int64_t* subset, int64_t subset_len, int64_t item_offset,
               int64_t* out_items, float* out_scores, int32_t* out_counts, void* stream) {
    if (!ix || n_queries < 0 || k < 1 || (n_queries > 0 && (!queries || !out_items || !out_scores || !out_counts))) {
        set_error("tav_search: invalid argument (k must be >= 1)");
        return TAV_ERR_INVALID;
    }
    if (int rc = check_subset_args("tav_search", flags, subset, subset_len, false)) return rc;
    if (n_queries == 0) return TAV_OK;
    std::lock_guard<std::mutex> lock(ix->mu);
    return search_locked(ix, queries, n_queries, k, min_score, flags, subset, subset_len, item_offset, out_items,
                         out_scores, out_counts, stream);
}

static int search_locked(tav_index* ix, const float* queries, int n_queries, int k, float min_score, int flags,
                         const int64_t* subset, int64_t subset_len, int64_t item_offset, int64_t* out_items,
                         float* out_scores, int32_t* out_counts, void* stream) {
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (int rc = enter_stream(ix, s)) return rc;
    const bool q_dev = flags & TAV_QUERIES_ON_DEVICE, o_dev = flags & TAV_OUTPUTS_ON_DEVICE;
    const uint32_t* d_mask = nullptr;
    QueryMasks qm;
    if (int rc = resolve_masks(ix, "tav_search", n_queries, flags, subset != nullptr, &d_mask, &qm)) return rc;
    const int ties_low = (flags & TAV_TIES_LOW_FIRST) ? 1 : 0;
    const int positions = (flags & TAV_ITEMS_AS_POSITIONS) && TAV_SHARDED_FILTER_MUTANT != 3 ? 1 : 0;

    int64_t* d_items = out_items;
    float* d_scores = out_scores;
    int32_t* d_counts = out_counts;
    const ResultPack pack(n_queries, k);
    // Small result sets are written by the kernels straight into the pinned host staging (zero
    // copy over PCIe: no D2H memcpy call on the single-lookup latency path).
    const bool zero_copy_out = !o_dev && pack.bytes() <= kZeroCopyOutLimit;

    const int64_t n_scan = subset ? subset_len : ix->size;
    TimedSearch* ts = begin_search(ix, 0);
    const bool timing = ts != &ix->untimed;

    // a NaN min_score admits nothing on every path (`scores >= nan` is all-false in the reference)
    if (n_scan == 0 || ix->size == 0 || ix->dim == 0 || min_score != min_score) {
        // empty corpus / empty subset: no hits (vectorbase.py:174-175, :214-215)
        if (o_dev) {
            TAV_CUDA(cudaMemsetAsync(d_counts, 0, static_cast<size_t>(n_queries) * sizeof(int32_t), s));
            return mark_queued(ix, s);
        }
        memset(out_counts, 0, static_cast<size_t>(n_queries) * sizeof(int32_t));
        return TAV_OK;
    }
    if (n_scan > 0xFFFFFFFFll) {
        set_error("tav_search: more than 2^32 rows per index are not supported; shard the corpus");
        return TAV_ERR_INVALID;
    }

    // subset ordinals: validate on the host (numpy raises IndexError)
    if (int rc = check_subset_ordinals(ix, subset, subset_len)) return rc;

    // path choice: tensor cores for batches on 16-bit storage, row scan otherwise
    bool use_mma = false, use_split = false;
    const bool mma_able = mma_supported(ix->dtype, ix->dim) || (ix->dtype == TAV_F32 && mma_split_supported(ix->dim));
    if (!(flags & TAV_FORCE_SCAN) && !subset && mma_able && k <= kPassK && !ties_low) {
        use_mma = (flags & TAV_FORCE_MMA) || (n_queries >= 16 && ix->size >= 4096);
        use_split = use_mma && ix->dtype == TAV_F32;
    }
    if ((flags & TAV_FORCE_MMA) && !use_mma) {
        set_error("tav_search: TAV_FORCE_MMA needs dim %% 8 == 0, no subset, k <= %d", kPassK);
        return TAV_ERR_INVALID;
    }

    // ---- every passing row of a large scan (k >= rows; the reference's max_hits = 0) ------------------
    // The threshold engine (collect scan + segmented sort) reads the rows once where the paged form would
    // run ceil(k / kPassK) passes; same kernels' dots and the same key order, so the same result, which is
    // then laid out as [n_queries, k] with -1 / 0 padding.  Regions of n_scan keys per query: no re-pass.
    if (!use_mma && !o_dev && k >= n_scan && n_scan > 4 * kPassK) {
        ts->path = 1;
        const float* d_q = nullptr;
        const int64_t* d_sub = nullptr;
        if (int rc = stage_inputs(ix, ts, timing, queries, n_queries, q_dev, false, subset, subset_len, &d_q, &d_sub, s))
            return rc;
        std::vector<int64_t> offsets;
        ix->range_total = 0;
        ix->range_grouped = false;
        ix->range_replaced = false;
        if (int rc = range_core(ix, ts, timing, d_q, n_queries, min_score, d_sub, n_scan, item_offset, d_mask, ties_low,
                                static_cast<int64_t>(n_queries) * n_scan, false, offsets, s, positions, qm))
            return rc;
        if (int rc = end_search(ix, ts, s)) return rc;
        ix->range_total = offsets[n_queries];
        // each query's hits straight into its row of the caller's arrays (copies from device memory into
        // pageable memory return when done), then the padding
        for (int q = 0; q < n_queries; ++q) {
            const int64_t c = offsets[q + 1] - offsets[q];
            int64_t* it = out_items + static_cast<size_t>(q) * k;
            float* sc = out_scores + static_cast<size_t>(q) * k;
            if (c > 0) {
                TAV_CUDA(cudaMemcpyAsync(it, static_cast<const int64_t*>(ix->range_items.p) + offsets[q],
                                         static_cast<size_t>(c) * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
                TAV_CUDA(cudaMemcpyAsync(sc, static_cast<const float*>(ix->range_scores.p) + offsets[q],
                                         static_cast<size_t>(c) * sizeof(float), cudaMemcpyDeviceToHost, s));
            }
        }
        TAV_CUDA(cudaStreamSynchronize(s));
        mark_done(ix);
        for (int q = 0; q < n_queries; ++q) {
            const int64_t c = offsets[q + 1] - offsets[q];
            std::fill(out_items + static_cast<size_t>(q) * k + c, out_items + static_cast<size_t>(q + 1) * k, int64_t(-1));
            std::fill(out_scores + static_cast<size_t>(q) * k + c, out_scores + static_cast<size_t>(q + 1) * k, 0.0f);
            out_counts[q] = static_cast<int32_t>(c);
        }
        return TAV_OK;
    }

    // result staging for host outputs (after the routing above, which needs none)
    if (zero_copy_out) {
        TAV_CUDA(ix->pin_out.ensure(pack.bytes()));
        pack.place(ix->pin_out.p, &d_items, &d_scores, &d_counts);
    } else if (!o_dev) {
        TAV_CUDA(ix->out_pack.ensure(pack.bytes()));
        pack.place(ix->out_pack.p, &d_items, &d_scores, &d_counts);
    }

    // ---- single-lookup latency form: ONE launch, no copies -------------------------------------
    // One host query with host outputs on the row-scan path: the query (and a short subset) ride in
    // the kernel parameters, the last CTA merges and writes the hits into mapped pinned memory and
    // raises a completion word the host spins on (tools/benchmark_vectorbase.py:97-158 is this call).
    if (!use_mma && n_queries == 1 && !q_dev && zero_copy_out && !(ix->flags & TAV_NORMALIZE) && k <= 1024 &&
        scan_max_queries(ix->dim, k) >= 1 && scan1_fits(ix->dim, k, n_scan, subset_len, subset != nullptr) &&
        static_cast<size_t>(n_scan) * ix->dim * dtype_size(ix->dtype) <= kFusedScanMaxBytes &&
        !(flags & TAV_NO_FUSED_SCAN)) {
        ts->path = 1;
        if (int rc = ensure_scan_counters(ix, s)) return rc;
        uint64_t* d_bound = static_cast<uint64_t*>(ix->cand_count.p);
        uint32_t* d_count = reinterpret_cast<uint32_t*>(d_bound + 8);
        ScanArgs a = scan_args(ix);
        a.n_scan = n_scan;
        a.nq = 1;
        a.floor_score = min_score;
        a.k = k;
        a.grid = scan1_grid(ix->device, ix->dim, k, n_scan);
        a.cand_stride = a.grid * std::max(k, 32);   // a CTA hands over its k best (room for a round of 32 rows)
        TAV_CUDA(ix->cand_keys.ensure(static_cast<size_t>(a.cand_stride) * sizeof(uint64_t)));
        a.cand_keys = static_cast<uint64_t*>(ix->cand_keys.p);
        a.cand_count = d_count;
        a.row_mask = d_mask;
        a.ties_low = ties_low;
        a.subset_in_params = subset ? 1 : 0;
        a.items_as_positions = positions;
        a.fused = 1;
        a.fused_ticket = d_count + 8;
        a.item_offset = item_offset;
        a.out_items = d_items;
        a.out_scores = d_scores;
        a.out_counts = d_counts;
        // Completion.  Small k: NO completion word and no system-scope fence in the kernel (that fence waits
        // ~1.8 us for the result stores to cross PCIe before the word may follow them): the host pre-fills the
        // mapped result slots with values no hit can have and watches the slots themselves — the count and
        // all k items and scores; every slot is one aligned store, so it arrives whole.  Larger k: one
        // completion word behind a fence.
        const bool watch_slots = k <= kWatchSlotsMaxK;
        volatile uint32_t* done = reinterpret_cast<volatile uint32_t*>(static_cast<char*>(ix->pin_out.p) + pack.off_done);
        volatile int64_t* w_items = reinterpret_cast<volatile int64_t*>(d_items);
        volatile uint32_t* w_scores = reinterpret_cast<volatile uint32_t*>(d_scores);
        volatile int32_t* w_count = reinterpret_cast<volatile int32_t*>(d_counts);
        if (watch_slots) {
            for (int j = 0; j < k; ++j) {
                w_items[j] = kNoItemYet;
                w_scores[j] = kNoScoreYet;
            }
            *w_count = -1;
        } else {
            a.done_flag = const_cast<uint32_t*>(done);
            a.done_seq = ++ix->done_seq;
            if (a.done_seq == 0) a.done_seq = ++ix->done_seq;
            *done = 0;
        }
        static const bool trace_on = getenv("TAV_TRACE") != nullptr;
        unsigned long long* trace_host = nullptr;
        unsigned long long t_host0 = 0;
        if (trace_on) {  // diagnostic: phase stamps of the kernel in mapped pinned memory, printed to stderr
            TAV_CUDA(ix->pin_in.ensure(4096));
            trace_host = reinterpret_cast<unsigned long long*>(static_cast<char*>(ix->pin_in.p) + 2048);
            memset(trace_host, 0, 64);
            a.trace = trace_host;
            timespec tsn;
            clock_gettime(CLOCK_MONOTONIC, &tsn);
            t_host0 = static_cast<unsigned long long>(tsn.tv_sec) * 1000000000ull + tsn.tv_nsec;
        }
        if (timing) TAV_CUDA(ev_record(ts->total[0], s));
        TAV_CUDA(timed_launch(ix, ts, timing, 0, s, [&] { return launch_scan1(a, queries, subset, s); }));
        ts->launches = 1;
        if (int rc = end_search(ix, ts, s)) return rc;
        // spin on the completion word (a stream synchronise costs several microseconds more); fall
        // back to the synchronise when the word does not show up quickly (error, or a busy GPU)
        bool seen = false;
        for (int spin = 0; spin < 4000000; ++spin) {
            if (watch_slots) {
                // ALL k slots (the kernel also writes the padding beyond `count`): once they are in, no store
                // of this launch is still on its way to the buffer the next call pre-fills
                if (*w_count >= 0) {
                    int j = 0;
                    while (j < k && w_items[j] != kNoItemYet && w_scores[j] != kNoScoreYet) ++j;
                    if (j >= k) {
                        seen = true;
                        break;
                    }
                }
            } else if (*done == a.done_seq) {
                seen = true;
                break;
            }
            if ((spin & 0x3FFF) == 0x3FFF && cudaStreamQuery(s) != cudaErrorNotReady) break;
        }
        if (!seen) TAV_CUDA(cudaStreamSynchronize(s));
        // the kernel started after the earlier calls' work (join_stream) and has written its hits: nothing of
        // this index is left queued (only its last CTA's counter reset may still be retiring)
        mark_done(ix);
        std::atomic_thread_fence(std::memory_order_acquire);  // the copies below read what the spin saw
        if (trace_host) {
            timespec tsn;
            clock_gettime(CLOCK_MONOTONIC, &tsn);
            const unsigned long long t_host1 = static_cast<unsigned long long>(tsn.tv_sec) * 1000000000ull + tsn.tv_nsec;
            cudaStreamSynchronize(s);
            static int printed = 0;
            if (++printed % 500 == 0)
                fprintf(stderr, "[tav trace] grid %d: staged +%.1f us, scanned +%.1f, handed +%.1f (CTA 0) | last CTA: merge starts at %.1f, hits "
                                "written +%.1f, flag +%.1f (kernel %.1f us) | host call until flag seen %.1f us\n", a.grid,
                        (trace_host[1] - trace_host[0]) / 1e3, (trace_host[2] - trace_host[1]) / 1e3,
                        (trace_host[3] - trace_host[2]) / 1e3, (trace_host[4] - trace_host[0]) / 1e3,
                        (trace_host[5] - trace_host[4]) / 1e3, (trace_host[6] - trace_host[5]) / 1e3,
                        (trace_host[6] - trace_host[0]) / 1e3, (t_host1 - t_host0) / 1e3);
        }
        pack.unpack(ix->pin_out.p, out_items, out_scores, out_counts);
        return TAV_OK;
    }

    // A deferred search redoes its flagged queries at tav_finish_search, after later searches on this index
    // have restaged ix->queries: normalised queries then go to a region of held_queries that is its own
    // until then.  When they do not fit, a buffer of at least twice the size takes over and the old one is
    // kept (not freed) until the searches that read it are finished: no search is finished early.
    const bool defer = (flags & TAV_DEFER_RETRY) && o_dev && q_dev;
    float* held = nullptr;
    size_t held_end = 0;
    if (use_mma && defer && (ix->flags & TAV_NORMALIZE)) {
        void* r = nullptr;
        if (int rc = hold_region(ix, static_cast<size_t>(n_queries) * ix->dim * sizeof(float), &r, &held_end)) return rc;
        held = static_cast<float*>(r);
    }

    const int64_t* d_subset = nullptr;
    const float* d_queries = nullptr;
    if (int rc = stage_inputs(ix, ts, timing, queries, n_queries, q_dev, o_dev, subset, subset_len, &d_queries, &d_subset, s,
                              held))
        return rc;

    if (use_split) {
        const int rc = ensure_split_planes(ix, ts, s);
        if (rc == TAV_ERR_OOM && !(flags & TAV_FORCE_MMA)) {
            use_mma = use_split = false;  // a speed choice, not a correctness one: the exact row scan serves it
        } else if (rc != TAV_OK) {
            return rc;
        }
    }

    if (use_mma) {
        ts->path = use_split ? 3 : 2;
        if (int rc = ensure_retry(ix, n_queries, std::min(n_queries, kMmaMaxQueries), s)) return rc;
        if (timing)
            if (int rc = create_events(ts)) return rc;
        // one launch sequence per slab of kMmaMaxQueries queries (in practice: one)
        for (int q0 = 0; q0 < n_queries; q0 += kMmaMaxQueries) {
            const int nq = std::min(kMmaMaxQueries, n_queries - q0);
            // bookkeeping slot of this (part of the) search
            if (static_cast<int>(ix->pending.size()) >= kMaxPending)
                if (int rc = finish_pending(ix, s, nullptr)) return rc;
            const int slot = ix->next_slot++;
            if (q0 == 0) ix->last_first_slot = slot;
            ix->last_n_slots = slot - ix->last_first_slot + 1;
            ix->last_split = use_split;
            MmaArgs m = mma_args(ix, use_split);
            m.split_overflow = use_split ? retry_totals(ix, slot) + 1 : nullptr;
            m.queries = d_queries + static_cast<size_t>(q0) * ix->dim;
            m.nq = nq;
            m.floor_score = min_score;
            m.k = k;
            m.item_offset = item_offset;
            m.out_items = d_items + static_cast<size_t>(q0) * k;
            m.out_scores = d_scores + static_cast<size_t>(q0) * k;
            m.out_counts = d_counts + q0;
            m.retry_flags = retry_flags(ix, slot);
            m.retry_total = retry_totals(ix, slot);
            m.retry_total_host = static_cast<int32_t*>(ix->retry_host.p) + 2 * slot;
            m.split_overflow_host = use_split ? static_cast<int*>(ix->retry_host.p) + 2 * slot + 1 : nullptr;
            m.row_mask = d_mask;
            m.qmask = qmask_from(qm, q0);
            int ev_used = 0;
            const bool slab_timed = timing && q0 == 0;
            m.ev = slab_timed ? ts->ev : nullptr;
            m.ev_kind = ts->kind;
            m.ev_max = kMaxTimedKernels;
            m.ev_used = &ev_used;
            m.ev_main_only = ix->timing_light ? 1 : 0;
            if (int rc = ensure_mma_ws(ix, mma_workspace_bytes(m), s)) return rc;
            int launches = 0;
            TAV_CUDA(launch_mma_search(m, ix->mma_ws.p, ix->mma_ws.bytes, s, &launches));
            if (slab_timed) ts->used = ev_used;
            ts->launches += launches;
            Pending p{m.queries, nq, k, min_score, item_offset, m.out_items, m.out_scores, m.out_counts, slot,
                      use_split, m.qmask.bits ? m.qmask.bits : d_mask, m.qmask.bits ? m.qmask.stride : 0};
            ix->pending.push_back(p);
            ix->held_used = std::max(ix->held_used, held_end);  // (a finish_pending above may have reset it)
        }
        // Queries the sampled admission threshold could not settle (fewer than k admitted rows
        // although rows were cut, or candidate overflow) are redone exactly by the row scan —
        // now, or in tav_finish_search when the caller defers the (synchronising) check.
        if (!defer)
            if (int rc = finish_pending(ix, s, nullptr)) return rc;
    } else {
        ts->path = 1;
        int rc = scan_search(ix, ts, timing, d_queries, n_queries, k, min_score, d_subset, n_scan, item_offset,
                             d_items, d_scores, d_counts, d_mask, ties_low, s, !(flags & TAV_NO_FUSED_SCAN), positions, qm);
        if (rc != TAV_OK) return rc;
    }
    if (int rc = end_search(ix, ts, s)) return rc;

    if (o_dev) return mark_queued(ix, s);
    if (zero_copy_out) {
        TAV_CUDA(cudaStreamSynchronize(s));
        pack.unpack(ix->pin_out.p, out_items, out_scores, out_counts);
    } else if (pack.bytes() <= kPinnedStageLimit) {
        TAV_CUDA(ix->pin_out.ensure(pack.bytes()));
        TAV_CUDA(cudaMemcpyAsync(ix->pin_out.p, ix->out_pack.p, pack.off_done, cudaMemcpyDeviceToHost, s));
        TAV_CUDA(cudaStreamSynchronize(s));
        pack.unpack(ix->pin_out.p, out_items, out_scores, out_counts);
    } else {
        if (int rc = copy_pack_out(pack, ix->out_pack.p, out_items, out_scores, out_counts, s)) return rc;
    }
    mark_done(ix);  // host outputs: s was synchronised above
    return TAV_OK;
}

// path choice of the threshold search, as in tav_search: tensor cores for batches (no subset), the row scan otherwise
static int range_path(const tav_index* ix, const char* fn, int n_queries, int flags, bool has_subset, bool* use_mma) {
    const bool mma_able = (mma_supported(ix->dtype, ix->dim) || (ix->dtype == TAV_F32 && mma_split_supported(ix->dim))) &&
                          !has_subset && n_queries <= kMmaMaxQueries && ix->size < (1ll << 31);
    *use_mma = !(flags & TAV_FORCE_SCAN) && mma_able &&
               ((flags & TAV_FORCE_MMA) || (n_queries >= 16 && ix->size >= 4096));
    if ((flags & TAV_FORCE_MMA) && !*use_mma) {
        set_error("%s: TAV_FORCE_MMA needs dim %% 8 == 0, no subset, at most %d queries", fn, kMmaMaxQueries);
        return TAV_ERR_INVALID;
    }
    return TAV_OK;
}

int tav_range_search(tav_index* ix, const float* queries, int n_queries, float min_score, int flags,
                     const int64_t* subset, int64_t subset_len, int64_t item_offset, int64_t expected_hits,
                     int64_t* out_offsets, void* stream) {
    if (!ix || n_queries < 0 || expected_hits < 0 || !out_offsets || (n_queries > 0 && !queries)) {
        set_error("tav_range_search: invalid argument");
        return TAV_ERR_INVALID;
    }
    if (int rc = check_subset_args("tav_range_search", flags, subset, subset_len, true)) return rc;
    std::lock_guard<std::mutex> lock(ix->mu);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (int rc = enter_stream(ix, s)) return rc;  // (also: a queued tav_range_fetch reads the hits replaced here)
    const bool q_dev = flags & TAV_QUERIES_ON_DEVICE, o_dev = flags & TAV_OUTPUTS_ON_DEVICE;
    ix->range_total = 0;
    ix->range_grouped = false;
    ix->range_replaced = false;
    std::vector<int64_t> offsets(static_cast<size_t>(n_queries) + 1, 0);
    const uint32_t* d_mask = nullptr;
    QueryMasks qm;
    if (int rc = resolve_masks(ix, "tav_range_search", n_queries, flags, subset != nullptr, &d_mask, &qm)) return rc;
    const int64_t n_scan = subset ? subset_len : ix->size;
    // NaN min_score, empty corpus or empty subset: no hits
    if (n_queries == 0 || n_scan == 0 || ix->size == 0 || ix->dim == 0 || min_score != min_score)
        return deliver_offsets(ix, offsets, out_offsets, o_dev, s);
    if (n_scan > 0xFFFFFFFFll) {
        set_error("tav_range_search: more than 2^32 rows per index are not supported; shard the corpus");
        return TAV_ERR_INVALID;
    }
    if (int rc = check_subset_ordinals(ix, subset, subset_len)) return rc;
    bool use_mma = false;
    if (int rc = range_path(ix, "tav_range_search", n_queries, flags, subset != nullptr, &use_mma)) return rc;
    TimedSearch* ts = begin_search(ix, use_mma ? (ix->dtype == TAV_F32 ? 3 : 2) : 1);
    const bool timing = ts != &ix->untimed;
    const float* d_queries = nullptr;
    const int64_t* d_subset = nullptr;
    if (int rc = stage_inputs(ix, ts, timing, queries, n_queries, q_dev, false, subset, subset_len, &d_queries, &d_subset, s))
        return rc;
    if (int rc = range_core(ix, ts, timing, d_queries, n_queries, min_score, d_subset, n_scan, item_offset, d_mask,
                            (flags & TAV_TIES_LOW_FIRST) ? 1 : 0, expected_hits, use_mma, offsets, s,
                            (flags & TAV_ITEMS_AS_POSITIONS) && TAV_SHARDED_FILTER_MUTANT != 3 ? 1 : 0, qm))
        return rc;
    if (int rc = end_search(ix, ts, s)) return rc;
    ix->range_total = offsets[n_queries];
    return deliver_offsets(ix, offsets, out_offsets, o_dev, s);
}

int tav_range_fetch(tav_index* ix, int64_t first, int64_t n, int64_t* out_items, float* out_scores, int flags,
                    void* stream) {
    if (!ix || first < 0 || n < 0 || (n > 0 && (!out_items || !out_scores))) {
        set_error("tav_range_fetch: invalid argument");
        return TAV_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lock(ix->mu);
    if (ix->range_replaced) {
        set_error("tav_range_fetch: a tav_range_search_into replaced the hits of the last range search");
        return TAV_ERR_STATE;
    }
    if (first + n > ix->range_total) {
        set_error("tav_range_fetch: hits [%lld, %lld) out of range (the last range search has %lld)", (long long)first,
                  (long long)(first + n), (long long)ix->range_total);
        return TAV_ERR_RANGE;
    }
    if (n == 0) return TAV_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (int rc = enter_stream(ix, s)) return rc;  // after the range search that wrote the hits
    const cudaMemcpyKind kind = (flags & TAV_OUTPUTS_ON_DEVICE) ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    TAV_CUDA(cudaMemcpyAsync(out_items, static_cast<const int64_t*>(ix->range_items.p) + first,
                             static_cast<size_t>(n) * sizeof(int64_t), kind, s));
    TAV_CUDA(cudaMemcpyAsync(out_scores, static_cast<const float*>(ix->range_scores.p) + first,
                             static_cast<size_t>(n) * sizeof(float), kind, s));
    if (flags & TAV_OUTPUTS_ON_DEVICE) return mark_queued(ix, s);
    TAV_CUDA(cudaStreamSynchronize(s));
    mark_done(ix);
    return TAV_OK;
}

// ---- grouped lookups: the k best groups of rows, each scored by its best row ------------------------------
int tav_set_row_groups(tav_index* ix, const int32_t* groups, int64_t n_rows, int on_device, void* stream) {
    if (!ix || n_rows < 0 || (n_rows > 0 && !groups)) {
        set_error("tav_set_row_groups: invalid argument");
        return TAV_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lock(ix->mu);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (int rc = enter_stream(ix, s)) return rc;  // queued searches read the old map
    if (int rc = finish_pending(ix, s, nullptr)) return rc;
    if (n_rows == 0) {
        ix->group_rows = 0;
        return TAV_OK;
    }
    if (n_rows != ix->size) {
        set_error("tav_set_row_groups: %lld groups for an index of %lld rows", (long long)n_rows, (long long)ix->size);
        return TAV_ERR_INVALID;
    }
    // into the stage, checked there: a refused map leaves the current one in place
    const size_t bytes = static_cast<size_t>(n_rows) * sizeof(int32_t);
    TAV_CUDA(ix->group_stage.ensure(bytes));
    TAV_CUDA(ix->group_stat.ensure(2 * sizeof(uint64_t)));
    TAV_CUDA(cudaMemcpyAsync(ix->group_stage.p, groups, bytes,
                             on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, s));
    TAV_CUDA(cudaMemsetAsync(ix->group_stat.p, 0, 2 * sizeof(uint64_t), s));
    TAV_CUDA(launch_group_check(static_cast<const int32_t*>(ix->group_stage.p), n_rows,
                                static_cast<uint64_t*>(ix->group_stat.p), s));
    uint64_t stat[2] = {0, 0};
    TAV_CUDA(cudaMemcpyAsync(stat, ix->group_stat.p, sizeof(stat), cudaMemcpyDeviceToHost, s));
    TAV_CUDA(cudaStreamSynchronize(s));
    mark_done(ix);
    if (stat[0]) {
        set_error("tav_set_row_groups: a group is negative (groups must lie in [0, 2^31))");
        return TAV_ERR_INVALID;
    }
    std::swap(ix->group_map, ix->group_stage);
    ix->group_rows = n_rows;
    ix->group_runs = static_cast<int64_t>(stat[1]);
    return TAV_OK;
}

static int check_groups(const tav_index* ix, const char* fn) {
    if (ix->group_rows == 0 || ix->group_rows != ix->size) {
        set_error("%s: no current group map (tav_set_row_groups after the last change of the rows)", fn);
        return TAV_ERR_STATE;
    }
    return TAV_OK;
}

constexpr int kGroupFlags = TAV_QUERIES_ON_DEVICE | TAV_OUTPUTS_ON_DEVICE | TAV_FORCE_SCAN | TAV_FORCE_MMA |
                            TAV_USE_ROW_MASK | TAV_USE_QUERY_MASKS | TAV_TIES_LOW_FIRST;

// The grouped threshold search of nq device queries: the leaders in ix->range_items (rows) / range_scores and their
// groups in ix->range_groups, CSR offsets[nq + 1] on the host.
static int range_groups_core(tav_index* ix, TimedSearch* ts, bool timing, const float* d_queries, int nq, float floor,
                             const uint32_t* d_mask, const QueryMasks& qm, int ties_low, int64_t expected_hits,
                             bool use_mma, std::vector<int64_t>& offsets, cudaStream_t s) {
    if (int rc = range_core(ix, ts, timing, d_queries, nq, floor, nullptr, ix->size, 0, d_mask, ties_low, expected_hits,
                            use_mma, offsets, s, 0, qm, true))
        return rc;
    const int64_t total = offsets[nq];
    if (int rc = range_alloc(ix->range_groups, static_cast<size_t>(total) * sizeof(int64_t), "the hit groups")) return rc;
    TAV_CUDA(launch_group_decode(total, static_cast<const int64_t*>(ix->range_items.p),
                                 static_cast<const int32_t*>(ix->group_map.p), static_cast<int64_t*>(ix->range_groups.p), s));
    ts->launches += total > 0;
    return TAV_OK;
}

int tav_range_search_groups(tav_index* ix, const float* queries, int n_queries, float min_score, int flags,
                            int64_t expected_hits, int64_t* out_offsets, void* stream) {
    if (!ix || n_queries < 0 || expected_hits < 0 || !out_offsets || (n_queries > 0 && !queries) ||
        (flags & ~kGroupFlags)) {
        set_error("tav_range_search_groups: invalid argument");
        return TAV_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lock(ix->mu);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (int rc = enter_stream(ix, s)) return rc;  // (also: a queued fetch reads the hits replaced here)
    const bool q_dev = flags & TAV_QUERIES_ON_DEVICE, o_dev = flags & TAV_OUTPUTS_ON_DEVICE;
    ix->range_total = 0;
    ix->range_grouped = false;
    ix->range_replaced = false;
    std::vector<int64_t> offsets(static_cast<size_t>(n_queries) + 1, 0);
    const uint32_t* d_mask = nullptr;
    QueryMasks qm;
    if (int rc = resolve_masks(ix, "tav_range_search_groups", n_queries, flags, false, &d_mask, &qm)) return rc;
    if (ix->size > 0)
        if (int rc = check_groups(ix, "tav_range_search_groups")) return rc;
    if (n_queries == 0 || ix->size == 0 || ix->dim == 0 || min_score != min_score)
        return deliver_offsets(ix, offsets, out_offsets, o_dev, s);
    if (ix->size > 0xFFFFFFFFll) {
        set_error("tav_range_search_groups: more than 2^32 rows per index are not supported; shard the corpus");
        return TAV_ERR_INVALID;
    }
    bool use_mma = false;
    if (int rc = range_path(ix, "tav_range_search_groups", n_queries, flags, false, &use_mma)) return rc;
    TimedSearch* ts = begin_search(ix, use_mma ? (ix->dtype == TAV_F32 ? 3 : 2) : 1);
    const bool timing = ts != &ix->untimed;
    const float* d_queries = nullptr;
    const int64_t* d_subset = nullptr;
    if (int rc = stage_inputs(ix, ts, timing, queries, n_queries, q_dev, false, nullptr, 0, &d_queries, &d_subset, s))
        return rc;
    if (int rc = range_groups_core(ix, ts, timing, d_queries, n_queries, min_score, d_mask, qm,
                                   (flags & TAV_TIES_LOW_FIRST) ? 1 : 0, expected_hits, use_mma, offsets, s))
        return rc;
    if (int rc = end_search(ix, ts, s)) return rc;
    ix->range_total = offsets[n_queries];
    ix->range_grouped = true;
    return deliver_offsets(ix, offsets, out_offsets, o_dev, s);
}

int tav_range_fetch_groups(tav_index* ix, int64_t first, int64_t n, int64_t* out_groups, float* out_scores,
                           int64_t* out_rows, int flags, void* stream) {
    if (!ix || first < 0 || n < 0 || (n > 0 && (!out_groups || !out_scores || !out_rows)) ||
        (flags & ~TAV_OUTPUTS_ON_DEVICE)) {
        set_error("tav_range_fetch_groups: invalid argument");
        return TAV_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lock(ix->mu);
    if (!ix->range_grouped) {
        set_error("tav_range_fetch_groups: the last threshold search was not a tav_range_search_groups");
        return TAV_ERR_STATE;
    }
    if (first + n > ix->range_total) {
        set_error("tav_range_fetch_groups: leaders [%lld, %lld) out of range (the last grouped search has %lld)",
                  (long long)first, (long long)(first + n), (long long)ix->range_total);
        return TAV_ERR_RANGE;
    }
    if (n == 0) return TAV_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (int rc = enter_stream(ix, s)) return rc;  // after the search that wrote the leaders
    const cudaMemcpyKind kind = (flags & TAV_OUTPUTS_ON_DEVICE) ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    TAV_CUDA(cudaMemcpyAsync(out_groups, static_cast<const int64_t*>(ix->range_groups.p) + first,
                             static_cast<size_t>(n) * sizeof(int64_t), kind, s));
    TAV_CUDA(cudaMemcpyAsync(out_scores, static_cast<const float*>(ix->range_scores.p) + first,
                             static_cast<size_t>(n) * sizeof(float), kind, s));
    TAV_CUDA(cudaMemcpyAsync(out_rows, static_cast<const int64_t*>(ix->range_items.p) + first,
                             static_cast<size_t>(n) * sizeof(int64_t), kind, s));
    if (flags & TAV_OUTPUTS_ON_DEVICE) return mark_queued(ix, s);
    TAV_CUDA(cudaStreamSynchronize(s));
    mark_done(ix);
    return TAV_OK;
}

// [nq, k] of grouped results from CSR leaders in ix->range_items / range_scores (host offsets), rows [q0, q0 + nq)
// of the result arrays: the first min(k, leaders) of each query, then group -1, score 0, row -1
static int group_layout(tav_index* ix, const std::vector<int64_t>& offsets, int k, int q0, int64_t* groups,
                        float* scores, int64_t* rows, int32_t* counts, cudaStream_t s) {
    const int nq = static_cast<int>(offsets.size()) - 1;
    if (int rc = range_alloc(ix->group_csr, offsets.size() * sizeof(int64_t), "the leader offsets")) return rc;
    // from pageable memory: consumed when the call returns
    TAV_CUDA(cudaMemcpyAsync(ix->group_csr.p, offsets.data(), offsets.size() * sizeof(int64_t), cudaMemcpyHostToDevice, s));
    const size_t at = static_cast<size_t>(q0) * k;
    TAV_CUDA(launch_subset_topk_layout(nq, k, static_cast<const int64_t*>(ix->group_csr.p),
                                       static_cast<const int64_t*>(ix->range_items.p),
                                       static_cast<const float*>(ix->range_scores.p), rows + at, scores + at, counts + q0, s));
    TAV_CUDA(launch_group_decode(static_cast<int64_t>(nq) * k, rows + at, static_cast<const int32_t*>(ix->group_map.p),
                                 groups + at, s));
    return TAV_OK;
}

int tav_search_groups(tav_index* ix, const float* queries, int n_queries, int k, float min_score, int flags,
                      int64_t* out_groups, float* out_scores, int64_t* out_rows, int32_t* out_counts, void* stream,
                      int* redone) {
    if (!ix || n_queries < 0 || k < 1 || (flags & ~kGroupFlags) ||
        (n_queries > 0 && (!queries || !out_groups || !out_scores || !out_rows || !out_counts))) {
        set_error("tav_search_groups: invalid argument (k must be >= 1)");
        return TAV_ERR_INVALID;
    }
    if (redone) *redone = 0;
    if (n_queries == 0) return TAV_OK;
    std::lock_guard<std::mutex> lock(ix->mu);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (int rc = enter_stream(ix, s)) return rc;
    const bool q_dev = flags & TAV_QUERIES_ON_DEVICE, o_dev = flags & TAV_OUTPUTS_ON_DEVICE;
    const int ties_low = (flags & TAV_TIES_LOW_FIRST) ? 1 : 0;
    const uint32_t* d_mask = nullptr;
    QueryMasks qm;
    if (int rc = resolve_masks(ix, "tav_search_groups", n_queries, flags, false, &d_mask, &qm)) return rc;
    if (ix->size > 0)
        if (int rc = check_groups(ix, "tav_search_groups")) return rc;
    if (ix->size > 0xFFFFFFFFll) {
        set_error("tav_search_groups: more than 2^32 rows per index are not supported; shard the corpus");
        return TAV_ERR_INVALID;
    }
    // the results on the device: the caller's arrays, or a staging of [groups | rows | scores | counts]
    const size_t nk = static_cast<size_t>(n_queries) * k;
    int64_t *groups = out_groups, *rows = out_rows;
    float* scores = out_scores;
    int32_t* counts = out_counts;
    if (!o_dev) {
        TAV_CUDA(ix->group_res.ensure(nk * (2 * sizeof(int64_t) + sizeof(float)) + n_queries * sizeof(int32_t)));
        groups = static_cast<int64_t*>(ix->group_res.p);
        rows = groups + nk;
        scores = reinterpret_cast<float*>(rows + nk);
        counts = reinterpret_cast<int32_t*>(scores + nk);
    }
    int n_redone = 0;
    if (ix->size == 0 || ix->dim == 0 || min_score != min_score) {  // no hits
        TAV_CUDA(cudaMemsetAsync(groups, 0xFF, nk * sizeof(int64_t), s));
        TAV_CUDA(cudaMemsetAsync(rows, 0xFF, nk * sizeof(int64_t), s));
        TAV_CUDA(cudaMemsetAsync(scores, 0, nk * sizeof(float), s));
        TAV_CUDA(cudaMemsetAsync(counts, 0, n_queries * sizeof(int32_t), s));
    } else {
        // The top-kp prefix of the hit list: its groups' first rows are the first leaders of the whole list, so
        // a query whose prefix is all of its hits, or holds k groups, is answered exactly by the prefix.  kp is k
        // times the rows per run of equal group ids (the map's mean multiplicity for contiguous groups), at most one
        // pass of the top-k kernels.  A prefix that covers the rows is the grouped threshold search itself.
        const int64_t mult = std::max<int64_t>(1, (ix->size + ix->group_runs - 1) / std::max<int64_t>(1, ix->group_runs));
        const int64_t kp = std::min<int64_t>(ix->size, std::max<int64_t>(k, std::min<int64_t>(kPassK, k * mult)));
        const bool prefix = kp < ix->size && !((flags & TAV_FORCE_MMA) && kp > kPassK);
        ix->range_total = 0;  // the leaders pass through the threshold search's buffers
        ix->range_grouped = false;
        ix->range_replaced = false;
        TimedSearch aux;  // the prefix search keeps the timing record; the steps after it are not timed
        std::vector<int64_t> offsets;
        std::vector<int> flagged;
        if (prefix) {
            const size_t nkp = static_cast<size_t>(n_queries) * kp;
            TAV_CUDA(ix->group_topk.ensure(nkp * (sizeof(int64_t) + sizeof(float)) + n_queries * sizeof(int32_t)));
            int64_t* p_rows = static_cast<int64_t*>(ix->group_topk.p);
            float* p_scores = reinterpret_cast<float*>(p_rows + nkp);
            int32_t* p_counts = reinterpret_cast<int32_t*>(p_scores + nkp);
            if (int rc = search_locked(ix, queries, n_queries, static_cast<int>(kp), min_score,
                                       flags | TAV_OUTPUTS_ON_DEVICE, nullptr, 0, 0,
                                       p_rows, p_scores, p_counts, stream))
                return rc;
            if (int rc = range_alloc(ix->group_keys, nkp * sizeof(uint64_t), "the prefix keys")) return rc;
            uint64_t* keys = static_cast<uint64_t*>(ix->group_keys.p);
            TAV_CUDA(launch_topk_keys(n_queries, static_cast<int>(kp), p_rows, p_scores, p_counts, ties_low, keys, s));
            std::vector<int32_t> cnt(static_cast<size_t>(n_queries));
            TAV_CUDA(cudaMemcpyAsync(cnt.data(), p_counts, cnt.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
            TAV_CUDA(cudaStreamSynchronize(s));
            std::vector<SortSeg> segs(static_cast<size_t>(n_queries));
            for (int q = 0; q < n_queries; ++q) {
                segs[q].keys = keys + static_cast<size_t>(q) * kp;
                segs[q].n = cnt[q];
            }
            if (int rc = reduce_leaders(ix, &aux, false, segs, offsets, ties_low, s)) return rc;
            for (int q = 0; q < n_queries; ++q)
                if (cnt[q] == kp && offsets[q + 1] - offsets[q] < k) flagged.push_back(q);
            if (int rc = range_sort(ix, &aux, false, segs, offsets[n_queries], nullptr, 0, ties_low, s)) return rc;
        } else {
            bool use_mma = false;
            if (int rc = range_path(ix, "tav_search_groups", n_queries, flags, false, &use_mma)) return rc;
            TimedSearch* ts = begin_search(ix, use_mma ? (ix->dtype == TAV_F32 ? 3 : 2) : 1);
            const bool timing = ts != &ix->untimed;
            const float* d_q = nullptr;
            const int64_t* d_sub = nullptr;
            if (int rc = stage_inputs(ix, ts, timing, queries, n_queries, q_dev, false, nullptr, 0, &d_q, &d_sub, s))
                return rc;
            if (int rc = range_groups_core(ix, ts, timing, d_q, n_queries, min_score, d_mask, qm, ties_low, 0, use_mma,
                                           offsets, s))
                return rc;
            if (int rc = end_search(ix, ts, s)) return rc;
        }
        if (int rc = group_layout(ix, offsets, k, 0, groups, scores, rows, counts, s)) return rc;
        // a query whose prefix held fewer than k groups: its grouped threshold search, alone (the row scan), cut to k
        for (int q : flagged) {
            const float* d_q = nullptr;
            const int64_t* d_sub = nullptr;
            if (int rc = stage_inputs(ix, &aux, false, queries + static_cast<size_t>(q) * ix->dim, 1, q_dev, false,
                                      nullptr, 0, &d_q, &d_sub, s))
                return rc;
            const uint32_t* mask = qm.bits ? qm.bits + static_cast<size_t>(q) * qm.stride : d_mask;
            std::vector<int64_t> off1;
            if (int rc = range_groups_core(ix, &aux, false, d_q, 1, min_score, mask, QueryMasks{}, ties_low, 0, false,
                                           off1, s))
                return rc;
            if (int rc = group_layout(ix, off1, k, q, groups, scores, rows, counts, s)) return rc;
        }
        n_redone = static_cast<int>(flagged.size());
        ix->range_total = 0;
        ix->range_grouped = false;
    }
    if (redone) *redone = n_redone;
    if (o_dev) return mark_queued(ix, s);
    TAV_CUDA(cudaMemcpyAsync(out_groups, groups, nk * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    TAV_CUDA(cudaMemcpyAsync(out_rows, rows, nk * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    TAV_CUDA(cudaMemcpyAsync(out_scores, scores, nk * sizeof(float), cudaMemcpyDeviceToHost, s));
    TAV_CUDA(cudaMemcpyAsync(out_counts, counts, n_queries * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    TAV_CUDA(cudaStreamSynchronize(s));
    mark_done(ix);
    return TAV_OK;
}

int tav_range_search_into(tav_index* ix, const float* queries, int n_queries, float min_score, int flags,
                          const int64_t* subset, int64_t subset_len, int64_t item_offset, int64_t expected_hits,
                          int64_t capacity, int64_t* out_offsets, int64_t* out_items, float* out_scores, void* stream) {
    constexpr int kAccepted = TAV_QUERIES_ON_DEVICE | TAV_FORCE_SCAN | TAV_FORCE_MMA | TAV_USE_ROW_MASK |
                              TAV_USE_QUERY_MASKS | TAV_TIES_LOW_FIRST | TAV_DEFER_RETRY;
    if (!ix || n_queries < 0 || expected_hits < 0 || capacity < 0 || (flags & ~kAccepted) || !out_offsets ||
        (n_queries > 0 && !queries) || (capacity > 0 && (!out_items || !out_scores))) {
        set_error("tav_range_search_into: invalid argument");
        return TAV_ERR_INVALID;
    }
    if (int rc = check_subset_args("tav_range_search_into", flags, subset, subset_len, false)) return rc;
    std::lock_guard<std::mutex> lock(ix->mu);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (int rc = enter_stream(ix, s)) return rc;
    const bool q_dev = flags & TAV_QUERIES_ON_DEVICE, defer = flags & TAV_DEFER_RETRY;
    ix->range_total = 0;  // the hits of the last tav_range_search are given up (the sort scratch is reused)
    ix->range_grouped = false;
    ix->range_replaced = true;
    const uint32_t* d_mask = nullptr;
    QueryMasks qm;
    if (int rc = resolve_masks(ix, "tav_range_search_into", n_queries, flags, subset != nullptr, &d_mask, &qm)) return rc;
    const int64_t n_scan = subset ? subset_len : ix->size;
    // NaN min_score, empty corpus or empty subset: no hits
    if (n_queries == 0 || n_scan == 0 || ix->size == 0 || ix->dim == 0 || min_score != min_score) {
        TAV_CUDA(cudaMemsetAsync(out_offsets, 0, (static_cast<size_t>(n_queries) + 1) * sizeof(int64_t), s));
        return mark_queued(ix, s);
    }
    if (n_scan > 0xFFFFFFFFll) {
        set_error("tav_range_search_into: more than 2^32 rows per index are not supported; shard the corpus");
        return TAV_ERR_INVALID;
    }
    if (int rc = check_subset_ordinals(ix, subset, subset_len)) return rc;
    // path choice as in tav_range_search
    const bool mma_able = (mma_supported(ix->dtype, ix->dim) || (ix->dtype == TAV_F32 && mma_split_supported(ix->dim))) &&
                          !subset && n_queries <= kMmaMaxQueries && ix->size < (1ll << 31);
    bool use_mma = !(flags & TAV_FORCE_SCAN) && mma_able &&
                   ((flags & TAV_FORCE_MMA) || (n_queries >= 16 && ix->size >= 4096));
    if ((flags & TAV_FORCE_MMA) && !use_mma) {
        set_error("tav_range_search_into: TAV_FORCE_MMA needs dim %% 8 == 0, no subset, at most %d queries", kMmaMaxQueries);
        return TAV_ERR_INVALID;
    }
    // bookkeeping slot (flags and flagged count of the plan), as for deferred top-k searches
    if (int rc = ensure_retry(ix, n_queries, n_queries, s)) return rc;
    if (static_cast<int>(ix->pending.size()) >= kMaxPending)
        if (int rc = finish_pending(ix, s, nullptr)) return rc;
    // a deferred search reads its queries and subset again at tav_finish_search: staged ones are held until then
    float* held_q = nullptr;
    int64_t* held_sub = nullptr;
    size_t held_end = 0;
    if (defer && (!q_dev || (ix->flags & TAV_NORMALIZE))) {
        void* r = nullptr;
        if (int rc = hold_region(ix, static_cast<size_t>(n_queries) * ix->dim * sizeof(float), &r, &held_end)) return rc;
        held_q = static_cast<float*>(r);
    }
    if (defer && subset) {
        void* r = nullptr;
        if (int rc = hold_region(ix, static_cast<size_t>(subset_len) * sizeof(int64_t), &r, &held_end)) return rc;
        held_sub = static_cast<int64_t*>(r);
    }
    TimedSearch* ts = begin_search(ix, use_mma ? (ix->dtype == TAV_F32 ? 3 : 2) : 1);
    const bool timing = ts != &ix->untimed;
    const float* d_queries = nullptr;
    const int64_t* d_subset = nullptr;
    if (int rc = stage_inputs(ix, ts, timing, queries, n_queries, q_dev, true, subset, subset_len, &d_queries, &d_subset, s,
                              held_q))
        return rc;
    if (held_sub) {
        TAV_CUDA(cudaMemcpyAsync(held_sub, d_subset, static_cast<size_t>(subset_len) * sizeof(int64_t),
                                 cudaMemcpyDeviceToDevice, s));
        d_subset = held_sub;
    }
    const int slot = ix->next_slot++;
    const int ties_low = (flags & TAV_TIES_LOW_FIRST) ? 1 : 0;
    const RangeOut out{out_offsets, out_items, out_scores, capacity};
    int per_chunk = 0, n_seg = 0;
    int rc = range_into_core(ix, ts, timing, d_queries, n_queries, min_score, d_subset, n_scan, item_offset, d_mask, qm,
                             ties_low, expected_hits, use_mma, slot, true, out, &per_chunk, &n_seg, s);
    if (rc == kRangeUseScan) {
        use_mma = false;
        ts->path = 1;
        rc = range_into_core(ix, ts, timing, d_queries, n_queries, min_score, d_subset, n_scan, item_offset, d_mask, qm,
                             ties_low, expected_hits, false, slot, true, out, &per_chunk, &n_seg, s);
    }
    if (rc == TAV_OK) rc = end_search(ix, ts, s);
    if (rc != TAV_OK) {
        // the slot goes back, clean: a kernel this call queued may have written its totals (the error stands)
        cudaStreamSynchronize(s);
        cudaMemset(retry_totals(ix, slot), 0, 2 * sizeof(int32_t));
        static_cast<int32_t*>(ix->retry_host.p)[2 * slot] = static_cast<int32_t*>(ix->retry_host.p)[2 * slot + 1] = 0;
        --ix->next_slot;
        return rc;
    }
    Pending p{d_queries, n_queries, 0, min_score, item_offset, out_items, out_scores, nullptr, slot,
              use_mma && ix->dtype == TAV_F32, qm.bits ? qm.bits : d_mask, qm.bits ? qm.stride : 0};
    p.offsets = out_offsets;
    p.cap = capacity;
    p.subset = d_subset;
    p.n_scan = n_scan;
    p.ties_low = ties_low;
    p.expected_hits = expected_hits;
    p.qm = qm;
    p.per_chunk = per_chunk;
    p.n_seg = n_seg;
    ix->pending.push_back(p);
    if (!defer) return finish_pending(ix, s, nullptr);  // redoes what the plan flagged now; synchronises s
    return mark_queued(ix, s);
}

}  // extern "C"

// ---- per-query subsets (tav_search_subsets, tav_range_search_subsets) ------------------------------------
constexpr int kSubsetsFlags = TAV_QUERIES_ON_DEVICE | TAV_OUTPUTS_ON_DEVICE | TAV_TIES_LOW_FIRST | TAV_ITEMS_AS_POSITIONS;

// the argument checks of both entry points that need no index state
static int check_subsets(const char* fn, int n_queries, int flags, const int64_t* offsets, const int64_t* ordinals) {
    if (flags & ~kSubsetsFlags) {
        set_error("%s: flags 0x%x are not available with per-query subsets", fn, flags & ~kSubsetsFlags);
        return TAV_ERR_INVALID;
    }
    if (!offsets || offsets[0] != 0) {
        set_error("%s: offsets must be n_queries + 1 values starting at 0", fn);
        return TAV_ERR_INVALID;
    }
    for (int q = 0; q < n_queries; ++q)
        if (offsets[q + 1] < offsets[q]) {
            set_error("%s: offsets decrease at query %d", fn, q);
            return TAV_ERR_INVALID;
        }
    if (offsets[n_queries] > 0xFFFFFFFFll) {  // flat positions live in the low word of a key
        set_error("%s: %lld ordinals; at most 2^32 - 1 per call", fn, (long long)offsets[n_queries]);
        return TAV_ERR_INVALID;
    }
    if (offsets[n_queries] > 0 && !ordinals) {
        set_error("%s: ordinals is NULL", fn);
        return TAV_ERR_INVALID;
    }
    return TAV_OK;
}

// Every entry of every query's subset scored in one gather, each query's admitted keys sorted: the hits in CSR
// order in ix->range_items / range_scores, csr[nq + 1] on the host.  Synchronises once, to learn the counts.
static int subsets_core(tav_index* ix, TimedSearch* ts, bool timing, const float* queries, int nq, int flags,
                        float floor, const int64_t* offsets, const int64_t* ordinals, std::vector<int64_t>& csr,
                        cudaStream_t s) {
    const bool q_dev = flags & TAV_QUERIES_ON_DEVICE;
    const int ties_low = (flags & TAV_TIES_LOW_FIRST) && TAV_SUBSETS_MUTANT != 3 ? 1 : 0;
    const int positions = (flags & TAV_ITEMS_AS_POSITIONS) ? 1 : 0;
    if (scan_collect_max_queries(ix->dim) < 1) {  // one query row in shared memory, as the row scan stages it
        set_error("per-query subsets: embedding size %d too large for the row-scan kernel", ix->dim);
        return TAV_ERR_INVALID;
    }
    const int64_t total = offsets[nq];
#if TAV_SUBSETS_MUTANT == 2
    std::vector<int64_t> wrapped(ordinals, ordinals + total);
    for (int64_t& o : wrapped)
        if (o < 0) o += ix->size;
    ordinals = wrapped.data();
#endif
    const float* d_queries = nullptr;
    const int64_t* d_ordinals = nullptr;
    if (int rc = stage_inputs(ix, ts, timing, queries, nq, q_dev, false, ordinals, total, &d_queries, &d_ordinals, s))
        return rc;
    // device [offsets | work0 | csr]: query q's work items (tiles of its entries) are [work0[q], work0[q + 1])
    const size_t n1 = static_cast<size_t>(nq) + 1;
    std::vector<int64_t> meta(2 * n1);
    memcpy(meta.data(), offsets, n1 * sizeof(int64_t));
    int64_t* work0 = meta.data() + n1;
    work0[0] = 0;
    for (int q = 0; q < nq; ++q) work0[q + 1] = work0[q] + (offsets[q + 1] - offsets[q] + kSubsetTile - 1) / kSubsetTile;
    if (int rc = range_alloc(ix->subsets_meta, 3 * n1 * sizeof(int64_t), "the subset offsets")) return rc;
    int64_t* d_meta = static_cast<int64_t*>(ix->subsets_meta.p);
    // from pageable memory: consumed when the call returns
    TAV_CUDA(cudaMemcpyAsync(d_meta, meta.data(), meta.size() * sizeof(int64_t), cudaMemcpyHostToDevice, s));
    if (int rc = range_alloc(ix->range_keys, static_cast<size_t>(total) * sizeof(uint64_t), "the hit regions")) return rc;
    if (int rc = range_alloc(ix->range_counts, static_cast<size_t>(nq) * sizeof(uint32_t), "the hit counters")) return rc;
    uint32_t* d_counts = static_cast<uint32_t*>(ix->range_counts.p);
    uint64_t* keys = static_cast<uint64_t*>(ix->range_keys.p);
    TAV_CUDA(cudaMemsetAsync(d_counts, 0, static_cast<size_t>(nq) * sizeof(uint32_t), s));

    SubsetArgs a{};
    a.corpus = ix->rows;
    a.dtype = ix->dtype;
    a.n_corpus = ix->size;
    a.dim = ix->dim;
    a.queries = d_queries;
    a.nq = nq;
    a.ordinals = d_ordinals;
    a.offsets = d_meta;
    a.work0 = d_meta + n1;
    a.n_work = work0[nq];
    a.floor_score = floor;
    a.ties_low = ties_low;
    a.keys = keys;
    a.counts = d_counts;
    TAV_CUDA(timed_launch(ix, ts, timing, 0, s, [&] { return launch_subset_gather(a, s); }));
    ts->launches += 1;

    std::vector<uint32_t> cnt(static_cast<size_t>(nq));
    TAV_CUDA(cudaMemcpyAsync(cnt.data(), d_counts, cnt.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    TAV_CUDA(cudaStreamSynchronize(s));
    csr.assign(n1, 0);
    std::vector<SortSeg> segs(static_cast<size_t>(nq));
    for (int q = 0; q < nq; ++q) {
        csr[q + 1] = csr[q] + cnt[q];
        segs[q].keys = keys + offsets[q];
        segs[q].out = csr[q];
        segs[q].n = cnt[q];
    }
    return range_sort(ix, ts, timing, segs, csr[nq], positions ? nullptr : d_ordinals, 0, ties_low, s);
}

// ---- per-query subsets from device memory (tav_search_subsets_into, tav_range_search_subsets_into) -----------
// The same gather and sort as above with no host round trip: the offsets are checked and the work items planned on
// the device (subset_plan_kernel), the gather runs over an upper bound of the items and range-checks every ordinal,
// and the sort is planned on the device (range_plan_subsets_kernel) and launched over upper bounds.  A refusal sets
// the search's status word: no work is planned (offsets) or no row address is formed from the ordinal, and the plan
// of the sort then gives every query 0 hits.
constexpr int kSubsetsIntoFlags = kSubsetsFlags | TAV_DEFER_RETRY;

// k > 0: the top-k form (its CSR hits in ix->range_items / range_scores, laid out into items / scores / counts);
// k == 0: the threshold form into `out`.  The caller has checked the arguments and entered s; B, the entries, the
// rows and min_score are not empty.
static int subsets_into(tav_index* ix, const char* fn, const float* queries, int nq, int k, float floor, int flags,
                        const int64_t* offsets, const int64_t* ordinals, int64_t n_ord, RangeOut out, int64_t* items,
                        float* scores, int32_t* counts, cudaStream_t s) {
    if (scan_collect_max_queries(ix->dim) < 1) {  // one query row in shared memory, as the row scan stages it
        set_error("%s: embedding size %d too large for the row-scan kernel", fn, ix->dim);
        return TAV_ERR_INVALID;
    }
    const bool defer = flags & TAV_DEFER_RETRY;
    const int ties_low = (flags & TAV_TIES_LOW_FIRST) ? 1 : 0;
    const int positions = (flags & TAV_ITEMS_AS_POSITIONS) ? 1 : 0;
    if (!ix->subsets_status.p) {
        TAV_CUDA(ix->subsets_status.ensure((kMaxPending + 1) * sizeof(int)));
        TAV_CUDA(cudaMemsetAsync(ix->subsets_status.p, 0, (kMaxPending + 1) * sizeof(int), s));
    }
    int slot = kMaxPending;  // the synchronous form's word
    float* held = nullptr;
    if (defer) {
        // a bookkeeping slot (its status word), as for the other deferred searches; nothing is redone at the finish
        if (int rc = ensure_retry(ix, 0, 0, s)) return rc;
        if (static_cast<int>(ix->pending.size()) >= kMaxPending)
            if (int rc = finish_pending(ix, s, nullptr)) return rc;
        if (ix->flags & TAV_NORMALIZE) {  // the normalised queries stay the search's own until the finish
            void* r = nullptr;
            size_t end = 0;
            if (int rc = hold_region(ix, static_cast<size_t>(nq) * ix->dim * sizeof(float), &r, &end)) return rc;
            held = static_cast<float*>(r);
        }
        slot = ix->next_slot++;
    }
    int* status = static_cast<int*>(ix->subsets_status.p) + slot;
    auto run = [&]() -> int {
        TimedSearch* ts = begin_search(ix, 1);
        const bool timing = ts != &ix->untimed;
        const float* d_queries = nullptr;
        const int64_t* no_subset = nullptr;
        if (int rc = stage_inputs(ix, ts, timing, queries, nq, true, true, nullptr, 0, &d_queries, &no_subset, s, held))
            return rc;
        ix->range_total = 0;  // the hits of the last tav_range_search are given up (the sort scratch is reused)
        ix->range_grouped = false;
        ix->range_replaced = true;
        // device [work0 | CSR offsets of the top-k form's hits | planned work items]
        const size_t n1 = static_cast<size_t>(nq) + 1;
        if (int rc = range_alloc(ix->subsets_meta, (2 * n1 + 1) * sizeof(int64_t), "the subset plan")) return rc;
        int64_t* work0 = static_cast<int64_t*>(ix->subsets_meta.p);
        int64_t* n_work = work0 + 2 * n1;
        if (k > 0) {
            if (int rc = range_alloc(ix->range_items, static_cast<size_t>(n_ord) * sizeof(int64_t), "the hits")) return rc;
            if (int rc = range_alloc(ix->range_scores, static_cast<size_t>(n_ord) * sizeof(float), "the hit scores"))
                return rc;
            out = RangeOut{work0 + n1, static_cast<int64_t*>(ix->range_items.p), static_cast<float*>(ix->range_scores.p),
                           n_ord};
        }
        if (int rc = range_alloc(ix->range_keys, static_cast<size_t>(n_ord) * sizeof(uint64_t), "the hit regions")) return rc;
        if (int rc = range_alloc(ix->range_counts, static_cast<size_t>(nq) * sizeof(uint32_t), "the hit counters")) return rc;
        uint32_t* d_counts = static_cast<uint32_t*>(ix->range_counts.p);
        uint64_t* keys = static_cast<uint64_t*>(ix->range_keys.p);
        TAV_CUDA(cudaMemsetAsync(status, 0, sizeof(int), s));
        TAV_CUDA(cudaMemsetAsync(d_counts, 0, static_cast<size_t>(nq) * sizeof(uint32_t), s));

        const SubsetPlanArgs pl{nq, offsets, n_ord, work0, n_work, status};
        TAV_CUDA(timed_launch(ix, ts, timing, 2, s, [&] { return launch_subset_plan(pl, s); }));
        ts->launches += 1;
        SubsetArgs a{};
        a.corpus = ix->rows;
        a.dtype = ix->dtype;
        a.n_corpus = ix->size;
        a.dim = ix->dim;
        a.queries = d_queries;
        a.nq = nq;
        a.ordinals = ordinals;
        a.offsets = offsets;
        a.work0 = work0;
        a.n_work = (n_ord + kSubsetTile - 1) / kSubsetTile + nq;  // >= the planned items (one partial tile per query)
        a.floor_score = floor;
        a.ties_low = ties_low;
        a.keys = keys;
        a.counts = d_counts;
        TAV_CUDA(timed_launch(ix, ts, timing, 0, s, [&] { return launch_subset_gather_dev(a, n_work, status, s); }));
        ts->launches += 1;

        PlanDest dest;
        dest.offsets = out.offsets;
        dest.abandon[0] = status;
        dest.key_off = offsets;
        dest.total_keys = n_ord;
        SortArgs sa;
        const int* sizes = nullptr;
        int64_t* dst_off = nullptr;
        // regions never overflow: fill = count, cap = every count
        if (int rc = range_plan(ix, ts, nq, d_counts, d_counts, 0xFFFFFFFFu, 0, 0, keys, positions ? nullptr : ordinals, 0,
                                ties_low, out, dest, &sa, &sizes, &dst_off, s))
            return rc;
        if (int rc = range_sort_dev(ix, ts, timing, sa, sizes, out.cap, s)) return rc;
        if (k > 0) {
            TAV_CUDA(launch_subset_topk_layout(nq, k, out.offsets, out.items, out.scores, items, scores, counts, s));
            ts->launches += 1;
        }
        return end_search(ix, ts, s);
    };
    if (int rc = run()) {
        if (defer) --ix->next_slot;  // the slot goes back (its status word is cleared by the next search that takes it)
        return rc;
    }
    if (defer) {
        // (the queries as the search read them: normalised into the held region, or the caller's)
        Pending p{held ? held : queries, nq, k, floor, 0, items, scores, counts, slot, false, nullptr, 0};
        p.offsets = k > 0 ? nullptr : out.offsets;
        p.cap = out.cap;
        p.n_scan = ix->size;
        p.subsets_status = status;
        ix->pending.push_back(p);
        return mark_queued(ix, s);
    }
    int st = 0;
    TAV_CUDA(cudaMemcpyAsync(&st, status, sizeof(int), cudaMemcpyDeviceToHost, s));
    TAV_CUDA(cudaStreamSynchronize(s));
    mark_done(ix);
    return st ? subsets_status_error(st, ix->size) : TAV_OK;
}

extern "C" {

int tav_search_subsets(tav_index* ix, const float* queries, int n_queries, int k, float min_score, int flags,
                       const int64_t* offsets, const int64_t* ordinals, int64_t* out_items, float* out_scores,
                       int32_t* out_counts, void* stream) {
    if (!ix || n_queries < 0 || k < 1 || (n_queries > 0 && (!queries || !out_items || !out_scores || !out_counts))) {
        set_error("tav_search_subsets: invalid argument (k must be >= 1)");
        return TAV_ERR_INVALID;
    }
    if (int rc = check_subsets("tav_search_subsets", n_queries, flags, offsets, ordinals)) return rc;
    if (n_queries == 0) return TAV_OK;
    std::lock_guard<std::mutex> lock(ix->mu);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (int rc = enter_stream(ix, s)) return rc;
    const bool o_dev = flags & TAV_OUTPUTS_ON_DEVICE;
    const ResultPack pack(n_queries, k);
    const size_t nk = pack.nk;
    const int64_t total = offsets[n_queries];
    // no entries, no rows or a NaN min_score: no hits (as tav_search, before the ordinals are looked at)
    if (total == 0 || ix->size == 0 || ix->dim == 0 || min_score != min_score) {
        if (o_dev) {
            TAV_CUDA(cudaMemsetAsync(out_items, 0xFF, nk * sizeof(int64_t), s));
            TAV_CUDA(cudaMemsetAsync(out_scores, 0, nk * sizeof(float), s));
            TAV_CUDA(cudaMemsetAsync(out_counts, 0, static_cast<size_t>(n_queries) * sizeof(int32_t), s));
            return mark_queued(ix, s);
        }
        std::fill(out_items, out_items + nk, int64_t(-1));
        std::fill(out_scores, out_scores + nk, 0.0f);
        std::fill(out_counts, out_counts + n_queries, 0);
        return TAV_OK;
    }
    if (int rc = check_subset_ordinals(ix, ordinals, total)) return rc;
    TimedSearch* ts = begin_search(ix, 1);
    const bool timing = ts != &ix->untimed;
    std::vector<int64_t> csr;
    ix->range_total = 0;  // the hits land in the threshold search's buffers
    ix->range_grouped = false;
    ix->range_replaced = false;
    if (int rc = subsets_core(ix, ts, timing, queries, n_queries, flags, min_score, offsets, ordinals, csr, s))
        return rc;
    ix->range_total = csr[n_queries];
    const size_t n1 = static_cast<size_t>(n_queries) + 1;
    int64_t* d_csr = static_cast<int64_t*>(ix->subsets_meta.p) + 2 * n1;
    // from pageable memory: consumed when the call returns
    TAV_CUDA(cudaMemcpyAsync(d_csr, csr.data(), n1 * sizeof(int64_t), cudaMemcpyHostToDevice, s));
    int64_t* d_items = out_items;
    float* d_scores = out_scores;
    int32_t* d_counts = out_counts;
    if (!o_dev) {
        TAV_CUDA(ix->out_pack.ensure(pack.counts_end()));
        pack.place(ix->out_pack.p, &d_items, &d_scores, &d_counts);
    }
    TAV_CUDA(launch_subset_topk_layout(n_queries, k, d_csr, static_cast<const int64_t*>(ix->range_items.p),
                                       static_cast<const float*>(ix->range_scores.p), d_items, d_scores, d_counts, s));
    ts->launches += 1;
    if (int rc = end_search(ix, ts, s)) return rc;
    if (o_dev) return mark_queued(ix, s);
    if (int rc = copy_pack_out(pack, ix->out_pack.p, out_items, out_scores, out_counts, s)) return rc;
    mark_done(ix);
    return TAV_OK;
}

int tav_range_search_subsets(tav_index* ix, const float* queries, int n_queries, float min_score, int flags,
                             const int64_t* offsets, const int64_t* ordinals, int64_t* out_offsets, void* stream) {
    if (!ix || n_queries < 0 || !out_offsets || (n_queries > 0 && !queries)) {
        set_error("tav_range_search_subsets: invalid argument");
        return TAV_ERR_INVALID;
    }
    if (int rc = check_subsets("tav_range_search_subsets", n_queries, flags, offsets, ordinals)) return rc;
    std::lock_guard<std::mutex> lock(ix->mu);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (int rc = enter_stream(ix, s)) return rc;  // (also: a queued tav_range_fetch reads the hits replaced here)
    const int64_t total = offsets[n_queries];
    const bool none = n_queries == 0 || total == 0 || ix->size == 0 || ix->dim == 0 || min_score != min_score;
    if (!none)
        if (int rc = check_subset_ordinals(ix, ordinals, total)) return rc;
    std::vector<int64_t> csr(static_cast<size_t>(n_queries) + 1, 0);
    ix->range_total = 0;
    ix->range_grouped = false;
    ix->range_replaced = false;
    if (!none) {
        TimedSearch* ts = begin_search(ix, 1);
        const bool timing = ts != &ix->untimed;
        if (int rc = subsets_core(ix, ts, timing, queries, n_queries, flags, min_score, offsets, ordinals, csr, s))
            return rc;
        if (int rc = end_search(ix, ts, s)) return rc;
        ix->range_total = csr[n_queries];
    }
    return deliver_offsets(ix, csr, out_offsets, flags & TAV_OUTPUTS_ON_DEVICE, s);
}

int tav_search_subsets_into(tav_index* ix, const float* queries, int n_queries, int k, float min_score, int flags,
                            const int64_t* offsets, const int64_t* ordinals, int64_t n_ordinals, int64_t* out_items,
                            float* out_scores, int32_t* out_counts, void* stream) {
    if (!ix || n_queries < 0 || k < 1 || (flags & ~kSubsetsIntoFlags) || n_ordinals < 0 || n_ordinals > 0xFFFFFFFFll ||
        !offsets || (n_ordinals > 0 && !ordinals) ||
        (n_queries > 0 && (!queries || !out_items || !out_scores || !out_counts))) {
        set_error("tav_search_subsets_into: invalid argument (k >= 1, 0 <= n_ordinals < 2^32, accepted flags)");
        return TAV_ERR_INVALID;
    }
    if (n_queries == 0) return TAV_OK;
    std::lock_guard<std::mutex> lock(ix->mu);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (int rc = enter_stream(ix, s)) return rc;
    // no entries, no rows or a NaN min_score: no hits (the ordinals are not looked at)
    if (n_ordinals == 0 || ix->size == 0 || ix->dim == 0 || min_score != min_score) {
        const size_t nk = static_cast<size_t>(n_queries) * k;
        TAV_CUDA(cudaMemsetAsync(out_items, 0xFF, nk * sizeof(int64_t), s));
        TAV_CUDA(cudaMemsetAsync(out_scores, 0, nk * sizeof(float), s));
        TAV_CUDA(cudaMemsetAsync(out_counts, 0, static_cast<size_t>(n_queries) * sizeof(int32_t), s));
        return mark_queued(ix, s);
    }
    return subsets_into(ix, "tav_search_subsets_into", queries, n_queries, k, min_score, flags, offsets, ordinals,
                        n_ordinals, RangeOut{}, out_items, out_scores, out_counts, s);
}

int tav_range_search_subsets_into(tav_index* ix, const float* queries, int n_queries, float min_score, int flags,
                                  const int64_t* offsets, const int64_t* ordinals, int64_t n_ordinals, int64_t capacity,
                                  int64_t* out_offsets, int64_t* out_items, float* out_scores, void* stream) {
    if (!ix || n_queries < 0 || (flags & ~kSubsetsIntoFlags) || n_ordinals < 0 || n_ordinals > 0xFFFFFFFFll ||
        capacity < 0 || !offsets || (n_ordinals > 0 && !ordinals) || !out_offsets || (n_queries > 0 && !queries) ||
        (capacity > 0 && (!out_items || !out_scores))) {
        set_error("tav_range_search_subsets_into: invalid argument (0 <= n_ordinals < 2^32, capacity >= 0, accepted "
                  "flags)");
        return TAV_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lock(ix->mu);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (int rc = enter_stream(ix, s)) return rc;
    // no queries, no entries, no rows or a NaN min_score: no hits (the ordinals are not looked at)
    if (n_queries == 0 || n_ordinals == 0 || ix->size == 0 || ix->dim == 0 || min_score != min_score) {
        TAV_CUDA(cudaMemsetAsync(out_offsets, 0, (static_cast<size_t>(n_queries) + 1) * sizeof(int64_t), s));
        return mark_queued(ix, s);
    }
    return subsets_into(ix, "tav_range_search_subsets_into", queries, n_queries, 0, min_score, flags, offsets, ordinals,
                        n_ordinals, RangeOut{out_offsets, out_items, out_scores, capacity}, nullptr, nullptr, nullptr, s);
}

int tav_mma_scores(tav_index* ix, const float* queries, int n_queries, int flags, float* out_device,
                   void* stream) {
    if (!ix || n_queries < 1 || !queries || !out_device) return TAV_ERR_INVALID;
    std::lock_guard<std::mutex> lock(ix->mu);
    const bool split = ix->dtype == TAV_F32;
    if (ix->size == 0 || !(split ? mma_split_supported(ix->dim) : mma_supported(ix->dtype, ix->dim))) {
        set_error("tav_mma_scores: needs a non-empty index with dim %% 8 == 0");
        return TAV_ERR_INVALID;
    }
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (int rc = enter_stream(ix, s)) return rc;
    // staged as a search stages them: normalised on a TAV_NORMALIZE index, so these are the search's dots
    TimedSearch not_timed;
    const float* d_queries = nullptr;
    const int64_t* no_subset = nullptr;
    if (int rc = stage_inputs(ix, &not_timed, false, queries, n_queries, flags & TAV_QUERIES_ON_DEVICE, false, nullptr, 0,
                              &d_queries, &no_subset, s))
        return rc;
    if (split)
        if (int rc = ensure_split_planes(ix, nullptr, s)) return rc;
    MmaArgs m = mma_args(ix, split);
    m.split_overflow = split ? static_cast<int*>(ix->split_flag.p) + 1 : nullptr;
    m.queries = d_queries;
    m.nq = n_queries;
    m.k = 1;
    if (int rc = ensure_mma_ws(ix, mma_workspace_bytes(m), s)) return rc;
    TAV_CUDA(launch_mma_dump(m, ix->mma_ws.p, ix->mma_ws.bytes, out_device, s));
    TAV_CUDA(cudaStreamSynchronize(s));
    mark_done(ix);
    return TAV_OK;
}

int tav_merge_topk(int device, int n_lists, int n_queries, int k, const int64_t* items,
                   const float* scores, const int32_t* counts, int64_t items_stride,
                   int64_t scores_stride, int64_t counts_stride, int64_t* out_items,
                   float* out_scores, int32_t* out_counts, void* stream) {
    if (n_lists < 1 || n_queries < 0 || k < 1 || !items || !scores || !counts || !out_items ||
        !out_scores || !out_counts) {
        set_error("tav_merge_topk: invalid argument");
        return TAV_ERR_INVALID;
    }
    if (static_cast<int64_t>(n_lists) * k > 0x7FFFFFFFll || k > kPassK * 4) {
        set_error("tav_merge_topk: n_lists * k too large");
        return TAV_ERR_INVALID;
    }
    if (n_queries == 0) return TAV_OK;
    TAV_CUDA(cudaSetDevice(device));
    if (items_stride < 0 || scores_stride < 0 || counts_stride < 0) return TAV_ERR_INVALID;
    TAV_CUDA(launch_merge(n_lists, n_queries, k, items, scores, counts, items_stride, scores_stride,
                          counts_stride, out_items, out_scores, out_counts,
                          static_cast<cudaStream_t>(stream)));
    return TAV_OK;
}

int tav_merge_topk_ordered(int device, int n_lists, int n_queries, int k, const int64_t* items,
                           const float* scores, const int32_t* counts, int64_t items_stride,
                           int64_t scores_stride, int64_t counts_stride, int order, int64_t* out_items,
                           float* out_scores, int32_t* out_counts, void* stream) {
    if (n_lists < 1 || n_queries < 0 || k < 1 || !items || !scores || !counts || !out_items ||
        !out_scores || !out_counts || items_stride < 0 || scores_stride < 0 || counts_stride < 0) {
        set_error("tav_merge_topk_ordered: invalid argument");
        return TAV_ERR_INVALID;
    }
    if (order < 0 || order > 3) {
        set_error("tav_merge_topk_ordered: order %d is not 0, 1, 2 or 3", order);
        return TAV_ERR_INVALID;
    }
    if (static_cast<int64_t>(n_lists) * k > 0x7FFFFFFFll || k > kPassK * 4) {
        set_error("tav_merge_topk_ordered: n_lists * k too large");
        return TAV_ERR_INVALID;
    }
    if (n_queries == 0) return TAV_OK;
    TAV_CUDA(cudaSetDevice(device));
    TAV_CUDA(launch_merge_ordered(n_lists, n_queries, k, items, scores, counts, items_stride, scores_stride,
                                  counts_stride, order, out_items, out_scores, out_counts,
                                  static_cast<cudaStream_t>(stream)));
    return TAV_OK;
}

int tav_map_items(int device, int64_t n, const int64_t* table, int64_t table_len, int64_t* items, void* stream) {
    if (n < 0 || table_len < 0 || (n > 0 && !items) || (n > 0 && table_len > 0 && !table)) {
        set_error("tav_map_items: invalid argument");
        return TAV_ERR_INVALID;
    }
    if (n == 0 || table_len == 0) return TAV_OK;
    TAV_CUDA(cudaSetDevice(device));
    TAV_CUDA(launch_map_items(n, table, table_len, items, static_cast<cudaStream_t>(stream)));
    return TAV_OK;
}

int tav_fold_groups(int device, int n_queries, int k, const int32_t* row_to_group, int64_t n_rows,
                    int64_t item_offset, int64_t* items, float* scores, int32_t* counts, void* stream) {
    if (n_queries < 0 || k < 1 || k > 8192 || !row_to_group || n_rows < 0 || !items || !scores || !counts) {
        set_error("tav_fold_groups: invalid argument (k <= 8192)");
        return TAV_ERR_INVALID;
    }
    if (n_queries == 0) return TAV_OK;
    TAV_CUDA(cudaSetDevice(device));
    TAV_CUDA(launch_fold_groups(n_queries, k, row_to_group, n_rows, item_offset, items, scores, counts,
                                static_cast<cudaStream_t>(stream)));
    return TAV_OK;
}

int tav_set_timing(tav_index* ix, int enabled) {
    if (!ix) return TAV_ERR_INVALID;
    std::lock_guard<std::mutex> lock(ix->mu);
    ix->timing_on = enabled != 0;
    ix->timing_light = enabled == 2;
    if (ix->timing_on && !ix->hist) {
        ix->hist = new (std::nothrow) TimedSearch[kHistory];
        if (!ix->hist) return TAV_ERR_OOM;
    }
    ix->search_seq = 0;
    ix->untimed.valid = false;
    return TAV_OK;
}

}  // extern "C"

// sums of one timed search by kernel kind; synchronises on its last event
static int timed_sums(TimedSearch* t, float* main_ms, float* sample_ms, float* aux_ms, float* total_ms) {
    TAV_CUDA(cudaEventSynchronize(t->total[1]));
    float total = 0.0f, sums[3] = {0.0f, 0.0f, 0.0f};
    TAV_CUDA(cudaEventElapsedTime(&total, t->total[0], t->total[1]));
    for (int i = 0; i < t->used; ++i) {
        float ms = 0.0f;
        TAV_CUDA(cudaEventElapsedTime(&ms, t->ev[i][0], t->ev[i][1]));
        sums[t->kind[i] >= 0 && t->kind[i] < 3 ? t->kind[i] : 2] += ms;
    }
    if (main_ms) *main_ms = sums[0];
    if (sample_ms) *sample_ms = sums[1];
    if (aux_ms) *aux_ms = sums[2];
    if (total_ms) *total_ms = total;
    return TAV_OK;
}

extern "C" {

int tav_timing_breakdown(tav_index* ix, float* ms, int* kinds, int capacity, int* n) {
    if (!ix || !n || capacity < 0) return TAV_ERR_INVALID;
    std::lock_guard<std::mutex> lock(ix->mu);
    TimedSearch* t = last_timed(ix);
    if (!t->valid || !ix->timing_on || t == &ix->untimed) {
        *n = 0;
        return TAV_OK;
    }
    if (int rc = set_device(ix)) return rc;
    TAV_CUDA(cudaEventSynchronize(t->total[1]));
    *n = t->used;
    for (int i = 0; i < t->used && i < capacity; ++i) {
        float v = 0.0f;
        TAV_CUDA(cudaEventElapsedTime(&v, t->ev[i][0], t->ev[i][1]));
        if (ms) ms[i] = v;
        if (kinds) kinds[i] = t->kind[i];
    }
    return TAV_OK;
}

int tav_last_timing(tav_index* ix, float* scan_ms, float* total_ms, int* launches, int* path) {
    if (!ix) return TAV_ERR_INVALID;
    std::lock_guard<std::mutex> lock(ix->mu);
    TimedSearch* t = last_timed(ix);
    if (!t->valid) {
        set_error("tav_last_timing: no search on this index yet");
        return TAV_ERR_STATE;
    }
    if (launches) *launches = t->launches;
    if (path) *path = t->path;
    if (t == &ix->untimed) {  // path / launch count only
        if (scan_ms) *scan_ms = -1.0f;
        if (total_ms) *total_ms = -1.0f;
        return TAV_OK;
    }
    if (int rc = set_device(ix)) return rc;
    return timed_sums(t, scan_ms, nullptr, nullptr, total_ms);
}

int tav_timing_history(tav_index* ix, int capacity, float* main_ms, float* sample_ms, float* aux_ms,
                       float* total_ms, int* n) {
    if (!ix || !n || capacity < 0) return TAV_ERR_INVALID;
    std::lock_guard<std::mutex> lock(ix->mu);
    *n = 0;
    if (!ix->timing_on || !ix->hist) return TAV_OK;
    if (int rc = set_device(ix)) return rc;
    const int64_t have = std::min<int64_t>(ix->search_seq, kHistory);
    const int64_t take = std::min<int64_t>(have, capacity);
    for (int64_t i = 0; i < take; ++i) {
        TimedSearch* t = &ix->hist[(ix->search_seq - take + i) % kHistory];
        if (!t->valid) continue;
        float m = 0, sm = 0, ax = 0, tot = 0;
        if (int rc = timed_sums(t, &m, &sm, &ax, &tot)) return rc;
        if (main_ms) main_ms[*n] = m;
        if (sample_ms) sample_ms[*n] = sm;
        if (aux_ms) aux_ms[*n] = ax;
        if (total_ms) total_ms[*n] = tot;
        ++*n;
    }
    return TAV_OK;
}

}  // extern "C"
