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

// a grow-only device buffer
struct DevBuf {
    void* p = nullptr;
    size_t bytes = 0;
    cudaError_t ensure(size_t need) {
        if (need <= bytes) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr;
        bytes = 0;
        size_t want = std::max(need, size_t(1) << 16);
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) bytes = want;
        return e;
    }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        bytes = 0;
    }
};

// a grow-only pinned host buffer (staging for truly asynchronous H2D / D2H of small payloads)
struct PinBuf {
    void* p = nullptr;
    size_t bytes = 0;
    cudaError_t ensure(size_t need) {
        if (need <= bytes) return cudaSuccess;
        if (p) cudaFreeHost(p);
        p = nullptr;
        bytes = 0;
        size_t want = std::max(need, size_t(1) << 16);
        cudaError_t e = cudaMallocHost(&p, want);
        if (e == cudaSuccess) bytes = want;
        return e;
    }
    void release() {
        if (p) cudaFreeHost(p);
        p = nullptr;
        bytes = 0;
    }
};

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
    cudaEvent_t ev[kMaxTimedKernels][2];
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
    bool split, masked;
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
    // float32 indexes: the rows as two fp16 planes for the tensor-core path (built lazily,
    // extended on append); split_flag[0] = a corpus value left the fp16 range
    DevBuf split_hi, split_lo, split_flag;
    int64_t split_rows = 0;      // rows [0, split_rows) of the planes are current
    int64_t split_cap = 0;
    // predicate pushdown: one bit per row (tav_set_row_mask)
    DevBuf row_mask;
    int64_t row_mask_rows = 0;   // 0 = no mask set
    // threshold search (tav_range_search): collect regions, re-pass regions, sort scratch, CSR result
    DevBuf range_keys, range_keys2, range_counts, range_qgather, range_tmp, range_sortws;
    DevBuf range_mmaws, range_mmaws2, range_mmaaux;  // tensor-core collection: workspaces, scratch
    DevBuf range_items, range_scores;
    int64_t range_total = 0;     // hits of the last range search held in range_items / range_scores
    cudaEvent_t ev_range = nullptr;  // end of the last range search (tav_range_fetch waits for it)

    // timing
    TimedSearch* hist = nullptr; // [kHistory], created by tav_set_timing(1)
    int64_t search_seq = 0;      // searches timed so far
    TimedSearch untimed;         // path / launch count of the last search when timing is off
    bool timing_on = false;
    bool timing_light = false;  // events only around the dominant kernel and the whole search
};

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

static int finish_pending(tav_index* ix, cudaStream_t s, int* redone);

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
    if (ix->rows && !ix->adopted) cudaFree(ix->rows);
    for (DevBuf* b : {&ix->queries, &ix->held_queries, &ix->subset, &ix->cand_keys, &ix->cand_count, &ix->out_pack, &ix->staging,
                      &ix->mma_ws, &ix->retry, &ix->split_hi, &ix->split_lo, &ix->split_flag, &ix->row_mask,
                      &ix->range_keys, &ix->range_keys2, &ix->range_counts, &ix->range_qgather, &ix->range_tmp,
                      &ix->range_sortws, &ix->range_items, &ix->range_scores, &ix->range_mmaws,
                      &ix->range_mmaws2, &ix->range_mmaaux})
        b->release();
    for (DevBuf& b : ix->held_retired) b.release();
    if (ix->ev_range) cudaEventDestroy(ix->ev_range);
    ix->pin_in.release();
    ix->pin_out.release();
    ix->retry_host.release();
    for (auto& b : ix->pin_append) b.release();
    if (ix->ev_pin_in) cudaEventDestroy(ix->ev_pin_in);
    for (auto& ev : ix->ev_append)
        if (ev) cudaEventDestroy(ev);
    destroy_history(ix);
    delete ix;
    return TAV_OK;
}

int tav_clear(tav_index* ix) {
    if (!ix) return TAV_ERR_INVALID;
    std::lock_guard<std::mutex> lock(ix->mu);
    if (ix->adopted) {
        ix->rows = nullptr;
        ix->adopted = false;
        ix->capacity = 0;
    }
    ix->size = 0;
    ix->split_rows = 0;
    ix->row_mask_rows = 0;
    if (ix->split_flag.p) {  // the sticky "a corpus value left the fp16 range" flag dies with the rows
        cudaSetDevice(ix->device);
        cudaMemset(ix->split_flag.p, 0, sizeof(int));
    }
    return TAV_OK;
}

static int reserve_locked(tav_index* ix, int64_t rows) {
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
    TAV_CUDA(cudaMalloc(&fresh, std::max<size_t>(static_cast<size_t>(rows) * row_bytes, 256)));
    if (ix->size > 0) {
        // in-order with whatever was enqueued on the index stream; then make it visible to all
        cudaError_t e = cudaMemcpy(fresh, ix->rows, static_cast<size_t>(ix->size) * row_bytes,
                                   cudaMemcpyDeviceToDevice);
        if (e != cudaSuccess) {
            cudaFree(fresh);
            set_error("tav_reserve: copy failed: %s", cudaGetErrorString(e));
            return TAV_ERR_CUDA;
        }
    }
    if (ix->rows) {
        cudaDeviceSynchronize();
        cudaFree(ix->rows);
    }
    ix->rows = fresh;
    ix->capacity = rows;
    return TAV_OK;
}

int tav_reserve(tav_index* ix, int64_t rows) {
    if (!ix || rows < 0) return TAV_ERR_INVALID;
    std::lock_guard<std::mutex> lock(ix->mu);
    return reserve_locked(ix, rows);
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
    if (int rc = set_device(ix)) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (ix->size + n > ix->capacity) {
        int64_t want = std::max<int64_t>(ix->size + n, ix->capacity * 2);
        want = std::max<int64_t>(want, 1024);
        TAV_CUDA(cudaStreamSynchronize(s));
        if (int rc = reserve_locked(ix, want)) return rc;
    }
    const size_t dst_row = static_cast<size_t>(ix->dim) * dtype_size(ix->dtype);
    const size_t src_row = static_cast<size_t>(ix->dim) * dtype_size(src_dtype);
    char* dst = static_cast<char*>(ix->rows) + static_cast<size_t>(ix->size) * dst_row;
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
    ix->size += n;
    return TAV_OK;
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
    cudaSetDevice(ix->device);
    if (ix->rows && !ix->adopted) {
        cudaDeviceSynchronize();
        cudaFree(ix->rows);
    }
    ix->dim = dim;
    ix->rows = device_rows;
    ix->split_rows = 0;
    if (ix->split_flag.p) cudaMemset(ix->split_flag.p, 0, sizeof(int));
    ix->row_mask_rows = 0;
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
    if (int rc = set_device(ix)) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
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
    return TAV_OK;
}

int tav_set_row_mask(tav_index* ix, const uint32_t* bits, int64_t n_rows, int on_device, void* stream) {
    if (!ix || n_rows < 0 || (n_rows > 0 && !bits)) return TAV_ERR_INVALID;
    std::lock_guard<std::mutex> lock(ix->mu);
    if (int rc = set_device(ix)) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (!ix->pending.empty()) {  // an outstanding search may still need the old mask for its exact redo
        int redone = 0;
        if (int rc = finish_pending(ix, s, &redone)) return rc;
    }
    if (n_rows == 0) {
        ix->row_mask_rows = 0;
        return TAV_OK;
    }
    if (n_rows != ix->size) {
        set_error("tav_set_row_mask: %lld bits for an index of %lld rows", (long long)n_rows, (long long)ix->size);
        return TAV_ERR_INVALID;
    }
    // padded to whole 256-row tiles (the tensor-core epilogue reads one word per 32 rows of a tile)
    const size_t words = static_cast<size_t>((n_rows + 255) / 256) * 8;
    const size_t src_words = static_cast<size_t>((n_rows + 31) / 32);
    TAV_CUDA(ix->row_mask.ensure(words * sizeof(uint32_t)));
    TAV_CUDA(cudaMemsetAsync(ix->row_mask.p, 0, words * sizeof(uint32_t), s));
    TAV_CUDA(cudaMemcpyAsync(ix->row_mask.p, bits, src_words * sizeof(uint32_t),
                             on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, s));
    if (!on_device) TAV_CUDA(cudaStreamSynchronize(s));
    ix->row_mask_rows = n_rows;
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
                       bool allow_fuse = true) {
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
            ScanArgs a{};
            a.corpus = ix->rows;
            a.dtype = ix->dtype;
            a.n_corpus = ix->size;
            a.dim = ix->dim;
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
            a.ties_low = ties_low;
            if (fuse) {
                a.fused = 1;
                a.fused_ticket = d_count + 8;
                a.item_offset = item_offset;
                a.out_items = d_items + static_cast<size_t>(q0) * k;
                a.out_scores = d_scores + static_cast<size_t>(q0) * k;
                a.out_counts = d_counts + q0;
            }
            const bool timed = timing && ts && ts->used < kMaxTimedKernels;
            if (timed) TAV_CUDA(ev_record(ts->ev[ts->used][0], s));
            TAV_CUDA(launch_scan(a, s));
            if (timed) {
                ts->kind[ts->used] = 0;
                TAV_CUDA(ev_record(ts->ev[ts->used++][1], s));
            }
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
            sel.subset = d_subset;
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

static inline int32_t* retry_totals(tav_index* ix, int slot) { return static_cast<int32_t*>(ix->retry.p) + 2 * slot; }
static inline int32_t* retry_flags(tav_index* ix, int slot) {
    return static_cast<int32_t*>(ix->retry.p) + 2 * kMaxPending + static_cast<size_t>(slot) * ix->retry_cap;
}

// Synchronising tail of the tensor-core searches: look at the "redo exactly" bookkeeping of every
// outstanding search and redo flagged queries with the row scan, into that search's own outputs.
static int finish_pending(tav_index* ix, cudaStream_t s, int* redone) {
    if (redone) *redone = 0;
    if (ix->pending.empty()) return TAV_OK;
    int32_t totals[2 * kMaxPending];
    int corpus_overflow = 0;
    bool any_split = false;
    for (const Pending& p : ix->pending) any_split |= p.split;
    if (any_split)
        TAV_CUDA(cudaMemcpyAsync(&corpus_overflow, ix->split_flag.p, sizeof(int), cudaMemcpyDeviceToHost, s));
    TAV_CUDA(cudaStreamSynchronize(s));
    memcpy(totals, ix->retry_host.p, sizeof(totals));  // written by the kernels through the mapping; current after the sync
    std::vector<Pending> todo;
    todo.swap(ix->pending);
    ix->next_slot = 0;
    bool dirty = false;
    int n_redone = 0;
    std::vector<int32_t> host;
    for (const Pending& p : todo) {
        const int flagged = totals[2 * p.slot], q_overflow = totals[2 * p.slot + 1];
        const bool redo_all = p.split && (corpus_overflow != 0 || q_overflow != 0);
        dirty |= flagged != 0 || q_overflow != 0;
        if (flagged == 0 && !redo_all) continue;
        host.assign(static_cast<size_t>(p.nq), 1);
        if (!redo_all) {
            TAV_CUDA(cudaMemcpyAsync(host.data(), retry_flags(ix, p.slot), static_cast<size_t>(p.nq) * sizeof(int32_t),
                                     cudaMemcpyDeviceToHost, s));
            TAV_CUDA(cudaStreamSynchronize(s));
        }
        const uint32_t* mask = p.masked ? static_cast<const uint32_t*>(ix->row_mask.p) : nullptr;
        for (int q = 0; q < p.nq; ++q) {
            if (!host[q]) continue;
            ++n_redone;
            int rc = scan_search(ix, nullptr, false, p.queries + static_cast<size_t>(q) * ix->dim, 1, p.k, p.floor, nullptr,
                                 ix->size, p.item_offset, p.items + static_cast<size_t>(q) * p.k,
                                 p.scores + static_cast<size_t>(q) * p.k, p.counts + q, mask, 0, s);
            if (rc != TAV_OK) return rc;
        }
    }
    if (dirty) TAV_CUDA(cudaMemsetAsync(ix->retry.p, 0, sizeof(totals), s));
    if (dirty || n_redone > 0) TAV_CUDA(cudaStreamSynchronize(s));
    if (dirty) memset(ix->retry_host.p, 0, sizeof(totals));
    // No queued work reads a held query region now, whatever stream a later search uses: the searches ended
    // at the first synchronisation above, their redo scans at the last.  So the regions can be reused and the
    // outgrown buffers freed.
    ix->held_used = 0;
    for (DevBuf& b : ix->held_retired) b.release();
    ix->held_retired.clear();
    if (redone) *redone = n_redone;
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
                         uint64_t* keys, int64_t stride, uint32_t* counts, cudaStream_t s) {
    const int qb = scan_collect_max_queries(ix->dim);  // a smaller last block takes a smaller instantiation
    if (qb < 1) {
        set_error("threshold search: embedding size %d too large for the row-scan kernel", ix->dim);
        return TAV_ERR_INVALID;
    }
    const int grid = scan_collect_grid(ix->device, ix->dim, qb, n_scan);
    for (int q0 = 0; q0 < nq; q0 += qb) {
        ScanArgs a{};
        a.corpus = ix->rows;
        a.dtype = ix->dtype;
        a.n_corpus = ix->size;
        a.dim = ix->dim;
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
        a.ties_low = ties_low;
        const bool timed = timing && ts->used < kMaxTimedKernels;
        if (timed) TAV_CUDA(ev_record(ts->ev[ts->used][0], s));
        TAV_CUDA(launch_scan_collect(a, s));
        if (timed) {
            ts->kind[ts->used] = 0;
            TAV_CUDA(ev_record(ts->ev[ts->used++][1], s));
        }
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
    const bool timed = timing && !ix->timing_light && ts->used < kMaxTimedKernels;
    if (timed) TAV_CUDA(ev_record(ts->ev[ts->used][0], s));
    TAV_CUDA(launch_segmented_sort(sa, s, &ts->launches));
    if (timed) {
        ts->kind[ts->used] = 2;
        TAV_CUDA(ev_record(ts->ev[ts->used++][1], s));
    }
    return TAV_OK;
}

// Row-scan collection: one collect scan per block of queries into regions sized from `expected_hits`; the
// counters keep counting past a region, so after the one synchronisation the totals are exact and the
// overflowed queries get exactly one more scan into regions of that size.
static int range_collect_scan(tav_index* ix, TimedSearch* ts, bool timing, const float* d_queries, int nq, float floor,
                              const int64_t* d_subset, int64_t n_scan, int64_t item_offset, const uint32_t* d_mask,
                              int ties_low, int64_t expected_hits, std::vector<int64_t>& offsets, cudaStream_t s) {
    const int64_t per = range_per_query(expected_hits, nq, n_scan);
    if (int rc = range_alloc(ix->range_keys, static_cast<size_t>(nq) * per * sizeof(uint64_t), "the hit regions")) return rc;
    if (int rc = range_alloc(ix->range_counts, static_cast<size_t>(nq) * sizeof(uint32_t), "the hit counters")) return rc;
    uint32_t* d_counts = static_cast<uint32_t*>(ix->range_counts.p);
    uint64_t* keys = static_cast<uint64_t*>(ix->range_keys.p);
    TAV_CUDA(cudaMemsetAsync(d_counts, 0, static_cast<size_t>(nq) * sizeof(uint32_t), s));
    if (int rc = collect_scans(ix, ts, timing, d_queries, nq, floor, d_subset, n_scan, d_mask, ties_low, keys, per,
                               d_counts, s))
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
        const size_t qrow = static_cast<size_t>(ix->dim) * sizeof(float);
        if (int rc = range_alloc(ix->range_keys2, static_cast<size_t>(no) * over_max * sizeof(uint64_t), "the re-pass regions"))
            return rc;
        if (int rc = range_alloc(ix->range_qgather, no * qrow, "the re-pass queries")) return rc;
        keys2 = static_cast<uint64_t*>(ix->range_keys2.p);
        char* qg = static_cast<char*>(ix->range_qgather.p);
        for (int i = 0; i < no; ++i)
            TAV_CUDA(cudaMemcpyAsync(qg + i * qrow, reinterpret_cast<const char*>(d_queries) + over[i] * qrow, qrow,
                                     cudaMemcpyDeviceToDevice, s));
        TAV_CUDA(cudaMemsetAsync(d_counts, 0, static_cast<size_t>(no) * sizeof(uint32_t), s));
        if (int rc = collect_scans(ix, ts, timing, reinterpret_cast<const float*>(qg), no, floor, d_subset, n_scan,
                                   d_mask, ties_low, keys2, over_max, d_counts, s))
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
    return range_sort(ix, ts, timing, segs, offsets[nq], d_subset, item_offset, ties_low, s);
}

constexpr int kRangeUseScan = 1;  // range_collect_mma: the tensor-core form cannot serve this search

// Tensor-core collection: the MAIN kernel without a sample pass and with the exact dot floor of min_score
// as threshold, segments sized from `expected_hits`, a count kernel; after the one synchronisation the
// overflowed queries get one more MAIN pass (only they, same rows per segment, segments of the counted size)
// and every query's keys are gathered in CSR order.  Returns kRangeUseScan when the float32 split form met
// a value beyond the fp16 range (the exact row scan then serves the search, as it does for top-k searches).
static int range_collect_mma(tav_index* ix, TimedSearch* ts, bool timing, const float* d_queries, int nq, float floor,
                             int64_t item_offset, const uint32_t* d_mask, int ties_low, int64_t expected_hits,
                             std::vector<int64_t>& offsets, cudaStream_t s) {
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
    if (timing)  // the launcher records into existing events
        for (int i = 0; i < kMaxTimedKernels; ++i)
            for (int j = 0; j < 2; ++j)
                if (!ts->ev[i][j]) TAV_CUDA(cudaEventCreate(&ts->ev[i][j]));
    MmaArgs m{};
    m.device = ix->device;
    m.corpus = split ? ix->split_hi.p : ix->rows;
    m.corpus_lo = split ? ix->split_lo.p : nullptr;
    m.split = split ? 1 : 0;
    m.split_overflow = split ? d_qflag : nullptr;
    m.dtype = ix->dtype;
    m.n_corpus = ix->size;
    m.dim = ix->dim;
    m.queries = d_queries;
    m.nq = nq;
    m.floor_score = floor;
    m.k = 1;
    m.item_offset = item_offset;
    m.retry_flags = reinterpret_cast<int32_t*>(aux);
    m.row_mask = d_mask;
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
        const size_t qrow = static_cast<size_t>(ix->dim) * sizeof(float);
        if (int rc = range_alloc(ix->range_qgather, no * qrow, "the re-pass queries")) return rc;
        char* qg = static_cast<char*>(ix->range_qgather.p);
        for (int i = 0; i < no; ++i)
            TAV_CUDA(cudaMemcpyAsync(qg + i * qrow, reinterpret_cast<const char*>(d_queries) + over[i] * qrow, qrow,
                                     cudaMemcpyDeviceToDevice, s));
        MmaArgs m2 = m;
        m2.queries = reinterpret_cast<const float*>(qg);
        m2.nq = no;
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
    return range_sort(ix, ts, timing, segs, total, nullptr, item_offset, ties_low, s);
}

// Every row with score >= floor, for each of nq device queries -> ix->range_items / range_scores in CSR order
// (offsets[nq + 1], host): collected by the tensor cores (use_mma) or the row scan, then the segmented sort.
static int range_core(tav_index* ix, TimedSearch* ts, bool timing, const float* d_queries, int nq, float floor,
                      const int64_t* d_subset, int64_t n_scan, int64_t item_offset, const uint32_t* d_mask,
                      int ties_low, int64_t expected_hits, bool use_mma, std::vector<int64_t>& offsets, cudaStream_t s) {
    if (use_mma) {
        const int rc = range_collect_mma(ix, ts, timing, d_queries, nq, floor, item_offset, d_mask, ties_low,
                                         expected_hits, offsets, s);
        if (rc != kRangeUseScan) return rc;
        ts->path = 1;  // a value beyond the fp16 range: the exact row scan serves the search
    }
    return range_collect_scan(ix, ts, timing, d_queries, nq, floor, d_subset, n_scan, item_offset, d_mask, ties_low,
                              expected_hits, offsets, s);
}

// the hits of the last threshold search are complete once this event has passed (tav_range_fetch waits)
static int range_mark_end(tav_index* ix, cudaStream_t s) {
    if (!ix->ev_range) TAV_CUDA(cudaEventCreateWithFlags(&ix->ev_range, cudaEventDisableTiming));
    TAV_CUDA(cudaEventRecord(ix->ev_range, s));
    return TAV_OK;
}

extern "C" {

const int32_t* tav_internal_retry_totals(tav_index* ix, int* count) {
    if (count) *count = 0;
    if (!ix || ix->last_first_slot < 0 || !ix->retry.p) return nullptr;
    if (count) *count = ix->last_n_slots;
    return retry_totals(ix, ix->last_first_slot);
}

int tav_finish_search(tav_index* ix, void* stream, int* redone) {
    if (!ix) return TAV_ERR_INVALID;
    std::lock_guard<std::mutex> lock(ix->mu);
    if (redone) *redone = 0;
    if (ix->pending.empty()) return TAV_OK;  // nothing deferred (row-scan path, or already finished)
    if (int rc = set_device(ix)) return rc;
    return finish_pending(ix, static_cast<cudaStream_t>(stream), redone);
}

int tav_search(tav_index* ix, const float* queries, int n_queries, int k, float min_score,
               int flags, const int64_t* subset, int64_t subset_len, int64_t item_offset,
               int64_t* out_items, float* out_scores, int32_t* out_counts, void* stream) {
    if (!ix || n_queries < 0 || k < 1 || (n_queries > 0 && (!queries || !out_items || !out_scores || !out_counts))) {
        set_error("tav_search: invalid argument (k must be >= 1)");
        return TAV_ERR_INVALID;
    }
    if ((subset && subset_len < 0) || (!subset && subset_len != 0)) {
        set_error("tav_search: subset / subset_len mismatch");
        return TAV_ERR_INVALID;
    }
    if (n_queries == 0) return TAV_OK;
    std::lock_guard<std::mutex> lock(ix->mu);
    if (int rc = set_device(ix)) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const bool q_dev = flags & TAV_QUERIES_ON_DEVICE, o_dev = flags & TAV_OUTPUTS_ON_DEVICE;
    const size_t nk = static_cast<size_t>(n_queries) * k;
    const uint32_t* d_mask = nullptr;
    if (flags & TAV_USE_ROW_MASK) {
        if (ix->row_mask_rows != ix->size || ix->size == 0) {
            set_error("tav_search: TAV_USE_ROW_MASK without a current row mask (tav_set_row_mask)");
            return TAV_ERR_STATE;
        }
        if (subset) {
            set_error("tav_search: a row mask and a subset cannot be combined");
            return TAV_ERR_INVALID;
        }
        d_mask = static_cast<const uint32_t*>(ix->row_mask.p);
    }
    const int ties_low = (flags & TAV_TIES_LOW_FIRST) ? 1 : 0;

    int64_t* d_items = out_items;
    float* d_scores = out_scores;
    int32_t* d_counts = out_counts;
    // host outputs: results are packed [items | scores | counts | done word] in one buffer so that a
    // single D2H copy (into pinned staging) brings them back
    const size_t off_scores = nk * sizeof(int64_t);
    const size_t off_counts = off_scores + ((nk * sizeof(float) + 7) & ~size_t(7));
    const size_t off_done = off_counts + ((static_cast<size_t>(n_queries) * sizeof(int32_t) + 7) & ~size_t(7));
    const size_t pack_bytes = off_done + 8;
    // Small result sets are written by the kernels straight into the pinned host staging (zero
    // copy over PCIe: no D2H memcpy call on the single-lookup latency path).
    const bool zero_copy_out = !o_dev && pack_bytes <= kZeroCopyOutLimit;

    const int64_t n_scan = subset ? subset_len : ix->size;
    ix->last_first_slot = -1;
    ix->last_n_slots = 0;
    TimedSearch* ts = cur_timed(ix);
    if (!ts) ts = &ix->untimed;
    const bool timing = ts != &ix->untimed;
    ts->used = 0;
    ts->launches = 0;
    ts->path = 0;
    ts->valid = false;

    // a NaN min_score admits nothing on every path (`scores >= nan` is all-false in the reference)
    if (n_scan == 0 || ix->size == 0 || ix->dim == 0 || min_score != min_score) {
        // empty corpus / empty subset: no hits (vectorbase.py:174-175, :214-215)
        if (o_dev) TAV_CUDA(cudaMemsetAsync(d_counts, 0, static_cast<size_t>(n_queries) * sizeof(int32_t), s));
        else memset(out_counts, 0, static_cast<size_t>(n_queries) * sizeof(int32_t));
        return TAV_OK;
    }
    if (n_scan > 0xFFFFFFFFll) {
        set_error("tav_search: more than 2^32 rows per index are not supported; shard the corpus");
        return TAV_ERR_INVALID;
    }

    // subset ordinals: validate on the host (numpy raises IndexError)
    if (subset) {
        for (int64_t i = 0; i < subset_len; ++i) {
            if (subset[i] < -ix->size || subset[i] >= ix->size) {
                set_error("index %lld is out of bounds for axis 0 with size %lld",
                          (long long)subset[i], (long long)ix->size);
                return TAV_ERR_RANGE;
            }
        }
    }

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
        if (int rc = range_core(ix, ts, timing, d_q, n_queries, min_score, d_sub, n_scan, item_offset, d_mask, ties_low,
                                static_cast<int64_t>(n_queries) * n_scan, false, offsets, s))
            return rc;
        if (timing) {
            TAV_CUDA(ev_record(ts->total[1], s));
            ++ix->search_seq;
        }
        ts->valid = true;
        ix->range_total = offsets[n_queries];
        if (int rc = range_mark_end(ix, s)) return rc;
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
        TAV_CUDA(ix->pin_out.ensure(pack_bytes));
        char* base = static_cast<char*>(ix->pin_out.p);
        d_items = reinterpret_cast<int64_t*>(base);
        d_scores = reinterpret_cast<float*>(base + off_scores);
        d_counts = reinterpret_cast<int32_t*>(base + off_counts);
    } else if (!o_dev) {
        TAV_CUDA(ix->out_pack.ensure(pack_bytes));
        char* base = static_cast<char*>(ix->out_pack.p);
        d_items = reinterpret_cast<int64_t*>(base);
        d_scores = reinterpret_cast<float*>(base + off_scores);
        d_counts = reinterpret_cast<int32_t*>(base + off_counts);
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
        ScanArgs a{};
        a.corpus = ix->rows;
        a.dtype = ix->dtype;
        a.n_corpus = ix->size;
        a.dim = ix->dim;
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
        volatile uint32_t* done = reinterpret_cast<volatile uint32_t*>(static_cast<char*>(ix->pin_out.p) + off_done);
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
        if (timing) {
            TAV_CUDA(ev_record(ts->total[0], s));
            TAV_CUDA(ev_record(ts->ev[0][0], s));
        }
        TAV_CUDA(launch_scan1(a, queries, subset, s));
        if (timing) {
            ts->kind[0] = 0;
            TAV_CUDA(ev_record(ts->ev[0][1], s));
            ts->used = 1;
            TAV_CUDA(ev_record(ts->total[1], s));
        }
        ts->launches = 1;
        ts->valid = true;
        if (timing) ++ix->search_seq;
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
        const char* h = static_cast<const char*>(ix->pin_out.p);
        memcpy(out_items, h, nk * sizeof(int64_t));
        memcpy(out_scores, h + off_scores, nk * sizeof(float));
        memcpy(out_counts, h + off_counts, sizeof(int32_t));
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
        const size_t q_bytes = (static_cast<size_t>(n_queries) * ix->dim * sizeof(float) + 255) & ~size_t(255);
        const size_t need = ix->held_used + q_bytes;
        if (need > ix->held_queries.bytes) {
            const size_t want = std::max(need, 2 * ix->held_queries.bytes);
            if (ix->held_used > 0) {  // pending searches read the current buffer
                ix->held_retired.push_back(ix->held_queries);
                ix->held_queries = DevBuf{};
                ix->held_used = 0;
            }
            TAV_CUDA(ix->held_queries.ensure(want));
        }
        held = reinterpret_cast<float*>(static_cast<char*>(ix->held_queries.p) + ix->held_used);
        held_end = ix->held_used + q_bytes;
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
        if (n_queries > ix->retry_cap || !ix->retry.p) {
            if (!ix->pending.empty()) {
                int redone = 0;
                if (int rc = finish_pending(ix, s, &redone)) return rc;
            }
            const int cap = std::max(std::min(n_queries, kMmaMaxQueries), 1024);
            const size_t bytes = (static_cast<size_t>(2) * kMaxPending + static_cast<size_t>(kMaxPending) * cap) * sizeof(int32_t);
            TAV_CUDA(ix->retry.ensure(bytes));
            TAV_CUDA(cudaMemsetAsync(ix->retry.p, 0, 2 * kMaxPending * sizeof(int32_t), s));
            TAV_CUDA(ix->retry_host.ensure(2 * kMaxPending * sizeof(int32_t)));
            memset(ix->retry_host.p, 0, 2 * kMaxPending * sizeof(int32_t));
            ix->retry_cap = cap;
        }
        if (timing)  // the events of this search exist before the launcher records them
            for (int i = 0; i < kMaxTimedKernels; ++i)
                for (int j = 0; j < 2; ++j)
                    if (!ts->ev[i][j]) TAV_CUDA(cudaEventCreate(&ts->ev[i][j]));
        // one launch sequence per slab of kMmaMaxQueries queries (in practice: one)
        for (int q0 = 0; q0 < n_queries; q0 += kMmaMaxQueries) {
            const int nq = std::min(kMmaMaxQueries, n_queries - q0);
            // bookkeeping slot of this (part of the) search
            if (static_cast<int>(ix->pending.size()) >= kMaxPending) {
                int redone = 0;
                if (int rc = finish_pending(ix, s, &redone)) return rc;
            }
            const int slot = ix->next_slot++;
            if (q0 == 0) ix->last_first_slot = slot;
            ix->last_n_slots = slot - ix->last_first_slot + 1;
            MmaArgs m{};
            m.device = ix->device;
            m.corpus = use_split ? ix->split_hi.p : ix->rows;
            m.corpus_lo = use_split ? ix->split_lo.p : nullptr;
            m.split = use_split ? 1 : 0;
            m.split_overflow = use_split ? retry_totals(ix, slot) + 1 : nullptr;
            m.dtype = ix->dtype;
            m.n_corpus = ix->size;
            m.dim = ix->dim;
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
            int ev_used = 0;
            const bool slab_timed = timing && q0 == 0;
            m.ev = slab_timed ? ts->ev : nullptr;
            m.ev_kind = ts->kind;
            m.ev_max = kMaxTimedKernels;
            m.ev_used = &ev_used;
            m.ev_main_only = ix->timing_light ? 1 : 0;
            const size_t ws = mma_workspace_bytes(m);
            if (ws > ix->mma_ws.bytes) {
                TAV_CUDA(cudaStreamSynchronize(s));  // earlier searches may still use the old workspace
                TAV_CUDA(ix->mma_ws.ensure(ws));
                // the sampler's unit counters (start of the workspace) must read zero
                TAV_CUDA(cudaMemsetAsync(ix->mma_ws.p, 0, std::min<size_t>(ix->mma_ws.bytes, 65536), s));
            }
            int launches = 0;
            TAV_CUDA(launch_mma_search(m, ix->mma_ws.p, ix->mma_ws.bytes, s, &launches));
            if (slab_timed) ts->used = ev_used;
            ts->launches += launches;
            Pending p{m.queries, nq, k, min_score, item_offset, m.out_items, m.out_scores, m.out_counts, slot,
                      use_split, d_mask != nullptr};
            ix->pending.push_back(p);
            ix->held_used = std::max(ix->held_used, held_end);  // (a finish_pending above may have reset it)
        }
        // Queries the sampled admission threshold could not settle (fewer than k admitted rows
        // although rows were cut, or candidate overflow) are redone exactly by the row scan —
        // now, or in tav_finish_search when the caller defers the (synchronising) check.
        if (!defer) {
            int redone = 0;
            if (int rc = finish_pending(ix, s, &redone)) return rc;
        }
    } else {
        ts->path = 1;
        int rc = scan_search(ix, ts, timing, d_queries, n_queries, k, min_score, d_subset, n_scan, item_offset,
                             d_items, d_scores, d_counts, d_mask, ties_low, s, !(flags & TAV_NO_FUSED_SCAN));
        if (rc != TAV_OK) return rc;
    }
    if (timing) {
        TAV_CUDA(ev_record(ts->total[1], s));
        ++ix->search_seq;
    }
    ts->valid = true;

    if (zero_copy_out) {
        TAV_CUDA(cudaStreamSynchronize(s));
        const char* h = static_cast<const char*>(ix->pin_out.p);
        memcpy(out_items, h, nk * sizeof(int64_t));
        memcpy(out_scores, h + off_scores, nk * sizeof(float));
        memcpy(out_counts, h + off_counts, static_cast<size_t>(n_queries) * sizeof(int32_t));
    } else if (!o_dev) {
        if (pack_bytes <= kPinnedStageLimit) {
            TAV_CUDA(ix->pin_out.ensure(pack_bytes));
            TAV_CUDA(cudaMemcpyAsync(ix->pin_out.p, ix->out_pack.p, off_done, cudaMemcpyDeviceToHost, s));
            TAV_CUDA(cudaStreamSynchronize(s));
            const char* h = static_cast<const char*>(ix->pin_out.p);
            memcpy(out_items, h, nk * sizeof(int64_t));
            memcpy(out_scores, h + off_scores, nk * sizeof(float));
            memcpy(out_counts, h + off_counts, static_cast<size_t>(n_queries) * sizeof(int32_t));
        } else {
            TAV_CUDA(cudaMemcpyAsync(out_items, d_items, nk * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
            TAV_CUDA(cudaMemcpyAsync(out_scores, d_scores, nk * sizeof(float), cudaMemcpyDeviceToHost, s));
            TAV_CUDA(cudaMemcpyAsync(out_counts, d_counts, static_cast<size_t>(n_queries) * sizeof(int32_t),
                                     cudaMemcpyDeviceToHost, s));
            TAV_CUDA(cudaStreamSynchronize(s));
        }
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
    if ((subset && subset_len < 0) || (!subset && subset_len != 0)) {
        set_error("tav_range_search: subset / subset_len mismatch");
        return TAV_ERR_INVALID;
    }
    if (flags & TAV_DEFER_RETRY) {
        set_error("tav_range_search: TAV_DEFER_RETRY is not available for threshold searches");
        return TAV_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lock(ix->mu);
    if (int rc = set_device(ix)) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const bool q_dev = flags & TAV_QUERIES_ON_DEVICE, o_dev = flags & TAV_OUTPUTS_ON_DEVICE;
    ix->range_total = 0;
    std::vector<int64_t> offsets(static_cast<size_t>(n_queries) + 1, 0);
    auto write_offsets = [&]() -> int {
        const size_t bytes = offsets.size() * sizeof(int64_t);
        if (o_dev) {  // from pageable memory: consumed when the call returns
            TAV_CUDA(cudaMemcpyAsync(out_offsets, offsets.data(), bytes, cudaMemcpyHostToDevice, s));
        } else {
            memcpy(out_offsets, offsets.data(), bytes);
        }
        return range_mark_end(ix, s);
    };
    const uint32_t* d_mask = nullptr;
    if (flags & TAV_USE_ROW_MASK) {
        if (ix->row_mask_rows != ix->size || ix->size == 0) {
            set_error("tav_range_search: TAV_USE_ROW_MASK without a current row mask (tav_set_row_mask)");
            return TAV_ERR_STATE;
        }
        if (subset) {
            set_error("tav_range_search: a row mask and a subset cannot be combined");
            return TAV_ERR_INVALID;
        }
        d_mask = static_cast<const uint32_t*>(ix->row_mask.p);
    }
    const int64_t n_scan = subset ? subset_len : ix->size;
    // NaN min_score, empty corpus or empty subset: no hits
    if (n_queries == 0 || n_scan == 0 || ix->size == 0 || ix->dim == 0 || min_score != min_score) return write_offsets();
    if (n_scan > 0xFFFFFFFFll) {
        set_error("tav_range_search: more than 2^32 rows per index are not supported; shard the corpus");
        return TAV_ERR_INVALID;
    }
    if (subset) {
        for (int64_t i = 0; i < subset_len; ++i) {
            if (subset[i] < -ix->size || subset[i] >= ix->size) {
                set_error("index %lld is out of bounds for axis 0 with size %lld", (long long)subset[i],
                          (long long)ix->size);
                return TAV_ERR_RANGE;
            }
        }
    }
    // path choice as in tav_search: tensor cores for batches (no subset), the row scan otherwise
    const bool mma_able = (mma_supported(ix->dtype, ix->dim) || (ix->dtype == TAV_F32 && mma_split_supported(ix->dim))) &&
                          !subset && n_queries <= kMmaMaxQueries && ix->size < (1ll << 31);
    const bool use_mma = !(flags & TAV_FORCE_SCAN) && mma_able &&
                         ((flags & TAV_FORCE_MMA) || (n_queries >= 16 && ix->size >= 4096));
    if ((flags & TAV_FORCE_MMA) && !use_mma) {
        set_error("tav_range_search: TAV_FORCE_MMA needs dim %% 8 == 0, no subset, at most %d queries", kMmaMaxQueries);
        return TAV_ERR_INVALID;
    }
    TimedSearch* ts = cur_timed(ix);
    if (!ts) ts = &ix->untimed;
    const bool timing = ts != &ix->untimed;
    ts->used = 0;
    ts->launches = 0;
    ts->path = use_mma ? (ix->dtype == TAV_F32 ? 3 : 2) : 1;
    ts->valid = false;
    const float* d_queries = nullptr;
    const int64_t* d_subset = nullptr;
    if (int rc = stage_inputs(ix, ts, timing, queries, n_queries, q_dev, false, subset, subset_len, &d_queries, &d_subset, s))
        return rc;
    if (int rc = range_core(ix, ts, timing, d_queries, n_queries, min_score, d_subset, n_scan, item_offset, d_mask,
                            (flags & TAV_TIES_LOW_FIRST) ? 1 : 0, expected_hits, use_mma, offsets, s))
        return rc;
    if (timing) {
        TAV_CUDA(ev_record(ts->total[1], s));
        ++ix->search_seq;
    }
    ts->valid = true;
    ix->range_total = offsets[n_queries];
    return write_offsets();
}

int tav_range_fetch(tav_index* ix, int64_t first, int64_t n, int64_t* out_items, float* out_scores, int flags,
                    void* stream) {
    if (!ix || first < 0 || n < 0 || (n > 0 && (!out_items || !out_scores))) {
        set_error("tav_range_fetch: invalid argument");
        return TAV_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lock(ix->mu);
    if (first + n > ix->range_total) {
        set_error("tav_range_fetch: hits [%lld, %lld) out of range (the last range search has %lld)", (long long)first,
                  (long long)(first + n), (long long)ix->range_total);
        return TAV_ERR_RANGE;
    }
    if (n == 0) return TAV_OK;
    if (int rc = set_device(ix)) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (ix->ev_range) TAV_CUDA(cudaStreamWaitEvent(s, ix->ev_range, 0));
    const cudaMemcpyKind kind = (flags & TAV_OUTPUTS_ON_DEVICE) ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    TAV_CUDA(cudaMemcpyAsync(out_items, static_cast<const int64_t*>(ix->range_items.p) + first,
                             static_cast<size_t>(n) * sizeof(int64_t), kind, s));
    TAV_CUDA(cudaMemcpyAsync(out_scores, static_cast<const float*>(ix->range_scores.p) + first,
                             static_cast<size_t>(n) * sizeof(float), kind, s));
    if (!(flags & TAV_OUTPUTS_ON_DEVICE)) TAV_CUDA(cudaStreamSynchronize(s));
    return TAV_OK;
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
    if (int rc = set_device(ix)) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    // staged as a search stages them: normalised on a TAV_NORMALIZE index, so these are the search's dots
    TimedSearch not_timed;
    const float* d_queries = nullptr;
    const int64_t* no_subset = nullptr;
    if (int rc = stage_inputs(ix, &not_timed, false, queries, n_queries, flags & TAV_QUERIES_ON_DEVICE, false, nullptr, 0,
                              &d_queries, &no_subset, s))
        return rc;
    if (split)
        if (int rc = ensure_split_planes(ix, nullptr, s)) return rc;
    MmaArgs m{};
    m.device = ix->device;
    m.corpus = split ? ix->split_hi.p : ix->rows;
    m.corpus_lo = split ? ix->split_lo.p : nullptr;
    m.split = split ? 1 : 0;
    m.split_overflow = split ? static_cast<int*>(ix->split_flag.p) + 1 : nullptr;
    m.dtype = ix->dtype;
    m.n_corpus = ix->size;
    m.dim = ix->dim;
    m.queries = d_queries;
    m.nq = n_queries;
    m.k = 1;
    const size_t ws = mma_workspace_bytes(m);
    if (ws > ix->mma_ws.bytes) {
        TAV_CUDA(cudaStreamSynchronize(s));
        TAV_CUDA(ix->mma_ws.ensure(ws));
        TAV_CUDA(cudaMemsetAsync(ix->mma_ws.p, 0, std::min<size_t>(ix->mma_ws.bytes, 65536), s));
    }
    TAV_CUDA(launch_mma_dump(m, ix->mma_ws.p, ix->mma_ws.bytes, out_device, s));
    TAV_CUDA(cudaStreamSynchronize(s));
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
        for (int h = 0; h < kHistory; ++h)
            for (auto& pr : ix->hist[h].ev) pr[0] = pr[1] = nullptr;
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
