// tav_multi.cu — one process, several devices (include/tavec.h, tav_multi_*): a row-sharded search over W
// borrowed tav_index shards, each holding one contiguous block of the rows on any device.  Every shard's search
// is launched on a stream of its own before anything waits, so the devices overlap; each shard's list is copied
// into a slab on the home device (cudaMemcpyPeerAsync), the home stream waits on the shards' events and merges
// with the library's merge kernels.  No process group, no CUDA IPC, no flags in peer memory: inside one process
// cross-device order is events and peer copies.

#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <mutex>
#include <new>
#include <string>
#include <vector>

#include "tav_common.cuh"
#include "tav_internal.h"

using tav::set_error;

namespace {

constexpr int kMultiMaxShards = 32;  // tav_merge_range's limit on lists
constexpr int kMultiMaxK = 4 * tav::kPassK;  // tav_merge_topk_ordered's limit on k
constexpr int kMultiFlags = TAV_FORCE_SCAN | TAV_FORCE_MMA | TAV_USE_ROW_MASK | TAV_TIES_LOW_FIRST;
constexpr int64_t kMultiMinRoom = 4096;  // hits a shard's threshold-search buffers hold at least

#define TAVM_CUDA(expr)                                                                        \
    do {                                                                                       \
        cudaError_t _e = (expr);                                                               \
        if (_e != cudaSuccess) {                                                               \
            set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return _e == cudaErrorMemoryAllocation ? TAV_ERR_OOM : TAV_ERR_CUDA;               \
        }                                                                                      \
    } while (0)

// grow-only memory on one device (device == -1: pinned host memory)
struct Buf {
    void* p = nullptr;
    size_t bytes = 0;
    Buf() = default;
    Buf(const Buf&) = delete;
    Buf& operator=(const Buf&) = delete;
    ~Buf() { release(); }
    int dev = -1;
    cudaError_t ensure(int device, size_t need) {
        if (p && dev == device && need <= bytes) return cudaSuccess;
        release();
        const size_t want = std::max(need, size_t(4096));
        cudaError_t e;
        if (device < 0) {
            e = cudaMallocHost(&p, want);
        } else {
            e = cudaSetDevice(device);
            if (e == cudaSuccess) e = cudaMalloc(&p, want);
        }
        if (e != cudaSuccess) {
            p = nullptr;
            cudaGetLastError();  // not sticky: the caller reports TAV_ERR_OOM and stays usable
            return e;
        }
        bytes = want;
        dev = device;
        return cudaSuccess;
    }
    void release() {
        if (p) (dev < 0 ? cudaFreeHost(p) : cudaFree(p));
        p = nullptr;
        bytes = 0;
    }
    template <class T>
    T* as() const { return static_cast<T*>(p); }
};

struct Shard {
    tav_index* ix = nullptr;
    int dev = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev = nullptr;
    Buf q;                        // the queries on the shard's device
    Buf items, scores, counts;    // top-k: its [B, k] list
    Buf offsets, hits, hit_scores;  // threshold: its CSR result
    int64_t room = 0;             // hits that hits / hit_scores hold
    int64_t total = 0;            // hits of its last threshold search
    std::vector<int64_t> pos;     // subset: positions of the share's entries in the caller's subset (ascending)
    std::vector<int64_t> local;   // ... and their block-local ordinals
};

// the first failure of a fan-out: its status and message, re-stated when the call returns
struct FirstError {
    int rc = TAV_OK;
    std::string msg;
    void note(int r) {
        if (r == TAV_OK || rc != TAV_OK) return;
        rc = r;
        const char* m = tav_last_error();
        msg = m ? m : "";
    }
    int give() const {
        if (rc != TAV_OK) set_error("%s", msg.c_str());
        return rc;
    }
};

// the caller's current device is restored on return
struct DeviceGuard {
    int prev = -1;
    DeviceGuard() {
        if (cudaGetDevice(&prev) != cudaSuccess) {
            cudaGetLastError();
            prev = -1;
        }
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

}  // namespace

struct tav_multi {
    std::mutex mu;
    int home = 0;
    int w = 0;
    cudaStream_t stream = nullptr;  // the home device's: merge and result copies
    Shard sh[kMultiMaxShards];
    Buf pin_q;                                   // pinned host copy of the queries
    Buf slab_items, slab_scores, slab_counts;    // top-k: W lists [B, k] on the home device
    Buf out_items, out_scores, out_counts;       // top-k: the merged [B, k]
    Buf slab_off, slab_hits, slab_hit_scores;    // threshold: W CSR results on the home device
    Buf res_off, res_items, res_scores;          // threshold: the merged result, until the next threshold search
    Buf pos_table, sub_table;                    // subset: the shares' positions, concatenated; the caller's subset
    int64_t res_total = 0;
};

namespace {

int sync_shards(tav_multi* m) {
    FirstError err;
    for (int g = 0; g < m->w; ++g) {
        cudaError_t e = cudaStreamSynchronize(m->sh[g].stream);
        if (e != cudaSuccess) {
            set_error("tav_multi: shard %d: %s", g, cudaGetErrorString(e));
            err.note(TAV_ERR_CUDA);
        }
    }
    return err.give();
}

// starts (host, W + 1) must describe the shards' blocks; flags must be the ones a multi-device search takes.
// *dim: the row width (0 when no shard has rows).
int check_layout(tav_multi* m, const char* fn, const int64_t* starts, int flags, int* dim) {
    if (flags & ~kMultiFlags) {
        set_error("%s: flags 0x%x are not available across devices", fn, flags & ~kMultiFlags);
        return TAV_ERR_INVALID;
    }
    if (starts[0] != 0) {
        set_error("%s: starts[0] is %lld, not 0", fn, (long long)starts[0]);
        return TAV_ERR_INVALID;
    }
    *dim = 0;
    for (int g = 0; g < m->w; ++g) {
        const int64_t rows = tav_size(m->sh[g].ix);
        if (starts[g + 1] - starts[g] != rows) {
            set_error("%s: block %d is rows [%lld, %lld), its shard holds %lld rows", fn, g, (long long)starts[g],
                      (long long)starts[g + 1], (long long)rows);
            return TAV_ERR_INVALID;
        }
        if (rows == 0) continue;
        const int d = tav_dim(m->sh[g].ix);
        if (*dim != 0 && d != *dim) {
            set_error("%s: shard %d has rows of %d elements, an earlier shard of %d", fn, g, d, *dim);
            return TAV_ERR_INVALID;
        }
        *dim = d;
    }
    return TAV_OK;
}

// The caller's subset split by block: numpy's IndexError for an ordinal outside [-N, N), before any work; negative
// ordinals wrap against the global row count N; a repeated ordinal is one entry per occurrence.
int split_subset(tav_multi* m, const int64_t* starts, const int64_t* subset, int64_t len) {
    const int64_t n = starts[m->w];
    for (int64_t i = 0; i < len; ++i)
        if (subset[i] < -n || subset[i] >= n) {
            set_error("index %lld is out of bounds for axis 0 with size %lld", (long long)subset[i], (long long)n);
            return TAV_ERR_RANGE;
        }
    for (int g = 0; g < m->w; ++g) {
        m->sh[g].pos.clear();
        m->sh[g].local.clear();
    }
    for (int64_t i = 0; i < len; ++i) {
        const int64_t r = subset[i] < 0 ? subset[i] + n : subset[i];
        const int g = static_cast<int>(std::upper_bound(starts + 1, starts + m->w + 1, r) - (starts + 1));
        m->sh[g].pos.push_back(i);
        m->sh[g].local.push_back(r - starts[g]);
    }
    return TAV_OK;
}

// the subset tables on the home device: the shares' global positions (concatenated, shard order) and the subset
int upload_subset(tav_multi* m, const int64_t* subset, int64_t len) {
    TAVM_CUDA(m->pos_table.ensure(m->home, static_cast<size_t>(len) * sizeof(int64_t)));
    TAVM_CUDA(m->sub_table.ensure(m->home, static_cast<size_t>(len) * sizeof(int64_t)));
    int64_t at = 0;
    for (int g = 0; g < m->w; ++g) {
        const size_t n = m->sh[g].pos.size();
        if (n)
            TAVM_CUDA(cudaMemcpyAsync(m->pos_table.as<int64_t>() + at, m->sh[g].pos.data(), n * sizeof(int64_t),
                                      cudaMemcpyHostToDevice, m->stream));
        at += static_cast<int64_t>(n);
    }
    if (len) TAVM_CUDA(cudaMemcpyAsync(m->sub_table.p, subset, static_cast<size_t>(len) * sizeof(int64_t),
                                       cudaMemcpyHostToDevice, m->stream));
    return TAV_OK;
}

// the shard's share-local positions in its slab list (n items) -> positions in the caller's subset
int map_share(tav_multi* m, int g, int64_t* items, int64_t n) {
    int64_t at = 0;
    for (int i = 0; i < g; ++i) at += static_cast<int64_t>(m->sh[i].pos.size());
    return tav_map_items(m->home, n, m->pos_table.as<int64_t>() + at, static_cast<int64_t>(m->sh[g].pos.size()), items,
                         m->stream);
}

// the shard's flags: an empty block returns nothing and has no row mask to name
int shard_flags(const Shard& s, int flags) {
    return tav_size(s.ix) == 0 ? flags & ~TAV_USE_ROW_MASK : flags;
}

int stage_queries(tav_multi* m, const float* queries, int nq, int dim) {
    const size_t bytes = static_cast<size_t>(nq) * dim * sizeof(float);
    TAVM_CUDA(m->pin_q.ensure(-1, bytes));
    memcpy(m->pin_q.p, queries, bytes);
    return TAV_OK;
}

int queries_to_shard(tav_multi* m, Shard& s, int nq, int dim) {
    const size_t bytes = static_cast<size_t>(nq) * dim * sizeof(float);
    TAVM_CUDA(s.q.ensure(s.dev, bytes));
    TAVM_CUDA(cudaSetDevice(s.dev));
    TAVM_CUDA(cudaMemcpyAsync(s.q.p, m->pin_q.p, bytes, cudaMemcpyHostToDevice, s.stream));
    return TAV_OK;
}

// completes every shard's deferred searches (the exact redo runs before anything is merged), whatever failed
int finish_shards(tav_multi* m, FirstError& err) {
    for (int g = 0; g < m->w; ++g) {
        int redone = 0;
        err.note(tav_finish_search(m->sh[g].ix, m->sh[g].stream, &redone));
    }
    if (err.rc != TAV_OK) {
        sync_shards(m);
        return err.give();
    }
    return TAV_OK;
}

// the home stream waits for the work queued on every shard stream so far
int join_home(tav_multi* m) {
    for (int g = 0; g < m->w; ++g) {
        TAVM_CUDA(cudaSetDevice(m->sh[g].dev));
        TAVM_CUDA(cudaEventRecord(m->sh[g].ev, m->sh[g].stream));
    }
    TAVM_CUDA(cudaSetDevice(m->home));
    for (int g = 0; g < m->w; ++g) TAVM_CUDA(cudaStreamWaitEvent(m->stream, m->sh[g].ev, 0));
    return TAV_OK;
}

int peer_copy(tav_multi* m, Shard& s, void* dst, const void* src, size_t bytes) {
    if (bytes == 0) return TAV_OK;
    TAVM_CUDA(cudaSetDevice(s.dev));
    TAVM_CUDA(cudaMemcpyPeerAsync(dst, m->home, src, s.dev, bytes, s.stream));
    return TAV_OK;
}

int multi_search_body(tav_multi* m, const int64_t* starts, const float* queries, int nq, int k, float min_score,
                      int flags, const int64_t* subset, int64_t subset_len, int64_t* out_items, float* out_scores,
                      int32_t* out_counts) {
    int dim = 0;
    if (int rc = check_layout(m, "tav_multi_search", starts, flags, &dim)) return rc;
    if (subset)
        if (int rc = split_subset(m, starts, subset, subset_len)) return rc;
    if (nq == 0) return TAV_OK;
    const int64_t n_scan = subset ? subset_len : starts[m->w];
    if (n_scan == 0 || dim == 0 || min_score != min_score) {
        memset(out_counts, 0, static_cast<size_t>(nq) * sizeof(int32_t));
        return TAV_OK;
    }
    if (int rc = stage_queries(m, queries, nq, dim)) return rc;
    const size_t list = static_cast<size_t>(nq) * k;
    const int64_t no_share = 0;  // the address an empty share names (TAV_ITEMS_AS_POSITIONS needs a subset)
    const int base = flags | TAV_QUERIES_ON_DEVICE | TAV_OUTPUTS_ON_DEVICE | TAV_DEFER_RETRY |
                     (subset ? TAV_ITEMS_AS_POSITIONS : 0);
    // fan out: every shard is launched before anything waits
    FirstError err;
    for (int g = 0; g < m->w && err.rc == TAV_OK; ++g) {
        Shard& s = m->sh[g];
        int rc = queries_to_shard(m, s, nq, dim);
        if (rc == TAV_OK && (s.items.ensure(s.dev, list * sizeof(int64_t)) != cudaSuccess ||
                             s.scores.ensure(s.dev, list * sizeof(float)) != cudaSuccess ||
                             s.counts.ensure(s.dev, static_cast<size_t>(nq) * sizeof(int32_t)) != cudaSuccess)) {
            set_error("tav_multi_search: shard %d: its [%d, %d] list does not fit in device memory", g, nq, k);
            rc = TAV_ERR_OOM;
        }
        if (rc == TAV_OK)
            rc = tav_search(s.ix, s.q.as<float>(), nq, k, min_score, shard_flags(s, base),
                            subset ? (s.local.empty() ? &no_share : s.local.data()) : nullptr,
                            subset ? static_cast<int64_t>(s.local.size()) : 0, subset ? 0 : starts[g],
                            s.items.as<int64_t>(), s.scores.as<float>(), s.counts.as<int32_t>(), s.stream);
        err.note(rc);
    }
    if (int rc = finish_shards(m, err)) return rc;
    // gather on the home device
    TAVM_CUDA(m->slab_items.ensure(m->home, m->w * list * sizeof(int64_t)));
    TAVM_CUDA(m->slab_scores.ensure(m->home, m->w * list * sizeof(float)));
    TAVM_CUDA(m->slab_counts.ensure(m->home, static_cast<size_t>(m->w) * nq * sizeof(int32_t)));
    TAVM_CUDA(m->out_items.ensure(m->home, list * sizeof(int64_t)));
    TAVM_CUDA(m->out_scores.ensure(m->home, list * sizeof(float)));
    TAVM_CUDA(m->out_counts.ensure(m->home, static_cast<size_t>(nq) * sizeof(int32_t)));
    for (int g = 0; g < m->w; ++g) {
        Shard& s = m->sh[g];
        if (int rc = peer_copy(m, s, m->slab_items.as<int64_t>() + g * list, s.items.p, list * sizeof(int64_t))) return rc;
        if (int rc = peer_copy(m, s, m->slab_scores.as<float>() + g * list, s.scores.p, list * sizeof(float))) return rc;
        if (int rc = peer_copy(m, s, m->slab_counts.as<int32_t>() + static_cast<size_t>(g) * nq, s.counts.p,
                               static_cast<size_t>(nq) * sizeof(int32_t)))
            return rc;
    }
    if (int rc = join_home(m)) return rc;
    const bool ties_low = flags & TAV_TIES_LOW_FIRST;
    int order = ties_low ? 1 : 0;  // equal scores: higher row first, as one index orders them (lower with ties-low)
    if (subset) {
        // positions are distinct: merged by position, later entry first as one index orders a subset's ties
        order = ties_low ? 3 : 2;
        if (int rc = upload_subset(m, subset, subset_len)) return rc;
        for (int g = 0; g < m->w; ++g)
            if (int rc = map_share(m, g, m->slab_items.as<int64_t>() + g * list, static_cast<int64_t>(list))) return rc;
    }
    if (int rc = tav_merge_topk_ordered(m->home, m->w, nq, k, m->slab_items.as<int64_t>(), m->slab_scores.as<float>(),
                                        m->slab_counts.as<int32_t>(), static_cast<int64_t>(list),
                                        static_cast<int64_t>(list), nq, order, m->out_items.as<int64_t>(),
                                        m->out_scores.as<float>(), m->out_counts.as<int32_t>(), m->stream))
        return rc;
    if (subset)
        if (int rc = tav_map_items(m->home, static_cast<int64_t>(list), m->sub_table.as<int64_t>(), subset_len,
                                   m->out_items.as<int64_t>(), m->stream))
            return rc;
    TAVM_CUDA(cudaMemcpyAsync(out_items, m->out_items.p, list * sizeof(int64_t), cudaMemcpyDeviceToHost, m->stream));
    TAVM_CUDA(cudaMemcpyAsync(out_scores, m->out_scores.p, list * sizeof(float), cudaMemcpyDeviceToHost, m->stream));
    TAVM_CUDA(cudaMemcpyAsync(out_counts, m->out_counts.p, static_cast<size_t>(nq) * sizeof(int32_t),
                              cudaMemcpyDeviceToHost, m->stream));
    TAVM_CUDA(cudaStreamSynchronize(m->stream));
    return TAV_OK;
}

int ensure_room(Shard& s, int nq, int64_t room) {
    TAVM_CUDA(s.offsets.ensure(s.dev, (static_cast<size_t>(nq) + 1) * sizeof(int64_t)));
    if (room > s.room || !s.hits.p || !s.hit_scores.p) {
        TAVM_CUDA(s.hits.ensure(s.dev, static_cast<size_t>(room) * sizeof(int64_t)));
        TAVM_CUDA(s.hit_scores.ensure(s.dev, static_cast<size_t>(room) * sizeof(float)));
        s.room = std::max(room, s.room);
    }
    return TAV_OK;
}

// one shard's threshold search into its own buffers: tav_range_search_into over its block (items global), or, with a
// subset, tav_range_search of its share with TAV_ITEMS_AS_POSITIONS, whose hits are fetched into the buffers (that
// form synchronises; its items are share-local positions)
int range_shard(tav_multi* m, int g, const int64_t* starts, int nq, int dim, float min_score, int flags, bool subset,
                int64_t hint, bool defer) {
    Shard& s = m->sh[g];
    if (!subset) {
        if (int rc = queries_to_shard(m, s, nq, dim)) return rc;
        if (int rc = ensure_room(s, nq, std::max(s.room, std::max(hint, kMultiMinRoom)))) return rc;
        return tav_range_search_into(s.ix, s.q.as<float>(), nq, min_score,
                                     shard_flags(s, flags) | TAV_QUERIES_ON_DEVICE | (defer ? TAV_DEFER_RETRY : 0),
                                     nullptr, 0, starts[g], hint, s.room, s.offsets.as<int64_t>(), s.hits.as<int64_t>(),
                                     s.hit_scores.as<float>(), s.stream);
    }
    if (int rc = ensure_room(s, nq, std::max(s.room, kMultiMinRoom))) return rc;
    std::vector<int64_t> off(static_cast<size_t>(nq) + 1, 0);
    if (!s.local.empty()) {
        if (int rc = tav_range_search(s.ix, m->pin_q.as<float>(), nq, min_score, flags | TAV_ITEMS_AS_POSITIONS,
                                      s.local.data(), static_cast<int64_t>(s.local.size()), 0, hint, off.data(), s.stream))
            return rc;
        if (int rc = ensure_room(s, nq, off[nq])) return rc;
        if (int rc = tav_range_fetch(s.ix, 0, off[nq], s.hits.as<int64_t>(), s.hit_scores.as<float>(),
                                     TAV_OUTPUTS_ON_DEVICE, s.stream))
            return rc;
    }
    TAVM_CUDA(cudaSetDevice(s.dev));
    TAVM_CUDA(cudaMemcpyAsync(s.offsets.p, off.data(), off.size() * sizeof(int64_t), cudaMemcpyHostToDevice, s.stream));
    TAVM_CUDA(cudaStreamSynchronize(s.stream));  // `off` is a local
    return TAV_OK;
}

int multi_range_body(tav_multi* m, const int64_t* starts, const float* queries, int nq, float min_score, int flags,
                     const int64_t* subset, int64_t subset_len, int64_t expected_hits, int64_t* out_offsets) {
    int dim = 0;
    if (int rc = check_layout(m, "tav_multi_range_search", starts, flags, &dim)) return rc;
    if (subset)
        if (int rc = split_subset(m, starts, subset, subset_len)) return rc;
    memset(out_offsets, 0, (static_cast<size_t>(nq) + 1) * sizeof(int64_t));
    const int64_t n_scan = subset ? subset_len : starts[m->w];
    if (nq == 0 || n_scan == 0 || dim == 0 || min_score != min_score) return TAV_OK;
    if (int rc = stage_queries(m, queries, nq, dim)) return rc;
    // each shard's share of the hint: the shares are rarely even, so twice the even share
    const int64_t hint = expected_hits > 0 ? 2 * ((expected_hits + m->w - 1) / m->w) : 0;
    FirstError err;
    for (int g = 0; g < m->w && err.rc == TAV_OK; ++g)
        err.note(range_shard(m, g, starts, nq, dim, min_score, flags, subset != nullptr, hint, true));
    if (int rc = finish_shards(m, err)) return rc;
    // every shard's total; a shard whose hits did not all fit is searched again with room for them
    for (int g = 0; g < m->w; ++g) {
        Shard& s = m->sh[g];
        TAVM_CUDA(cudaSetDevice(s.dev));
        TAVM_CUDA(cudaMemcpyAsync(&s.total, s.offsets.as<int64_t>() + nq, sizeof(int64_t), cudaMemcpyDeviceToHost,
                                  s.stream));
    }
    if (int rc = sync_shards(m)) return rc;
    for (int g = 0; g < m->w; ++g) {
        Shard& s = m->sh[g];
        if (s.total <= s.room) continue;  // a subset's share is always fetched whole
        if (int rc = ensure_room(s, nq, s.total)) return rc;
        const int rc = range_shard(m, g, starts, nq, dim, min_score, flags, false, hint, false);
        if (rc != TAV_OK) {
            sync_shards(m);
            return rc;
        }
        TAVM_CUDA(cudaMemcpy(&s.total, s.offsets.as<int64_t>() + nq, sizeof(int64_t), cudaMemcpyDeviceToHost));
    }
    int64_t total = 0, widest = 1;
    for (int g = 0; g < m->w; ++g) {
        total += m->sh[g].total;
        widest = std::max(widest, m->sh[g].total);
    }
    const size_t offs = static_cast<size_t>(nq) + 1;
    TAVM_CUDA(m->slab_off.ensure(m->home, m->w * offs * sizeof(int64_t)));
    TAVM_CUDA(m->slab_hits.ensure(m->home, m->w * static_cast<size_t>(widest) * sizeof(int64_t)));
    TAVM_CUDA(m->slab_hit_scores.ensure(m->home, m->w * static_cast<size_t>(widest) * sizeof(float)));
    TAVM_CUDA(m->res_off.ensure(m->home, offs * sizeof(int64_t)));
    TAVM_CUDA(m->res_items.ensure(m->home, static_cast<size_t>(total) * sizeof(int64_t)));
    TAVM_CUDA(m->res_scores.ensure(m->home, static_cast<size_t>(total) * sizeof(float)));
    for (int g = 0; g < m->w; ++g) {
        Shard& s = m->sh[g];
        const size_t n = static_cast<size_t>(s.total);
        if (int rc = peer_copy(m, s, m->slab_off.as<int64_t>() + g * offs, s.offsets.p, offs * sizeof(int64_t))) return rc;
        if (int rc = peer_copy(m, s, m->slab_hits.as<int64_t>() + g * widest, s.hits.p, n * sizeof(int64_t))) return rc;
        if (int rc = peer_copy(m, s, m->slab_hit_scores.as<float>() + g * widest, s.hit_scores.p, n * sizeof(float)))
            return rc;
    }
    if (int rc = join_home(m)) return rc;
    if (subset) {
        if (int rc = upload_subset(m, subset, subset_len)) return rc;
        for (int g = 0; g < m->w; ++g)
            if (int rc = map_share(m, g, m->slab_hits.as<int64_t>() + g * widest, m->sh[g].total)) return rc;
    }
    if (int rc = tav_merge_range(m->home, m->w, nq, m->slab_off.as<int64_t>(), static_cast<int64_t>(offs),
                                 m->slab_hits.as<int64_t>(), widest, m->slab_hit_scores.as<float>(), widest,
                                 (flags & TAV_TIES_LOW_FIRST) ? 1 : 0, m->res_off.as<int64_t>(),
                                 m->res_items.as<int64_t>(), m->res_scores.as<float>(), m->stream))
        return rc;
    if (subset)
        if (int rc = tav_map_items(m->home, total, m->sub_table.as<int64_t>(), subset_len, m->res_items.as<int64_t>(),
                                   m->stream))
            return rc;
    TAVM_CUDA(cudaMemcpyAsync(out_offsets, m->res_off.p, offs * sizeof(int64_t), cudaMemcpyDeviceToHost, m->stream));
    TAVM_CUDA(cudaStreamSynchronize(m->stream));
    m->res_total = total;
    return TAV_OK;
}

}  // namespace

extern "C" {

int tav_multi_destroy(tav_multi* m) {
    if (!m) return TAV_OK;
    DeviceGuard guard;
    for (int g = 0; g < m->w; ++g) {
        Shard& s = m->sh[g];
        cudaSetDevice(s.dev);
        if (s.stream) {
            cudaStreamSynchronize(s.stream);
            cudaStreamDestroy(s.stream);
        }
        if (s.ev) cudaEventDestroy(s.ev);
    }
    if (m->stream) {
        cudaSetDevice(m->home);
        cudaStreamSynchronize(m->stream);
        cudaStreamDestroy(m->stream);
    }
    delete m;
    return TAV_OK;
}

int tav_multi_create(int home_device, int n_shards, tav_index* const* shards, tav_multi** out) {
    if (!out || !shards || n_shards < 1 || n_shards > kMultiMaxShards) {
        set_error("tav_multi_create: invalid argument (1 to %d shards)", kMultiMaxShards);
        return TAV_ERR_INVALID;
    }
    *out = nullptr;
    for (int g = 0; g < n_shards; ++g) {
        if (!shards[g]) {
            set_error("tav_multi_create: shard %d is NULL", g);
            return TAV_ERR_INVALID;
        }
        for (int h = 0; h < g; ++h)
            if (shards[h] == shards[g]) {
                set_error("tav_multi_create: shards %d and %d are the same index", h, g);
                return TAV_ERR_INVALID;
            }
    }
    int n_dev = 0;
    cudaError_t e = cudaGetDeviceCount(&n_dev);
    if (e != cudaSuccess || n_dev == 0) {
        cudaGetLastError();
        set_error("tav_multi_create: no CUDA device available; libtavec has no CPU fallback");
        return TAV_ERR_CUDA;
    }
    if (home_device < 0 || home_device >= n_dev) {
        set_error("tav_multi_create: device %d out of range (have %d)", home_device, n_dev);
        return TAV_ERR_INVALID;
    }
    DeviceGuard guard;
    tav_multi* m = new (std::nothrow) tav_multi();
    if (!m) return TAV_ERR_OOM;
    m->home = home_device;
    std::vector<int> devs{home_device};
    auto fail = [&](cudaError_t err, const char* what) {
        set_error("tav_multi_create: %s: %s", what, cudaGetErrorString(err));
        cudaGetLastError();
        tav_multi_destroy(m);
        return err == cudaErrorMemoryAllocation ? TAV_ERR_OOM : TAV_ERR_CUDA;
    };
    for (int g = 0; g < n_shards; ++g) {
        Shard& s = m->sh[g];
        s.ix = shards[g];
        s.dev = tav_device(s.ix);
        m->w = g + 1;  // destroy releases what exists so far
        if ((e = cudaSetDevice(s.dev)) != cudaSuccess) return fail(e, "cudaSetDevice");
        if ((e = cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking)) != cudaSuccess)
            return fail(e, "stream creation");
        if ((e = cudaEventCreateWithFlags(&s.ev, cudaEventDisableTiming)) != cudaSuccess)
            return fail(e, "event creation");
        if (std::find(devs.begin(), devs.end(), s.dev) == devs.end()) devs.push_back(s.dev);
    }
    if ((e = cudaSetDevice(home_device)) != cudaSuccess) return fail(e, "cudaSetDevice");
    if ((e = cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking)) != cudaSuccess)
        return fail(e, "stream creation");
    // peer access between the distinct devices, where the hardware allows it (else the copies go through the host)
    for (int a : devs)
        for (int b : devs) {
            if (a == b) continue;
            int can = 0;
            if ((e = cudaDeviceCanAccessPeer(&can, a, b)) != cudaSuccess) return fail(e, "cudaDeviceCanAccessPeer");
            if (!can) continue;
            if ((e = cudaSetDevice(a)) != cudaSuccess) return fail(e, "cudaSetDevice");
            e = cudaDeviceEnablePeerAccess(b, 0);
            if (e == cudaErrorPeerAccessAlreadyEnabled) {
                cudaGetLastError();
            } else if (e != cudaSuccess) {
                return fail(e, "cudaDeviceEnablePeerAccess");
            }
        }
    *out = m;
    return TAV_OK;
}

int tav_multi_search(tav_multi* m, const int64_t* starts, const float* queries, int n_queries, int k, float min_score,
                     int flags, const int64_t* subset, int64_t subset_len, int64_t* out_items, float* out_scores,
                     int32_t* out_counts) {
    if (!m || !starts || n_queries < 0 || k < 1 || subset_len < 0 || (!subset && subset_len != 0) ||
        (n_queries > 0 && (!queries || !out_items || !out_scores || !out_counts))) {
        set_error("tav_multi_search: invalid argument (k must be >= 1)");
        return TAV_ERR_INVALID;
    }
    if (k > kMultiMaxK) {
        set_error("tav_multi_search: k = %d above %d; tav_multi_range_search returns every hit", k, kMultiMaxK);
        return TAV_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lock(m->mu);
    DeviceGuard guard;
    return multi_search_body(m, starts, queries, n_queries, k, min_score, flags, subset, subset_len, out_items,
                             out_scores, out_counts);
}

int tav_multi_range_search(tav_multi* m, const int64_t* starts, const float* queries, int n_queries, float min_score,
                           int flags, const int64_t* subset, int64_t subset_len, int64_t expected_hits,
                           int64_t* out_offsets) {
    if (!m || !starts || n_queries < 0 || expected_hits < 0 || !out_offsets || subset_len < 0 ||
        (!subset && subset_len != 0) || (n_queries > 0 && !queries)) {
        set_error("tav_multi_range_search: invalid argument");
        return TAV_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lock(m->mu);
    DeviceGuard guard;
    m->res_total = 0;
    return multi_range_body(m, starts, queries, n_queries, min_score, flags, subset, subset_len, expected_hits,
                            out_offsets);
}

int tav_multi_range_fetch(tav_multi* m, int64_t first, int64_t n, int64_t* out_items, float* out_scores) {
    if (!m || first < 0 || n < 0 || (n > 0 && (!out_items || !out_scores))) {
        set_error("tav_multi_range_fetch: invalid argument");
        return TAV_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lock(m->mu);
    if (first + n > m->res_total) {
        set_error("tav_multi_range_fetch: hits [%lld, %lld) out of range (the last range search has %lld)",
                  (long long)first, (long long)(first + n), (long long)m->res_total);
        return TAV_ERR_RANGE;
    }
    if (n == 0) return TAV_OK;
    DeviceGuard guard;
    TAVM_CUDA(cudaSetDevice(m->home));
    TAVM_CUDA(cudaMemcpyAsync(out_items, m->res_items.as<int64_t>() + first, static_cast<size_t>(n) * sizeof(int64_t),
                              cudaMemcpyDeviceToHost, m->stream));
    TAVM_CUDA(cudaMemcpyAsync(out_scores, m->res_scores.as<float>() + first, static_cast<size_t>(n) * sizeof(float),
                              cudaMemcpyDeviceToHost, m->stream));
    TAVM_CUDA(cudaStreamSynchronize(m->stream));
    return TAV_OK;
}

}  // extern "C"
