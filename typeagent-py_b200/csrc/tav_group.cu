// tav_group.cu — the row-sharded search of libtavec over the GPUs of one NVSwitch box
// (include/tavec.h: tav_group_*, tav_sharded_search, tav_sharded_finish; SURVEY.md §8e).
//
// The reference has one VectorBase over the whole corpus (aitools/vectorbase.py:163-201); sharded,
// every rank searches its contiguous row block and the per-rank [B, k] candidate lists are merged
// (top-k is a decomposable reduction).  The exchange is NOT a library collective: every rank owns an
// "exchange region" in its HBM, exported to its peers as a CUDA IPC handle; after the local search a
// PUBLISH kernel stores this rank's packed list straight into every peer's region over NVLink (plain
// st.global on peer-mapped pointers) and raises a sequence flag with a system-scope release; the MERGE
// kernel of every rank spins (acquire) until all ranks' flags reached the search's sequence number,
// merges the world's lists from its own HBM and — its last CTA — acknowledges to the peers, so that a
// slot is never overwritten while a slower rank still reads it: two launches per exchange, no NCCL call,
// no host synchronisation.  Pipelined (TAV_DEFER_RETRY) searches run the exchange on the group's own
// stream behind an event, so that the next search's kernels do not queue behind the wait for the slowest
// rank.  One process per GPU; the handles travel once, through whatever the host side has
// (torch.distributed.all_gather_object in the Python class).
//
// Region layout (device memory of the owning rank):
//   arrive[world]  u32   arrive[r] = sequence number of the last search rank r PUBLISHED here
//   ack[world]     u32   ack[r]    = sequence number of the last search rank r MERGED (it no longer
//                                    reads what this rank published for it)
//   slots[depth][world][slot_bytes]   packed lists [items i64 | scores f32 | counts i32 | tail] (8-byte
//                                    aligned sections, the layout ShardedVectorBase always used; tail word
//                                    0 = queries the rank's exact redo will still correct at finish, word 1 =
//                                    status: 1 when the rank's local search failed and it published no hits)
// `depth` searches may be in flight (deferred) before a rank has to wait for its peers' acks.
//
// Failure protocol.  A rank whose local search fails on the host side (an invalid argument, a missing mask, an
// allocation: any status but TAV_ERR_CUDA) still publishes, an empty list with status 1, and merges, so that no
// peer waits for it; its call returns its own error.  Every merge adds the world's status words up into a mapped
// host word per slot, and every rank reports TAV_ERR_PEER for a search whose sum is not zero: a synchronous call
// on return, a deferred one at tav_sharded_finish.  A CUDA error cannot be published (the device may be unusable):
// the call returns without publishing and its peers' waits end in the ~4 s trap of spin_until.

#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <new>
#include <string>
#include <vector>

#include "tav_common.cuh"
#include "tav_internal.h"

namespace tav {

namespace {

constexpr int kMaxWorld = 16;

struct PeerTable {
    char* region[kMaxWorld];  // region[r] = base of rank r's exchange region as mapped in THIS process
};

// Publish: this rank's packed list (already in its own slot of its own region) -> the same slot in
// every peer's region, then arrive[me] = seq everywhere.  Waits first until every peer acknowledged
// the search that used this slot `depth` searches ago.
// The last 16 bytes of a slot are its tail: word 0 = number of this rank's queries that its exact redo
// will still correct at finish (read here from the local search's device counters and, for a split search,
// the index's corpus flag), exactly the number tav_finish_search will redo; word 1 = `status`.
__global__ void __launch_bounds__(256)
publish_kernel(PeerTable peers, int me, int world, size_t off_ack, size_t off_slot, size_t bytes, uint32_t seq,
               uint32_t need_ack, uint32_t* ticket, const int32_t* retry_totals, int n_retry, const int* corpus_flag,
               int nq, uint32_t status) {
    __shared__ int s_last;
    const char* src = peers.region[me] + off_slot;
    if (blockIdx.x == 0 && threadIdx.x < world && threadIdx.x != me) {
        // ack[r] lives in MY region, written by rank r
        spin_until(reinterpret_cast<const uint32_t*>(peers.region[me] + off_ack) + threadIdx.x, need_ack);
    }
    // every CTA needs the acks before it overwrites peer slots: CTA 0 spins, the others wait on it via
    // the ticket's high bit (set by CTA 0 once the acks are in)
    if (blockIdx.x == 0) {
        __syncthreads();
        if (threadIdx.x == 0) atomicOr(ticket, 0x80000000u);
    } else if (threadIdx.x == 0) {
        const long long t0 = clock64();
        while (!(atomicAdd(ticket, 0u) & 0x80000000u)) {
            if (clock64() - t0 > kSpinLimit) __trap();
            __nanosleep(32);
        }
    }
    __syncthreads();
    if (blockIdx.x == 0 && threadIdx.x < world) {
        // per bookkeeping slot (a slab of up to kMmaMaxQueries queries): its flagged queries, or all of them when
        // the split form left the fp16 range in the corpus or in one of its queries (finish then redoes the slab)
        const bool corpus_out = corpus_flag && __ldcg(corpus_flag);
        uint32_t flagged = 0;
        for (int i = 0; i < n_retry; ++i) {
            const int slab = min(kMmaMaxQueries, nq - i * kMmaMaxQueries);
            flagged += static_cast<uint32_t>(corpus_out || __ldcg(&retry_totals[2 * i + 1]) ? slab
                                                                                          : __ldcg(&retry_totals[2 * i]));
        }
        uint32_t* tail = reinterpret_cast<uint32_t*>(peers.region[threadIdx.x] + off_slot + bytes - 16);
        tail[0] = TAV_GROUP_MUTANT == 1 ? 0u : flagged;
        tail[1] = status;
    }
    // sections are padded to 16 bytes by the host side; the tail goes separately
    const size_t n16 = (bytes - 16) / 16 - (TAV_GROUP_MUTANT == 2 ? 1 : 0);
    for (int w = 0; w < world; ++w) {
        if (w == me) continue;
        uint4* dst = reinterpret_cast<uint4*>(peers.region[w] + off_slot);
        const uint4* s4 = reinterpret_cast<const uint4*>(src);
        for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n16;
             i += static_cast<size_t>(gridDim.x) * blockDim.x)
            dst[i] = s4[i];
    }
    // ONE system-scope fence per CTA, by the thread that takes the ticket: the barrier orders the CTA's peer
    // stores before it (a membar.sys in each of the 32k threads was most of this kernel's time)
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence_system();
        const uint32_t t = atomicAdd(ticket, 1u) & 0x7FFFFFFFu;
        s_last = t == gridDim.x - 1;
    }
    __syncthreads();
    if (s_last) {
        if (threadIdx.x < world) {
            __threadfence_system();
            st_release_sys(reinterpret_cast<uint32_t*>(peers.region[threadIdx.x]) + me, seq);  // arrive[me] at rank w
        }
        if (threadIdx.x == 0) *ticket = 0;
    }
}

}  // namespace

}  // namespace tav

using namespace tav;

struct tav_group {
    int device = 0, rank = 0, world = 1, depth = 2;
    int max_queries = 0, max_k = 0;
    size_t slot_bytes = 0, off_ack = 0, off_slots = 0, region_bytes = 0;
    char* region = nullptr;           // this rank's exchange region (cudaMalloc)
    PeerTable peers{};                // region of every rank, as mapped here
    bool connected = false;
    uint32_t seq = 0;                 // searches published so far
    uint32_t* ticket = nullptr;       // device counter of the publish kernel
    uint32_t* flagged_host = nullptr; // pinned, mapped: [depth] world-wide "still to be corrected" counts per slot
    uint32_t* status_host = nullptr;  // pinned, mapped: [depth] world-wide sums of the status words per slot
    // Deferred searches run their exchange (publish + merge) on the group's own stream, behind an event that
    // follows the local search: the next search's kernels start at once on the caller's stream and the wait
    // for the slowest rank no longer sits between two searches.  tav_sharded_finish joins the streams.
    cudaStream_t xstream = nullptr;
    cudaEvent_t ev_local[64] = {};    // [depth] local search of the slot's search done (caller's stream)
    cudaEvent_t ev_merged[64] = {};   // [depth] merged result complete (exchange stream)
    bool x_pending = false;           // something was enqueued on xstream since the last join
    struct OpenSearch {               // a deferred search since the last finish: what a re-merge needs
        uint32_t seq;
        int nq, k;
        int order;                    // the merge's order (tav_merge_topk_ordered): a repair merges in it again
        uint32_t status;              // this rank's status word (1: its local search failed)
        int64_t* items;
        float* scores;
        int32_t* counts;
    };
    std::vector<OpenSearch> open;     // ascending, consecutive sequence numbers ending at `seq`
    int outstanding = 0;              // deferred sharded searches since the last finish
};

static inline size_t a16(size_t v) { return (v + 15) & ~size_t(15); }
static inline size_t a8(size_t v) { return (v + 7) & ~size_t(7); }

// the packed layout of one rank's list (as typeagent_py_b200/sharded.py:packed_layout), padded to 16 bytes
static void packed_offsets(int nq, int k, size_t* off_scores, size_t* off_counts, size_t* total) {
    *off_scores = a8(static_cast<size_t>(nq) * k * 8);
    *off_counts = *off_scores + a8(static_cast<size_t>(nq) * k * 4);
    *total = a16(*off_counts + a8(static_cast<size_t>(nq) * 4)) + 16;  // + the tail
}

#define TAVG_CUDA(expr)                                                                            \
    do {                                                                                           \
        cudaError_t _e = (expr);                                                                   \
        if (_e != cudaSuccess) {                                                                   \
            set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return _e == cudaErrorMemoryAllocation ? TAV_ERR_OOM : TAV_ERR_CUDA;                   \
        }                                                                                          \
    } while (0)

extern "C" {

int tav_group_handle_bytes(void) { return static_cast<int>(sizeof(cudaIpcMemHandle_t)); }

int tav_group_create(int device, int rank, int world, int max_queries, int max_k, int depth, tav_group** out) {
    if (!out || world < 1 || world > kMaxWorld || rank < 0 || rank >= world || max_queries < 1 || max_k < 1 ||
        depth < 1 || depth > 64) {
        set_error("tav_group_create: invalid argument (world <= %d, depth 1..64)", kMaxWorld);
        return TAV_ERR_INVALID;
    }
    TAVG_CUDA(cudaSetDevice(device));
    tav_group* g = new (std::nothrow) tav_group();
    if (!g) return TAV_ERR_OOM;
    g->device = device;
    g->rank = rank;
    g->world = world;
    g->depth = depth;
    g->max_queries = max_queries;
    g->max_k = max_k;
    size_t os, oc;
    packed_offsets(max_queries, max_k, &os, &oc, &g->slot_bytes);
    g->off_ack = a16(static_cast<size_t>(world) * 4);
    g->off_slots = (g->off_ack + a16(static_cast<size_t>(world) * 4) + 255) & ~size_t(255);
    g->region_bytes = g->off_slots + static_cast<size_t>(depth) * world * g->slot_bytes;
    cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&g->region), g->region_bytes);
    if (e == cudaSuccess) e = cudaMemset(g->region, 0, g->off_slots);
    if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void**>(&g->ticket), 64);
    if (e == cudaSuccess) e = cudaMemset(g->ticket, 0, 64);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&g->xstream, cudaStreamNonBlocking);
    for (int i = 0; e == cudaSuccess && i < depth; ++i) {
        e = cudaEventCreateWithFlags(&g->ev_local[i], cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&g->ev_merged[i], cudaEventDisableTiming);
    }
    if (e == cudaSuccess) e = cudaMallocHost(reinterpret_cast<void**>(&g->flagged_host), 2 * 64 * sizeof(uint32_t));
    if (e == cudaSuccess) {
        memset(g->flagged_host, 0, 2 * 64 * sizeof(uint32_t));
        g->status_host = g->flagged_host + 64;
    }
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
        set_error("tav_group_create: %s", cudaGetErrorString(e));
        tav_group_destroy(g);
        return e == cudaErrorMemoryAllocation ? TAV_ERR_OOM : TAV_ERR_CUDA;
    }
    g->peers.region[rank] = g->region;
    g->connected = world == 1;
    *out = g;
    return TAV_OK;
}

int tav_group_local_handle(tav_group* g, void* handle_out) {
    if (!g || !handle_out) return TAV_ERR_INVALID;
    TAVG_CUDA(cudaSetDevice(g->device));
    cudaIpcMemHandle_t h;
    TAVG_CUDA(cudaIpcGetMemHandle(&h, g->region));
    memcpy(handle_out, &h, sizeof(h));
    return TAV_OK;
}

int tav_group_connect(tav_group* g, const void* handles) {
    if (!g || !handles) return TAV_ERR_INVALID;
    TAVG_CUDA(cudaSetDevice(g->device));
    for (int r = 0; r < g->world; ++r) {
        if (r == g->rank) continue;
        cudaIpcMemHandle_t h;
        memcpy(&h, static_cast<const char*>(handles) + static_cast<size_t>(r) * sizeof(h), sizeof(h));
        void* p = nullptr;
        TAVG_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
        g->peers.region[r] = static_cast<char*>(p);
    }
    g->connected = true;
    return TAV_OK;
}

int tav_group_destroy(tav_group* g) {
    if (!g) return TAV_OK;
    cudaSetDevice(g->device);
    cudaDeviceSynchronize();
    for (int r = 0; r < g->world; ++r)
        if (r != g->rank && g->peers.region[r]) cudaIpcCloseMemHandle(g->peers.region[r]);
    if (g->region) cudaFree(g->region);
    if (g->ticket) cudaFree(g->ticket);
    if (g->flagged_host) cudaFreeHost(g->flagged_host);
    for (int i = 0; i < 64; ++i) {
        if (g->ev_local[i]) cudaEventDestroy(g->ev_local[i]);
        if (g->ev_merged[i]) cudaEventDestroy(g->ev_merged[i]);
    }
    if (g->xstream) cudaStreamDestroy(g->xstream);
    delete g;
    return TAV_OK;
}

int tav_group_capacity(const tav_group* g, int* max_queries, int* max_k, int* depth) {
    if (!g) return TAV_ERR_INVALID;
    if (max_queries) *max_queries = g->max_queries;
    if (max_k) *max_k = g->max_k;
    if (depth) *depth = g->depth;
    return TAV_OK;
}

// exchange + merge of the list this rank holds in its own slot for sequence number `seq`
static int publish_and_merge(tav_group* g, int nq, int k, uint32_t seq, int order, uint32_t status,
                             const int32_t* retry_totals, int n_retry, const int* corpus_flag, int64_t* out_items,
                             float* out_scores, int32_t* out_counts, cudaStream_t s) {
    const int slot = static_cast<int>(seq % static_cast<uint32_t>(g->depth));
    size_t off_scores, off_counts, bytes;
    packed_offsets(nq, k, &off_scores, &off_counts, &bytes);
    const size_t off_mine = g->off_slots + (static_cast<size_t>(slot) * g->world + g->rank) * g->slot_bytes;
    if (g->world > 1) {
        // enough CTAs to keep the NVLink stores in flight (2.1 MB at B = 256, k = 100 over 8 ranks): one per 2 KB
        const int grid = static_cast<int>(std::min<size_t>(128, std::max<size_t>(1, bytes / 2048)));
        // the slot was last used by search seq - depth: every peer must have merged that one
        const uint32_t need_ack = seq - static_cast<uint32_t>(g->depth);
        const uint32_t need = seq > static_cast<uint32_t>(g->depth) ? need_ack : 0u;
        publish_kernel<<<grid, 256, 0, s>>>(g->peers, g->rank, g->world, g->off_ack, off_mine, bytes, seq, need,
                                            g->ticket, retry_totals, retry_totals ? n_retry : 0, corpus_flag, nq,
                                            status);
        TAVG_CUDA(cudaGetLastError());
    }
    // lists of all ranks for this slot lie side by side in MY region: strides between ranks = slot_bytes.
    // The merge itself waits for every rank's publish (acquire spin on the arrive words), and its last CTA
    // acknowledges to the peers and sums the slot tails: no separate wait / ack launches.
    const char* base = g->region + g->off_slots + static_cast<size_t>(slot) * g->world * g->slot_bytes;
    MergeSync sync{};
    if (g->world > 1) {
        sync.arrive = reinterpret_cast<const uint32_t*>(g->region);
        sync.world = g->world;
        sync.seq = seq;
        for (int w = 0; w < g->world; ++w)
            sync.ack[w] = reinterpret_cast<uint32_t*>(g->peers.region[w] + g->off_ack) + g->rank;
        sync.me = g->rank;
        sync.ticket = g->ticket + 8;
        sync.tails = base + bytes - 16;
        sync.slot_bytes = g->slot_bytes;
        sync.flagged_host = g->flagged_host + slot;
        sync.status_host = g->status_host + slot;
    }
    TAVG_CUDA(launch_merge_ordered(g->world, nq, k, reinterpret_cast<const int64_t*>(base),
                                   reinterpret_cast<const float*>(base + off_scores),
                                   reinterpret_cast<const int32_t*>(base + off_counts),
                                   static_cast<int64_t>(g->slot_bytes / 8), static_cast<int64_t>(g->slot_bytes / 4),
                                   static_cast<int64_t>(g->slot_bytes / 4), order, out_items, out_scores, out_counts,
                                   s, g->world > 1 ? &sync : nullptr));
    return TAV_OK;
}

}  // extern "C"

// One sharded search: `local(mine, off_scores, off_counts, &searched)` writes this rank's packed list into its
// slot (searched = false when it wrote only zero counts and ran no search), then the list is published and merged
// in `order`.  Argument errors come from replicated arguments and return before anything is published.
template <typename Local>
static int sharded_run(const char* fn, tav_index* ix, tav_group* g, int n_queries, int k, int flags, int order,
                       Local local, int64_t* out_items, float* out_scores, int32_t* out_counts, void* stream) {
    if (!g->connected) {
        set_error("%s: tav_group_connect has not run", fn);
        return TAV_ERR_STATE;
    }
    if (n_queries > g->max_queries || k > g->max_k) {
        set_error("%s: %d queries x top-%d exceed the group's capacity (%d x %d)", fn, n_queries, k,
                  g->max_queries, g->max_k);
        return TAV_ERR_INVALID;
    }
    TAVG_CUDA(cudaSetDevice(g->device));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const bool defer = (flags & TAV_DEFER_RETRY) != 0;
    if (g->outstanding >= g->depth) {
        // the next sequence number's slot still belongs to the oldest open search
        if (defer) {
            set_error("%s: %d deferred searches outstanding (the group's depth); call tav_sharded_finish", fn,
                      g->outstanding);
            return TAV_ERR_STATE;
        }
        int redone = 0;
        const int frc = tav_sharded_finish(ix, g, stream, &redone);
        if (frc != TAV_OK) return frc;
    }
    const uint32_t seq = ++g->seq;
    const int slot = static_cast<int>(seq % static_cast<uint32_t>(g->depth));
    size_t off_scores, off_counts, bytes;
    packed_offsets(n_queries, k, &off_scores, &off_counts, &bytes);
    char* mine = g->region + g->off_slots + (static_cast<size_t>(slot) * g->world + g->rank) * g->slot_bytes;
    bool searched = false;
    const int lrc = local(mine, off_scores, off_counts, &searched);
    if (lrc == TAV_ERR_CUDA) {
        --g->seq;  // nothing was published under this number (see the failure protocol above)
        return lrc;
    }
    // any other failure: publish an empty list with status 1 so that no peer waits for this rank
    std::string error;
    if (lrc != TAV_OK) {
        error = tav_last_error();
        searched = false;
        // A failed allocation (TAV_ERR_OOM from a cudaMalloc inside the local search) leaves the runtime's last
        // error set; the publish's launch check would read it and return before the merge, which would then never
        // acknowledge this sequence number to the peers.  Such errors are not sticky: clear it.
        cudaGetLastError();
        TAVG_CUDA(cudaMemsetAsync(mine + off_counts, 0, static_cast<size_t>(n_queries) * 4, s));
    }
    int n_retry = 0;
    const int32_t* retry_totals = searched ? tav_internal_retry_totals(ix, &n_retry) : nullptr;
    const int* corpus_flag = searched ? tav_internal_split_flag(ix) : nullptr;
    // deferred (pipelined) searches: exchange on the group's stream, ordered after the local search by an event
    cudaStream_t xs = s;
    if (defer && g->world > 1) {
        TAVG_CUDA(cudaEventRecord(g->ev_local[slot], s));
        TAVG_CUDA(cudaStreamWaitEvent(g->xstream, g->ev_local[slot], 0));
        xs = g->xstream;
    } else if (g->x_pending) {  // a synchronous search after deferred ones: their exchanges come first
        TAVG_CUDA(cudaEventRecord(g->ev_merged[slot], g->xstream));
        TAVG_CUDA(cudaStreamWaitEvent(s, g->ev_merged[slot], 0));
        g->x_pending = false;
    }
    const uint32_t status = lrc != TAV_OK ? 1u : 0u;
    int rc = publish_and_merge(g, n_queries, k, seq, order, status, retry_totals, n_retry, corpus_flag, out_items,
                               out_scores, out_counts, xs);
    if (rc != TAV_OK) return rc;
    if (xs != s) g->x_pending = true;
    g->open.push_back({seq, n_queries, k, order, status, out_items, out_scores, out_counts});
    g->outstanding += 1;
    if (!defer) {
        int redone = 0;
        rc = tav_sharded_finish(ix, g, stream, &redone);
    }
    if (lrc != TAV_OK) {  // this rank's own error comes first
        set_error("%s", error.c_str());
        return lrc;
    }
    return rc;
}

extern "C" {

int tav_sharded_search(tav_index* ix, tav_group* g, const float* queries_device, int n_queries, int k,
                       float min_score, int flags, int64_t item_offset, int64_t* out_items, float* out_scores,
                       int32_t* out_counts, void* stream) {
    if (!ix || !g || n_queries < 1 || k < 1 || !queries_device || !out_items || !out_scores || !out_counts) {
        set_error("tav_sharded_search: invalid argument");
        return TAV_ERR_INVALID;
    }
    // local search straight into this rank's slot (global ordinals through item_offset)
    const int sflags = (flags & (TAV_FORCE_SCAN | TAV_FORCE_MMA | TAV_USE_ROW_MASK | TAV_USE_QUERY_MASKS |
                                 TAV_TIES_LOW_FIRST)) |
                       TAV_QUERIES_ON_DEVICE | TAV_OUTPUTS_ON_DEVICE | TAV_DEFER_RETRY;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    auto local = [&](char* mine, size_t off_scores, size_t off_counts, bool* searched) -> int {
        if (tav_size(ix) == 0) {
            TAVG_CUDA(cudaMemsetAsync(mine + off_counts, 0, static_cast<size_t>(n_queries) * 4, s));
            return TAV_OK;
        }
        *searched = true;
        return tav_search(ix, queries_device, n_queries, k, min_score, sflags, nullptr, 0, item_offset,
                          reinterpret_cast<int64_t*>(mine), reinterpret_cast<float*>(mine + off_scores),
                          reinterpret_cast<int32_t*>(mine + off_counts), stream);
    };
    // lists in rank order, each rank's block in ascending rows: order 1 is the lower row first
    return sharded_run("tav_sharded_search", ix, g, n_queries, k, flags, (flags & TAV_TIES_LOW_FIRST) ? 1 : 0, local,
                       out_items, out_scores, out_counts, stream);
}

int tav_sharded_search_subset(tav_index* ix, tav_group* g, const float* queries_device, int n_queries, int k,
                              float min_score, int flags, const int64_t* subset, int64_t subset_len,
                              const int64_t* offsets, const int64_t* positions_device, int64_t* out_items,
                              float* out_scores, int32_t* out_counts, void* stream) {
    if (!ix || !g || n_queries < 1 || k < 1 || !queries_device || !out_items || !out_scores || !out_counts ||
        subset_len < 0 || (subset_len > 0 && (!subset || !positions_device)) ||
        (offsets && (offsets[0] != 0 || offsets[n_queries] != subset_len))) {
        set_error("tav_sharded_search_subset: invalid argument");
        return TAV_ERR_INVALID;
    }
    const bool ties_low = (flags & TAV_TIES_LOW_FIRST) != 0;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    auto local = [&](char* mine, size_t off_scores, size_t off_counts, bool* searched) -> int {
        int64_t* items = reinterpret_cast<int64_t*>(mine);
        if (tav_size(ix) == 0 || subset_len == 0) {  // no share of the subset(s) on this rank
            TAVG_CUDA(cudaMemsetAsync(mine + off_counts, 0, static_cast<size_t>(n_queries) * 4, s));
            return TAV_OK;
        }
        *searched = true;
        const int pos = TAV_ITEMS_AS_POSITIONS | TAV_QUERIES_ON_DEVICE | TAV_OUTPUTS_ON_DEVICE |
                        (ties_low ? TAV_TIES_LOW_FIRST : 0);
        int rc = offsets ? tav_search_subsets(ix, queries_device, n_queries, k, min_score, pos, offsets, subset,
                                              items, reinterpret_cast<float*>(mine + off_scores),
                                              reinterpret_cast<int32_t*>(mine + off_counts), stream)
                         : tav_search(ix, queries_device, n_queries, k, min_score,
                                      pos | (flags & TAV_FORCE_SCAN) | TAV_DEFER_RETRY, subset, subset_len, 0, items,
                                      reinterpret_cast<float*>(mine + off_scores),
                                      reinterpret_cast<int32_t*>(mine + off_counts), stream);
        if (rc != TAV_OK || TAV_PEER_FILTER_MUTANT == 1) return rc;
        // positions in this rank's share -> positions in the caller's list(s), in the slot, before the publish
        TAVG_CUDA(launch_map_items(static_cast<int64_t>(n_queries) * k, positions_device, subset_len, items, s));
        return TAV_OK;
    };
    // positions are distinct across the ranks' shares: merged by position, later entry first (order 2)
    return sharded_run("tav_sharded_search_subset", ix, g, n_queries, k, flags, ties_low ? 3 : 2, local, out_items,
                       out_scores, out_counts, stream);
}

int tav_sharded_finish(tav_index* ix, tav_group* g, void* stream, int* redone_total) {
    if (!ix || !g) return TAV_ERR_INVALID;
    if (redone_total) *redone_total = 0;
    if (g->outstanding == 0) return TAV_OK;
    TAVG_CUDA(cudaSetDevice(g->device));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (g->x_pending) {  // join: the merged results of the deferred searches are complete on the caller's stream
        const int slot = static_cast<int>(g->seq % static_cast<uint32_t>(g->depth));
        TAVG_CUDA(cudaEventRecord(g->ev_merged[slot], g->xstream));
        TAVG_CUDA(cudaStreamWaitEvent(s, g->ev_merged[slot], 0));
        g->x_pending = false;
    }
    int redone = 0;
    int rc = tav_finish_search(ix, stream, &redone);  // corrects this rank's slot(s) in place
    if (rc != TAV_OK) return rc;
    // Every rank summed the same slot tails in its wait kernel: the world-wide number of queries that some
    // rank has just corrected.  One stream synchronise (tav_finish_search already did it when anything
    // was pending on this rank) makes the mapped words current; no second exchange.
    TAVG_CUDA(cudaStreamSynchronize(s));
    // which of the open searches had candidates corrected somewhere in the world (identical on every rank: all
    // ranks summed the same tails).  Read BEFORE any re-merge reuses a slot.
    std::vector<tav_group::OpenSearch> open;
    open.swap(g->open);
    g->outstanding = 0;
    std::vector<uint32_t> flagged(open.size(), 0);
    uint32_t total = 0, failed = 0;
    for (size_t i = 0; i < open.size(); ++i) {
        if (g->world > 1) failed += g->status_host[open[i].seq % static_cast<uint32_t>(g->depth)];
        // one rank: no tails were exchanged; the local redo count says "something changed", re-merge them all
        flagged[i] = g->world > 1 ? g->flagged_host[open[i].seq % static_cast<uint32_t>(g->depth)]
                                  : static_cast<uint32_t>(redone);
        total += flagged[i];
    }
    if (g->world == 1) total = static_cast<uint32_t>(redone);
    if (total > 0) {
        // Some rank corrected (in its own slot, tav_finish_search above) candidates it had already published:
        // publish and merge those searches again, oldest first.  A repair takes a fresh sequence number, whose
        // slot is that of an open search no younger than the one being repaired (the open searches are the last
        // `outstanding` <= depth consecutive ones) — i.e. one that is unflagged or already repaired; its peers'
        // acknowledgements are what the publish kernel waits for anyway.
        // The repair merges in the search's own order, but only order-0 searches can be flagged today: a flag
        // comes from the tensor-core path, which takes neither a subset nor TAV_TIES_LOW_FIRST.  A flagged subset
        // search would also need more than a re-merge: the redo writes block-local positions into the slot, and
        // nothing here maps them through the search's positions (tav_map_items) again.
        for (size_t i = 0; i < open.size(); ++i) {
            if (flagged[i] == 0) continue;
            const tav_group::OpenSearch& o = open[i];
            const uint32_t seq = ++g->seq;
            const int old_slot = static_cast<int>(o.seq % static_cast<uint32_t>(g->depth));
            const int new_slot = static_cast<int>(seq % static_cast<uint32_t>(g->depth));
            if (new_slot != old_slot && TAV_GROUP_MUTANT != 3) {
                size_t os, oc, bytes;
                packed_offsets(o.nq, o.k, &os, &oc, &bytes);
                const char* from = g->region + g->off_slots + (static_cast<size_t>(old_slot) * g->world + g->rank) * g->slot_bytes;
                char* to = g->region + g->off_slots + (static_cast<size_t>(new_slot) * g->world + g->rank) * g->slot_bytes;
                TAVG_CUDA(cudaMemcpyAsync(to, from, bytes, cudaMemcpyDeviceToDevice, s));
            }
            rc = publish_and_merge(g, o.nq, o.k, seq, o.order, o.status, nullptr, 0,
                                   nullptr, o.items, o.scores, o.counts, s);
            if (rc != TAV_OK) return rc;
        }
        TAVG_CUDA(cudaStreamSynchronize(s));
    }
    if (redone_total) *redone_total = static_cast<int>(total);
    if (failed) {
        set_error("tav_sharded_finish: a rank's local search failed (%u failures among the %zu searches finished); "
                  "their results are not valid", failed, open.size());
        return TAV_ERR_PEER;
    }
    return TAV_OK;
}

}  // extern "C"
