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
//
// Threshold searches (tav_sharded_range_*) have results whose size is known only after the local search, so they
// use a second allocation of the group, the "range inbox", with its own IPC handle and its own sequence numbers:
//   range_arrive[world] u32 | range_ack[world] u32 |
//   hdr[world][hdr_stride] int64      rank r's CSR offsets [B + 1], then a word: status | hits-included << 1
//   items[world][cap] int64 | scores[world][cap] float32
// Section r of every rank's inbox is written only by rank r, so tav_merge_range merges the world's lists in place.
// A round: the local search (it synchronises), this rank's header and (when they fit in `cap`) its hits stored into
// every peer's section r, range_arrive[me] = seq released at system scope; a one-CTA wait spins on the arrive words
// and copies the world's headers to the host, which sizes the result.  When some rank's hits did not fit, the host
// side reserves larger inboxes on every rank (tav_group_range_reserve: the totals are replicated, so every rank
// takes that branch) and every rank republishes its whole list, still held by the index.  After the merge an ack
// kernel stores range_ack[me] = seq into every peer's inbox; a publish first waits for every peer's ack of the
// previous round.  A reserve starts the sequence numbers of the new inbox from 0, as its arrive / ack words do.

#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <atomic>
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

// Where rank r's section lies in every range inbox (byte offsets; strides in elements)
struct RangeLayout {
    size_t off_ack, off_hdr, off_items, off_scores;
    int64_t hdr_stride, cap;
};

// Range publish: this rank's section of its own inbox — n_hdr16 16-byte vectors of header, n_items16 of items,
// n_scores16 of scores — into the same section of every peer's inbox, then range_arrive[me] = seq everywhere.  Waits
// first until every peer acknowledged the previous round (range_ack[w] >= seq - 1 in this rank's inbox).
__global__ void __launch_bounds__(256)
range_publish_kernel(PeerTable inbox, int me, int world, RangeLayout L, int64_t n_hdr16, int64_t n_items16,
                     int64_t n_scores16, uint32_t seq, uint32_t* ticket) {
    __shared__ int s_last;
    if (blockIdx.x == 0 && threadIdx.x < world && threadIdx.x != me)
        spin_until(reinterpret_cast<const uint32_t*>(inbox.region[me] + L.off_ack) + threadIdx.x, seq - 1);
    if (blockIdx.x == 0) {  // the other CTAs wait for CTA 0's acks through the ticket's high bit (publish_kernel)
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
    const size_t hdr = L.off_hdr + static_cast<size_t>(me) * L.hdr_stride * 8;
    const size_t items = L.off_items + static_cast<size_t>(me) * L.cap * 8;
    const size_t scores = L.off_scores + static_cast<size_t>(me) * L.cap * 4;
    const int64_t n = n_hdr16 + n_items16 + n_scores16;
    for (int w = 0; w < world; ++w) {
        if (w == me) continue;
        for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
             i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
            size_t off;
            if (i < n_hdr16) off = hdr + 16 * i;
            else if (i < n_hdr16 + n_items16) off = items + 16 * (i - n_hdr16);
            else off = scores + 16 * (i - n_hdr16 - n_items16);
            *reinterpret_cast<uint4*>(inbox.region[w] + off) = *reinterpret_cast<const uint4*>(inbox.region[me] + off);
        }
    }
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
            st_release_sys(reinterpret_cast<uint32_t*>(inbox.region[threadIdx.x]) + me, seq);  // range_arrive[me]
        }
        if (threadIdx.x == 0) *ticket = 0;
    }
}

// Range wait: every rank's round `seq` arrived in this inbox; its headers (n_words each) -> out [world][n_words]
// (mapped pinned host memory)
__global__ void __launch_bounds__(256)
range_wait_kernel(const char* inbox, int world, RangeLayout L, uint32_t seq, int n_words, int64_t* out) {
    if (threadIdx.x < world) spin_until(reinterpret_cast<const uint32_t*>(inbox) + threadIdx.x, seq);
    __syncthreads();
    const int64_t* hdr = reinterpret_cast<const int64_t*>(inbox + L.off_hdr);
    for (int i = threadIdx.x; i < world * n_words; i += blockDim.x) {
        const int r = i / n_words;
        out[i] = __ldcg(hdr + r * L.hdr_stride + (i - r * n_words));
    }
}

// Range ack: this rank no longer reads round `seq` of its inbox: range_ack[me] = seq in every peer's inbox
__global__ void range_ack_kernel(PeerTable inbox, int me, int world, size_t off_ack, uint32_t seq) {
    if (threadIdx.x < world && threadIdx.x != me) {
        __threadfence_system();
        st_release_sys(reinterpret_cast<uint32_t*>(inbox.region[threadIdx.x] + off_ack) + me, seq);
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
    // threshold searches (tav_group_range_*, tav_sharded_range_*): the range inbox
    char* rin = nullptr;              // this rank's range inbox (cudaMalloc), or none
    PeerTable rpeers{};               // range inbox of every rank, as mapped here
    RangeLayout rl{};
    size_t rin_bytes = 0;
    int rin_queries = 0;              // queries a header holds
    bool rin_connected = false;
    int64_t rin_limit = -1;           // tests: the largest inbox a reserve may allocate (-1: no cap)
    uint32_t rseq = 0;                // rounds published into the current inbox
    uint32_t* rticket = nullptr;      // device counter of the range publish kernel
    int64_t* rhdr_host = nullptr;     // pinned, mapped: the world's headers of the last round
    struct OpenRange {                // the range search between tav_sharded_range_search and its merge
        bool open = false;
        tav_index* ix = nullptr;
        int nq = 0;
        int64_t total = 0;
        bool positions_form = false;
        int64_t* positions = nullptr;  // device copy of the caller's positions (stream-ordered), until the close
        int64_t positions_len = 0;
        std::vector<int64_t> hdr;     // this rank's header: offsets [nq + 1], status | included << 1
    } rs;
};

static std::atomic<int64_t> g_range_bytes{0};  // range inbox bytes held by every group of the process

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

// the device copy of an open range search's positions, freed (the device is idle or the call synchronises)
static void range_drop_positions(tav_group* g) {
    if (g->rs.positions) cudaFree(g->rs.positions);
    g->rs.positions = nullptr;
}

// the range inbox and its peers' mappings, gone: the next threshold search needs a reserve
static void range_free(tav_group* g) {
    for (int r = 0; r < g->world; ++r) {
        if (r != g->rank && g->rpeers.region[r]) cudaIpcCloseMemHandle(g->rpeers.region[r]);
        g->rpeers.region[r] = nullptr;
    }
    if (g->rin) {
        cudaFree(g->rin);
        g_range_bytes -= static_cast<int64_t>(g->rin_bytes);
    }
    if (g->rhdr_host) cudaFreeHost(g->rhdr_host);
    g->rin = nullptr;
    g->rhdr_host = nullptr;
    g->rin_bytes = 0;
    g->rin_queries = 0;
    g->rl = RangeLayout{};
    g->rin_connected = false;
    g->rseq = 0;
    g->rs.open = false;
}

int tav_group_destroy(tav_group* g) {
    if (!g) return TAV_OK;
    cudaSetDevice(g->device);
    cudaDeviceSynchronize();
    range_free(g);
    range_drop_positions(g);
    if (g->rticket) cudaFree(g->rticket);
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

// ---- threshold searches through the range inbox ----------------------------------------------------------------

int tav_group_range_reserve(tav_group* g, int max_queries, int64_t capacity) {
    if (!g || max_queries < 0 || capacity < 0) {
        set_error("tav_group_range_reserve: invalid argument");
        return TAV_ERR_INVALID;
    }
    TAVG_CUDA(cudaSetDevice(g->device));
    const bool open = g->rs.open;  // a grow between the rounds of a search keeps it open (its state is host-side)
    range_free(g);
    if (max_queries == 0 || capacity == 0) {
        range_drop_positions(g);
        return TAV_OK;
    }
    RangeLayout L{};
    L.hdr_stride = (static_cast<int64_t>(max_queries) + 2 + 1) & ~int64_t(1);  // 16-byte rows
    L.cap = (capacity + 15) & ~int64_t(15);                                    // 16-byte item and score sections
    const size_t W = static_cast<size_t>(g->world);
    L.off_ack = a16(W * 4);
    L.off_hdr = (L.off_ack + a16(W * 4) + 255) & ~size_t(255);
    L.off_items = (L.off_hdr + W * L.hdr_stride * 8 + 255) & ~size_t(255);
    L.off_scores = (L.off_items + W * L.cap * 8 + 255) & ~size_t(255);
    const size_t bytes = L.off_scores + W * L.cap * 4;
    if (g->rin_limit >= 0 && bytes > static_cast<size_t>(g->rin_limit)) {
        range_drop_positions(g);
        set_error("tav_group_range_reserve: an inbox of %zu bytes exceeds the test cap of %lld", bytes,
                  static_cast<long long>(g->rin_limit));
        return TAV_ERR_OOM;
    }
    cudaError_t e = cudaSuccess;
    if (!g->rticket) {
        e = cudaMalloc(reinterpret_cast<void**>(&g->rticket), 64);
        if (e == cudaSuccess) e = cudaMemset(g->rticket, 0, 64);
    }
    if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void**>(&g->rin), bytes);
    if (e == cudaSuccess) {
        g->rin_bytes = bytes;
        g_range_bytes += static_cast<int64_t>(bytes);
        e = cudaMemset(g->rin, 0, L.off_hdr);  // arrive and ack words
    }
    if (e == cudaSuccess) e = cudaMallocHost(reinterpret_cast<void**>(&g->rhdr_host), W * L.hdr_stride * 8);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();  // the words are zero before a peer can map them
    if (e != cudaSuccess) {
        set_error("tav_group_range_reserve: %s (an inbox of %zu bytes)", cudaGetErrorString(e), bytes);
        range_free(g);
        range_drop_positions(g);
        return e == cudaErrorMemoryAllocation ? TAV_ERR_OOM : TAV_ERR_CUDA;
    }
    g->rl = L;
    g->rin_queries = max_queries;
    g->rpeers.region[g->rank] = g->rin;
    g->rin_connected = g->world == 1;
    g->rs.open = open;
    return TAV_OK;
}

int tav_group_range_handle(tav_group* g, void* handle_out) {
    if (!g || !handle_out || !g->rin) {
        set_error("tav_group_range_handle: no range inbox (tav_group_range_reserve)");
        return TAV_ERR_STATE;
    }
    TAVG_CUDA(cudaSetDevice(g->device));
    cudaIpcMemHandle_t h;
    TAVG_CUDA(cudaIpcGetMemHandle(&h, g->rin));
    memcpy(handle_out, &h, sizeof(h));
    return TAV_OK;
}

int tav_group_range_connect(tav_group* g, const void* handles) {
    if (!g || !handles || !g->rin) {
        set_error("tav_group_range_connect: no range inbox (tav_group_range_reserve)");
        return TAV_ERR_STATE;
    }
    TAVG_CUDA(cudaSetDevice(g->device));
    for (int r = 0; r < g->world; ++r) {
        if (r == g->rank || g->rpeers.region[r]) continue;
        cudaIpcMemHandle_t h;
        memcpy(&h, static_cast<const char*>(handles) + static_cast<size_t>(r) * sizeof(h), sizeof(h));
        void* p = nullptr;
        TAVG_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
        g->rpeers.region[r] = static_cast<char*>(p);
    }
    g->rin_connected = true;
    return TAV_OK;
}

int tav_group_range_capacity(const tav_group* g, int* max_queries, int64_t* capacity) {
    if (!g) return TAV_ERR_INVALID;
    if (max_queries) *max_queries = g->rin_connected ? g->rin_queries : 0;
    if (capacity) *capacity = g->rin_connected ? g->rl.cap : 0;
    return TAV_OK;
}

int tav_internal_range_bytes(const tav_group* g, int64_t* group_bytes, int64_t* process_bytes) {
    if (!g) return TAV_ERR_INVALID;
    if (group_bytes) *group_bytes = static_cast<int64_t>(g->rin_bytes);
    if (process_bytes) *process_bytes = g_range_bytes.load();
    return TAV_OK;
}

int tav_internal_range_cap(tav_group* g, int64_t max_bytes) {
    if (!g || max_bytes < -1) return TAV_ERR_INVALID;
    g->rin_limit = max_bytes;
    return TAV_OK;
}

}  // extern "C"

// One round of the open range search: this rank's header, and its hits when `hits` (fetched from the index into its
// own section, mapped to the caller's positions for the subset forms), published into every peer's inbox; then the
// wait for every rank's round and the world's headers on the host.  Synchronises `s`.
static int range_round(tav_group* g, bool hits, cudaStream_t s) {
    tav_group::OpenRange& o = g->rs;
    const RangeLayout& L = g->rl;
    const uint32_t seq = ++g->rseq;
    char* hdr = g->rin + L.off_hdr + static_cast<size_t>(g->rank) * L.hdr_stride * 8;
    int64_t* items = reinterpret_cast<int64_t*>(g->rin + L.off_items + static_cast<size_t>(g->rank) * L.cap * 8);
    float* scores = reinterpret_cast<float*>(g->rin + L.off_scores + static_cast<size_t>(g->rank) * L.cap * 4);
    const int n_words = o.nq + 2;
    TAVG_CUDA(cudaMemcpyAsync(hdr, o.hdr.data(), static_cast<size_t>(n_words) * 8, cudaMemcpyHostToDevice, s));
    const int64_t n = hits ? o.total : 0;
    if (n > 0) {
        if (int rc = tav_range_fetch(o.ix, 0, n, items, scores, TAV_OUTPUTS_ON_DEVICE, s)) return rc;
        if (o.positions_form) TAVG_CUDA(launch_map_items(n, o.positions, o.positions_len, items, s));
    }
    if (g->world > 1) {
        int64_t n_items16 = (n * 8 + 15) / 16, n_scores16 = (n * 4 + 15) / 16;
        if (TAV_PEER_RANGE_MUTANT == 1 && n_items16 > 0) n_items16 -= 1;
        if (TAV_PEER_RANGE_MUTANT == 2 && g->rs.hdr[o.nq + 1] & 4) n_items16 = n_scores16 = 0;
        const size_t bytes = static_cast<size_t>(n_words) * 8 + static_cast<size_t>(n) * 12;
        const int grid = static_cast<int>(std::min<size_t>(128, std::max<size_t>(1, bytes / 2048)));
        range_publish_kernel<<<grid, 256, 0, s>>>(g->rpeers, g->rank, g->world, L, (n_words * 8 + 15) / 16, n_items16,
                                                  n_scores16, seq, g->rticket);
        TAVG_CUDA(cudaGetLastError());
    }
    // (one rank publishes nothing: its wait only copies its own header out)
    range_wait_kernel<<<1, 256, 0, s>>>(g->rin, g->world, L, g->world > 1 ? seq : 0u, n_words, g->rhdr_host);
    TAVG_CUDA(cudaGetLastError());
    TAVG_CUDA(cudaStreamSynchronize(s));
    return TAV_OK;
}

// Close the open range search: this rank acknowledges its last round to every peer (nobody will wait for this rank
// at the next publish) and frees the search's positions.
static int range_close(tav_group* g, cudaStream_t s) {
    g->rs.open = false;
    if (g->rs.positions) {
        cudaError_t e = cudaFreeAsync(g->rs.positions, s);
        g->rs.positions = nullptr;
        TAVG_CUDA(e);
    }
    if (g->world == 1 || !g->rin_connected) return TAV_OK;
    range_ack_kernel<<<1, 32, 0, s>>>(g->rpeers, g->rank, g->world, g->rl.off_ack, g->rseq);
    TAVG_CUDA(cudaGetLastError());
    return TAV_OK;
}

extern "C" {

int tav_sharded_range_search(tav_index* ix, tav_group* g, const float* queries, int n_queries, float min_score,
                             int flags, const int64_t* subset, int64_t subset_len, const int64_t* offsets,
                             const int64_t* positions, int64_t item_offset, int64_t expected_hits,
                             int64_t* world_headers, void* stream) {
    const bool positions_form = (flags & TAV_ITEMS_AS_POSITIONS) != 0;
    if (!ix || !g || n_queries < 1 || !queries || !world_headers || subset_len < 0 || expected_hits < 0 ||
        (positions_form && subset_len > 0 && (!subset || !positions)) ||
        (offsets && (!positions_form || offsets[0] != 0 || offsets[n_queries] != subset_len))) {
        set_error("tav_sharded_range_search: invalid argument");
        return TAV_ERR_INVALID;
    }
    if (!g->rin_connected) {
        set_error("tav_sharded_range_search: no connected range inbox (tav_group_range_reserve / _connect)");
        return TAV_ERR_STATE;
    }
    if (n_queries > g->rin_queries) {
        set_error("tav_sharded_range_search: %d queries exceed the range inbox's %d", n_queries, g->rin_queries);
        return TAV_ERR_INVALID;
    }
    TAVG_CUDA(cudaSetDevice(g->device));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (g->rs.open)  // a search the caller left open (neither merged nor aborted) is closed first
        if (int rc = range_close(g, s)) return rc;
    tav_group::OpenRange& o = g->rs;
    o.ix = ix;
    o.nq = n_queries;
    o.positions_form = positions_form;
    o.positions_len = subset_len;
    o.hdr.assign(static_cast<size_t>(n_queries) + 2, 0);
    int lrc = TAV_OK;
    const bool local = tav_size(ix) > 0 && !(positions_form && subset_len == 0);
    if (local && positions_form) {
        // the positions on the device, for tav_map_items at each round; a failure here is published like the
        // search's own allocations
        const size_t bytes = static_cast<size_t>(subset_len) * sizeof(int64_t);
        cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&o.positions), bytes, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(o.positions, positions, bytes, cudaMemcpyHostToDevice, s);
        if (e == cudaErrorMemoryAllocation) {
            o.positions = nullptr;
            set_error("tav_sharded_range_search: %zu bytes of positions: %s", bytes, cudaGetErrorString(e));
            lrc = TAV_ERR_OOM;
        } else {
            TAVG_CUDA(e);
        }
    }
    if (local && lrc == TAV_OK) {
        const int ties = flags & TAV_TIES_LOW_FIRST;
        if (offsets)
            lrc = tav_range_search_subsets(ix, queries, n_queries, min_score, TAV_ITEMS_AS_POSITIONS | ties, offsets,
                                           subset, o.hdr.data(), stream);
        else
            lrc = tav_range_search(ix, queries, n_queries, min_score,
                                   flags & (TAV_FORCE_SCAN | TAV_FORCE_MMA | TAV_USE_ROW_MASK | TAV_USE_QUERY_MASKS |
                                            TAV_TIES_LOW_FIRST | TAV_ITEMS_AS_POSITIONS),
                                   positions_form ? subset : nullptr, positions_form ? subset_len : 0,
                                   positions_form ? 0 : item_offset, expected_hits, o.hdr.data(), stream);
    }
    if (lrc == TAV_ERR_CUDA) {  // not published (the failure protocol of the top-k exchange)
        range_drop_positions(g);
        return lrc;
    }
    std::string error;
    if (lrc != TAV_OK) {  // published as status 1 with no hits, so that no peer waits for this rank
        error = tav_last_error();
        cudaGetLastError();  // a failed allocation inside the search is not sticky (sharded_run)
        std::fill(o.hdr.begin(), o.hdr.end(), 0);
    }
    o.total = o.hdr[n_queries];
    const bool included = o.total <= g->rl.cap;
    o.hdr[n_queries + 1] = (lrc != TAV_OK ? 1 : 0) | (included ? 2 : 0);
    o.open = true;
    if (int rc = range_round(g, included, s)) return rc;
    const int n_words = n_queries + 2;
    memcpy(world_headers, g->rhdr_host, static_cast<size_t>(g->world) * n_words * 8);
    int failed = 0;
    for (int r = 0; r < g->world; ++r)
        if (TAV_PEER_RANGE_MUTANT != 3 || r == g->rank)
            failed += static_cast<int>(world_headers[r * n_words + n_queries + 1] & 1);
    if (lrc != TAV_OK || failed) {  // nobody merges this round: acknowledge it now
        if (int rc = range_close(g, s)) return rc;
        if (lrc != TAV_OK) {
            set_error("%s", error.c_str());
            return lrc;
        }
        set_error("tav_sharded_range_search: a rank's local search failed (%d of %d ranks)", failed, g->world);
        return TAV_ERR_PEER;
    }
    return TAV_OK;
}

int tav_sharded_range_republish(tav_group* g, void* stream) {
    if (!g || !g->rs.open || !g->rin_connected) {
        set_error("tav_sharded_range_republish: no open range search, or no connected range inbox");
        return TAV_ERR_STATE;
    }
    tav_group::OpenRange& o = g->rs;
    if (o.nq > g->rin_queries || o.total > g->rl.cap) {
        set_error("tav_sharded_range_republish: %d queries, %lld hits exceed the range inbox (%d, %lld)", o.nq,
                  static_cast<long long>(o.total), g->rin_queries, static_cast<long long>(g->rl.cap));
        range_close(g, static_cast<cudaStream_t>(stream));
        return TAV_ERR_INVALID;
    }
    TAVG_CUDA(cudaSetDevice(g->device));
    o.hdr[o.nq + 1] = 2 | 4;  // hits included (a failed search never gets here); 4: a republish (not read by the merge)
    return range_round(g, true, static_cast<cudaStream_t>(stream));
}

int tav_sharded_range_merge(tav_group* g, int ties_low_first, int64_t* out_offsets, int64_t* out_items,
                            float* out_scores, void* stream) {
    if (!g || !g->rs.open) {
        set_error("tav_sharded_range_merge: no open range search");
        return TAV_ERR_STATE;
    }
    TAVG_CUDA(cudaSetDevice(g->device));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const RangeLayout& L = g->rl;
    const int rc = tav_merge_range(g->device, g->world, g->rs.nq, reinterpret_cast<const int64_t*>(g->rin + L.off_hdr),
                                   L.hdr_stride, reinterpret_cast<const int64_t*>(g->rin + L.off_items), L.cap,
                                   reinterpret_cast<const float*>(g->rin + L.off_scores), L.cap, ties_low_first,
                                   out_offsets, out_items, out_scores, stream);
    std::string error = rc != TAV_OK ? tav_last_error() : "";
    const int arc = range_close(g, s);  // also after a failed merge: no peer may wait for this round
    if (rc != TAV_OK) {
        set_error("%s", error.c_str());
        return rc;
    }
    return arc;
}

int tav_sharded_range_abort(tav_group* g, void* stream) {
    if (!g) return TAV_ERR_INVALID;
    if (!g->rs.open) return TAV_OK;
    TAVG_CUDA(cudaSetDevice(g->device));
    return range_close(g, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
