// tav_internal.h — launch interfaces between the translation units of libtavec.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/tavec.h"

namespace tav {

struct MergeSync;  // tav_common.cuh

// Per-query row masks (TAV_USE_QUERY_MASKS): query q of a launch may return row r when bit r of mask row
// m = (map ? map[q] : q) is set, that row being `stride` words at bits + m * stride (whole 256-row tiles).
// `map` serves a re-pass over gathered queries: each keeps the mask it was issued with.
struct QueryMasks {
    const uint32_t* bits = nullptr;  // device, nullptr = no per-query masks
    int64_t stride = 0;              // words per mask row (a multiple of 8)
    const int32_t* map = nullptr;    // device [nq], or nullptr = identity
    const uint32_t* pop = nullptr;   // device: allowed rows per mask row (indexed like the rows), or nullptr
};
// masks of the queries [q0, ...) of a launch
inline QueryMasks qmask_from(QueryMasks m, int q0) {
    if (m.map) m.map += q0;
    else if (m.bits) {
        m.bits += static_cast<int64_t>(q0) * m.stride;
        if (m.pop) m.pop += q0;
    }
    return m;
}

// TAV_QUERY_MASK_MUTANT (tests only, never set by build.py): 1..3 compile one deliberate defect each, so that
// tests/test_gpu_query_masks.py can show its exact checks catch it: 1 the tensor-core MAIN epilogue tests the
// other query's (h ^ 1) mask, 2 the exact redo of a flagged query uses mask 0, 3 the threshold search's
// re-pass over gathered queries drops their mask map.
#ifndef TAV_QUERY_MASK_MUTANT
#define TAV_QUERY_MASK_MUTANT 0
#endif

// allowed rows (set bits below n_rows) of each of n_masks mask rows, `stride` words apart -> pop[n_masks]
cudaError_t launch_mask_popcount(const uint32_t* bits, int n_masks, int64_t n_rows, int64_t stride, uint32_t* pop,
                                 cudaStream_t s);

// ---- row-scan path (tav_scan.cu) -------------------------------------------------------
struct ScanArgs {
    const void* corpus;       // [n_corpus, dim] storage dtype, row-major dense
    int dtype;                // tav_dtype
    int64_t n_corpus;
    int dim;
    const int64_t* subset;    // device, or nullptr = all rows
    int64_t n_scan;           // rows scanned (subset_len or n_corpus)
    const float* queries;     // device float32 [nq, dim]
    int nq;                   // 1..8 queries scored per pass over the rows
    float floor_score;        // (float)min_score
    const uint64_t* bound;    // per query: admit only keys < bound (multi-pass), or nullptr
    int k;                    // hits kept per query this pass (<= kPassK)
    uint64_t* cand_keys;      // [nq, cand_stride] per-query global candidate buffers
    int cand_stride;
    uint32_t* cand_count;     // [nq], zero on entry (the select kernel re-zeroes it)
    int grid;                 // CTAs to launch (cand_stride >= grid * k)
    const uint32_t* row_mask; // optional: bit r set = corpus row r may be returned (predicate pushdown)
    int ties_low;             // 1: equal scores -> LOWER position first (reference predicate path)
    // single-launch form (launch_scan1): the last CTA merges all survivors and writes the hits
    int subset_in_params;     // the subset ordinals travel in the kernel parameters
    int fused;
    uint32_t* fused_ticket;   // device counter, zero on entry (self-resetting)
    int64_t item_offset;
    int64_t* out_items;       // [nq, k]   (device, or mapped pinned host memory)
    float* out_scores;
    int32_t* out_counts;
    uint32_t* done_flag;      // mapped pinned host word set to done_seq once the hits are written, or nullptr
    uint32_t done_seq;
    unsigned long long* trace;  // diagnostic (TAV_TRACE=1): %globaltimer stamps of the single-launch form's phases
    // collect mode (launch_scan_collect): query q's keys go to cand_keys + q * collect_stride; cand_count[q]
    // (zero on entry) counts every admitted row, also those beyond collect_stride, which are not stored
    int64_t collect_stride;
    int items_as_positions;   // single-launch form: items = the subset position (TAV_ITEMS_AS_POSITIONS)
    QueryMasks qmask;         // per-query masks of queries [0, nq) of this pass (instead of row_mask; no subset)
};
constexpr int kFusedSelectMax = 8192;   // survivors the last CTA of the single-launch form can merge
constexpr int kFusedSelOut = 1024;      // ... of which it sorts at most this many after the histogram selection
constexpr int kParamQuerySmall = 1024;  // floats of query carried in a 4 KB kernel-parameter blob
constexpr int kParamQueryBig = 3072;    // ... in the 28 KB blob (with up to kParamSubsetMax ordinals)
constexpr int kParamSubsetMax = 4096;
constexpr int kParamSubsetSmall = 1024; // ordinals in the 8 KB blob (with a query of <= kParamQuerySmall floats)
bool scan1_fits(int dim, int k, int64_t n_scan, int64_t subset_len, bool has_subset);
int scan1_grid(int device, int dim, int k, int64_t n_scan);
// q_host: float32 [dim] on the host; sub_host: int64 [n_scan] validated ordinals or nullptr
cudaError_t launch_scan1(const ScanArgs& a, const float* q_host, const int64_t* sub_host, cudaStream_t s);
int scan_max_queries(int dim, int k);            // how many queries one pass can take (smem)
int scan_grid(int device, int dtype, int dim, int nq, int k, int64_t n_scan);
cudaError_t launch_scan(const ScanArgs& a, cudaStream_t s);
int scan_collect_max_queries(int dim);          // queries one collect-mode pass can take (1/2/4/8)
int scan_collect_grid(int device, int dim, int nq, int64_t n_scan);
cudaError_t launch_scan_collect(const ScanArgs& a, cudaStream_t s);

// ---- per-query subsets (tav_search_subsets / tav_range_search_subsets, tav_scan.cu) ------
// Query q scores the entries [offsets[q], offsets[q + 1]) of one flat ordinal list.  The work is a flat space of
// (query, tile of kSubsetTile entries) items: query q's tiles are [work0[q], work0[q + 1]).  Every admitted
// entry j appends the key (score, j, or ~j with ties_low) to keys + offsets[q] through counts[q]: a query
// admits at most its own entries, so its region never overflows.
constexpr int kSubsetTile = 256;
struct SubsetArgs {
    const void* corpus;       // [n_corpus, dim] storage dtype
    int dtype;
    int64_t n_corpus;
    int dim;
    const float* queries;     // device float32 [nq, dim]
    int nq;
    const int64_t* ordinals;  // device [offsets[nq]], validated, numpy-style negatives
    const int64_t* offsets;   // device [nq + 1]
    const int64_t* work0;     // device [nq + 1]
    int64_t n_work;
    float floor_score;
    int ties_low;
    uint64_t* keys;           // [offsets[nq]]
    uint32_t* counts;         // [nq], zero on entry
};
cudaError_t launch_subset_gather(const SubsetArgs& a, cudaStream_t s);
// [nq, k] layout of sorted CSR hits: the first min(k, count) of each query, -1 / 0 padding after them
cudaError_t launch_subset_topk_layout(int nq, int k, const int64_t* csr_offsets, const int64_t* hits,
                                      const float* hit_scores, int64_t* out_items, float* out_scores,
                                      int32_t* out_counts, cudaStream_t s);

// TAV_SUBSETS_MUTANT (tests only, never set by build.py): 1..3 compile one deliberate defect each, so that
// tests/test_gpu_subsets.py can show its exact checks catch it: 1 a query's later tiles start one entry late
// when its length is not a multiple of the tile, 2 negative ordinals come back wrapped, 3 ties-low ignored.
#ifndef TAV_SUBSETS_MUTANT
#define TAV_SUBSETS_MUTANT 0
#endif

// Per-query subsets from device memory (tav_search_subsets_into / tav_range_search_subsets_into): the offsets are
// checked and the work items planned on the device.  The status word: bit 0 malformed offsets (the planner plans
// no work), bit 1 an ordinal outside [-n_corpus, n_corpus) (the gather never forms that row's address).
constexpr int kSubsetBadOffsets = 1, kSubsetBadOrdinal = 2;
struct SubsetPlanArgs {
    int nq;
    const int64_t* offsets;   // device [nq + 1], the caller's
    int64_t n_ordinals;       // offsets[nq] must equal it
    int64_t* work0;           // device [nq + 1]
    int64_t* n_work;          // device [1]: work0[nq], 0 when the offsets are refused
    int* status;
};
cudaError_t launch_subset_plan(const SubsetPlanArgs& a, cudaStream_t s);
// the gather over a device plan: a.n_work is an upper bound (ceil(n_ordinals / kSubsetTile) + nq), the items at or
// past *n_work return at once, and each ordinal is range-checked before its row is read
cudaError_t launch_subset_gather_dev(const SubsetArgs& a, const int64_t* n_work, int* status, cudaStream_t s);

// TAV_SUBSETS_DEVICE_MUTANT (tests only, never set by build.py): 1..3 compile one deliberate defect each into the
// device form, so that tests/test_gpu_subsets_device.py can show its checks catch it: 1 the planner drops the last
// tile of a query whose length is a non-zero multiple of kSubsetTile, 2 a deferred finish ignores the status word,
// 3 the plan of the sort ignores the status word (a refused search keeps its partial offsets).  No variant reads or
// writes outside a buffer.
#ifndef TAV_SUBSETS_DEVICE_MUTANT
#define TAV_SUBSETS_DEVICE_MUTANT 0
#endif

// TAV_SCALE_MUTANT (tests only, never set by build.py): 1..3 compile one deliberate defect each that only shows on
// corpora or subsets past 2^24 entries, so that tests/test_gpu_scale_exact.py can show its exact checks catch what
// the small exact tests cannot: 1 the tensor-core MAIN epilogue keeps 24 bits of the row in its keys, 2 the subset
// gather keeps 24 bits of the flat index j, 3 the segmented radix sort skips the byte of bits 24..31 of the position.
#ifndef TAV_SCALE_MUTANT
#define TAV_SCALE_MUTANT 0
#endif

// ---- segmented sort of the threshold search's keys (tav_sort.cu) -----------------------
// One segment per query: n keys (unsorted, unique) at `keys`; sorted descending and decoded into
// out_items / out_scores [out, out + n).  Segments above kSmallSortMax keys also need `tmp` (n keys of
// scratch) and their radix tiles [tile0, tile0 + ceil(n / kRadixTile)).
struct SortSeg {
    uint64_t* keys;
    uint64_t* tmp;
    int64_t out;
    int64_t n;
    int64_t tile0;
};
constexpr int kSmallSortMax = 4096;  // keys one CTA sorts in shared memory
constexpr int kRadixTile = 8192;     // keys per CTA in a radix pass
struct SortArgs {
    const SortSeg* segs;      // device [n_segs]: every query
    int n_segs;
    const int* large;         // device [n_large]: indexes of the segments above kSmallSortMax
    int n_large;
    const int* tile_seg;      // device [n_tiles]: large segment (index into `large`) of every radix tile
    int64_t n_tiles;
    uint64_t* minmax;         // device [2 * n_large] scratch
    uint32_t* hist;           // device [n_tiles * 256] scratch
    uint32_t* offs;           // device [n_tiles * 256] scratch
    const int64_t* subset;    // item = subset[pos] (or pos) + item_offset
    int64_t item_offset;
    int ties_low;
    int64_t* out_items;
    float* out_scores;
};
// returns the number of kernels launched in *launches
cudaError_t launch_segmented_sort(const SortArgs& a, cudaStream_t s, int* launches);

// The device plan of a threshold search into caller buffers (tav_range_search_into): the collect counters ->
// the CSR offsets, the overflow flags and everything the segmented sort needs, with no host round trip.
struct RangePlanArgs {
    int nq;
    const uint32_t* count;   // [nq] rows admitted (exact, also past a full region)
    const uint32_t* fill;    // [nq] compared with cap: > cap = the query's region or fullest segment overflowed
    uint32_t cap;
    int64_t key_stride;      // > 0: query q's keys at keys + q * key_stride (row scan); 0: packed in query order
                             // with the overflowed queries left out (tensor cores, gathered to dst_off)
    uint64_t* keys;
    uint64_t* tmp;           // radix scratch, laid out like keys
    int64_t* out_offsets;    // [nq + 1] the CSR offsets of the result, or nullptr (a re-pass: out_base)
    const int64_t* out_base; // [nq] a re-pass: where each query's hits go (its offset in the search it redoes)
    const int* abandon[2];   // words (or nullptr): either set -> nothing is sorted or gathered
    int64_t* dst_off;        // [nq] packed only: key offset of the query, -1 when not gathered; else nullptr
    int32_t* flags;          // [nq] or nullptr: 0, or the fill of an overflowed query
    int32_t* n_flagged;      // or nullptr: the number of flagged queries (device) ...
    int32_t* n_flagged_host; // ... and its mapped pinned twin, or nullptr
    SortSeg* segs;           // [nq]
    int* large;              // [nq] at most
    int* tile_seg;           // [upper bound of the radix tiles]
    uint64_t* minmax;        // [2 * nq] at most (initialised here for the large segments)
    int* sizes;              // [2] large segments, radix tiles
};
cudaError_t launch_range_plan(const RangePlanArgs& a, cudaStream_t s);
// the same plan over per-query subsets: query q's keys (and radix scratch) at keys + key_off[q] (tmp + key_off[q]),
// key_stride unused; when an abandon word is set every query counts 0 hits (all offsets 0)
cudaError_t launch_range_plan_subsets(const RangePlanArgs& a, const int64_t* key_off, cudaStream_t s);
// launch_segmented_sort over a device plan: a.n_large / a.n_tiles are upper bounds (the plan's sizes give the
// counts), and hits at CSR positions >= cap are not written
cudaError_t launch_segmented_sort_dev(const SortArgs& a, const int* sizes, int64_t cap, cudaStream_t s, int* launches);

// ---- grouped lookups (tav_leaders.cu) ----------------------------------------------------
// Leader reduction of one query's unsorted keys (n of them at `keys`): its open-addressing table is the slot_mask + 1
// (a power of two >= 2n, or 0 slots when n == 0) slots from slot0 of the shared table, and its tiles of the flat key
// (slot) space start at key_tile0 (slot_tile0).  The segments are in ascending tile order.
constexpr int kLeaderTileKeys = 4096;
struct LeaderSeg {
    uint64_t* keys;
    int64_t n;
    int64_t slot0;
    uint32_t slot_mask;
    int64_t key_tile0;
    int64_t slot_tile0;
};
// every segment's keys -> the keys of its groups' leaders (groups[position of the key]), compacted in place, in no
// order; counts[q] (zero on entry) = its leaders.  tgroup (-1) and tkey (0) are the table, initialised by the caller.
cudaError_t launch_leaders(const LeaderSeg* segs, int nq, int64_t key_tiles, int64_t slot_tiles, const int32_t* groups,
                           int ties_low, int32_t* tgroup, uint64_t* tkey, uint32_t* counts, cudaStream_t s);
// the group map's check: stat[0] (zero on entry) |= 1 when some value is negative, stat[1] (zero on entry) += the
// runs of equal consecutive values
cudaError_t launch_group_check(const int32_t* groups, int64_t n, uint64_t* stat, cudaStream_t s);
// [nq, k] top-k rows / scores / counts -> the library's keys of each query's hits at keys + q * k
cudaError_t launch_topk_keys(int nq, int k, const int64_t* rows, const float* scores, const int32_t* counts,
                             int ties_low, uint64_t* keys, cudaStream_t s);
// out_groups[i] = groups[rows[i]] for rows[i] >= 0, else -1
cudaError_t launch_group_decode(int64_t n, const int64_t* rows, const int32_t* groups, int64_t* out_groups,
                                cudaStream_t s);

struct SelectArgs {
    const uint64_t* cand_keys;   // [nq, cand_stride]
    int cand_stride;
    const uint32_t* cand_count;  // [nq]
    uint32_t* cand_count_reset;  // same array: zeroed by the kernel once consumed
    int nq;
    int k;                       // hits this pass
    int out_stride;              // row stride of out_items/out_scores (the caller's total k)
    int out_offset;              // column where this pass starts
    const int64_t* subset;       // device copy of the caller's ordinals, or nullptr
    int64_t item_offset;
    int64_t* out_items;          // already offset to the first query of this chunk
    float* out_scores;
    int32_t* out_counts;
    uint64_t* bound_out;         // [nq] next-pass bound (last key, 0 if exhausted), or nullptr
    int accumulate;              // counts += n instead of counts = n
    int ties_low;                // keys carry ~position (see ScanArgs)
};
cudaError_t launch_select(const SelectArgs& a, cudaStream_t s);

// in place: hits sorted by score -> first hit of every group (row_to_group[item - item_offset]), the
// reference's chunk -> message fold (storage/memory/messageindex.py:185-207)
cudaError_t launch_fold_groups(int n_queries, int k, const int32_t* row_to_group, int64_t n_rows,
                               int64_t item_offset, int64_t* items, float* scores, int32_t* counts,
                               cudaStream_t s);

cudaError_t launch_merge(int n_lists, int n_queries, int k, const int64_t* items,
                         const float* scores, const int32_t* counts, int64_t items_stride,
                         int64_t scores_stride, int64_t counts_stride, int64_t* out_items,
                         float* out_scores, int32_t* out_counts, cudaStream_t s);
// the same merge with tav_merge_topk_ordered's `order` (0..3) among equal scores; with `sync` the fused wait /
// merge / acknowledge of the peer exchange (tav_group.cu)
cudaError_t launch_merge_ordered(int n_lists, int n_queries, int k, const int64_t* items, const float* scores,
                                 const int32_t* counts, int64_t items_stride, int64_t scores_stride,
                                 int64_t counts_stride, int order, int64_t* out_items, float* out_scores,
                                 int32_t* out_counts, cudaStream_t s, const MergeSync* sync = nullptr);
// in place: items[i] = table[items[i]] where 0 <= items[i] < table_len
cudaError_t launch_map_items(int64_t n, const int64_t* table, int64_t table_len, int64_t* items, cudaStream_t s);

// TAV_SHARDED_FILTER_MUTANT (tests only, never set by build.py): 1..3 compile one deliberate defect each, so
// that tests/test_gpu_sharded_filter.py can show its exact checks catch it: 1 the merge's order argument
// ignored, 2 the position key of orders 2 / 3 replaced by the list / slot key, 3 subset[pos] decoded despite
// TAV_ITEMS_AS_POSITIONS.
#ifndef TAV_SHARDED_FILTER_MUTANT
#define TAV_SHARDED_FILTER_MUTANT 0
#endif

// TAV_GROUP_MUTANT (tests only, never set by build.py): 1..3 compile one deliberate defect each into the peer
// exchange (tav_group.cu), so that tests/test_gpu_peer_exchange.py can show its exact checks catch it: 1 the
// published tail is always 0 (no search is ever repaired), 2 one 16-byte vector fewer of each list is stored
// into the peers (its last counts reach them stale), 3 a repair publishes from its new slot without copying the
// list there.  Every wait of the protocol stays satisfiable: the results are wrong, nothing spins out.
#ifndef TAV_GROUP_MUTANT
#define TAV_GROUP_MUTANT 0
#endif

// TAV_PEER_FILTER_MUTANT (tests only, never set by build.py): 1..2 compile one deliberate defect each into the
// filtered and subset searches of the peer exchange, so that tests/test_gpu_peer_filtered.py can show its checks
// catch it: 1 a subset search publishes its share's positions without mapping them to the caller's list
// (tav_map_items), 2 the merge ignores the slot tails' status words (a peer's failure is not reported).  Every wait
// of the protocol stays satisfiable.
#ifndef TAV_PEER_FILTER_MUTANT
#define TAV_PEER_FILTER_MUTANT 0
#endif

// TAV_PEER_RANGE_MUTANT (tests only, never set by build.py): 1..3 compile one deliberate defect each into the
// threshold search of the peer exchange (tav_sharded_range_*), so that tests/test_gpu_peer_range.py can show its
// checks catch it: 1 a publish stores one 16-byte vector fewer of the items into the peers, 2 a republish after a grow
// stores the header (and raises the flag) but no hits, 3 a rank adds up only its own status word (a peer's failure is
// not reported).  Every wait of the protocol stays satisfiable and nothing is read outside an allocation.
#ifndef TAV_PEER_RANGE_MUTANT
#define TAV_PEER_RANGE_MUTANT 0
#endif

// ---- compaction after a removal (tav_compact.cu) -----------------------------------------
// keys: device [m], keys[i] = rem[i] - i over the sorted distinct removed ordinals.  Destinations
// [d_begin, d_end) of the compacted rows: dst row (d - d_base) = src row (d + #{keys <= d}).  src and dst
// must not overlap.
cudaError_t launch_compact_gather(const void* src, void* dst, const int64_t* keys, int64_t m, int64_t d_begin,
                                  int64_t d_end, int64_t d_base, size_t row_bytes, cudaStream_t s);
// n_rows whole rows src -> dst (no overlap), on `device`
cudaError_t launch_compact_copy(int device, const void* src, void* dst, int64_t n_rows, size_t row_bytes,
                                cudaStream_t s);

// rows [n, dim] of src dtype -> dst dtype (RNE), optionally L2-normalised per row (fp32 math)
cudaError_t launch_convert(const void* src, int src_dtype, void* dst, int dst_dtype, int64_t n,
                           int dim, int normalize, cudaStream_t s);

// ---- tensor-core path (tav_mma.cu) -----------------------------------------------------
struct MmaPlan;  // opaque: tensor maps + workspace for one (index, batch shape)
bool mma_supported(int dtype, int dim);   // bf16 / fp16 storage
bool mma_split_supported(int dim);        // float32 storage carried as two fp16 planes
// float32 rows -> fp16 planes hi, lo with x ~= hi + lo / 2048; *overflow |= 1 if some |x| > fp16 range
cudaError_t launch_split_rows(const float* src, void* hi, void* lo, int64_t n, int dim, int* overflow,
                              cudaStream_t s);
// returns cudaSuccess and fills outputs exactly like scan+select; see tav_mma.cu
struct MmaArgs {
    int device;
    const void* corpus;    // storage rows; for split float32 data: the hi plane (fp16)
    const void* corpus_lo; // split only: the lo plane (fp16)
    int split;             // 1: float32 index searched through its two fp16 planes
    int* split_overflow;   // split only: device flag set when a value left the fp16 range
    int dtype;             // storage dtype of the index (TAV_F32 when split)
    int64_t n_corpus;
    int dim;
    const float* queries;  // device float32 [nq, dim]
    int nq;
    float floor_score;
    int k;
    int64_t item_offset;
    int64_t* out_items;    // device [nq, k]
    float* out_scores;
    int32_t* out_counts;
    int32_t* retry_flags;  // device [nq]: set to 1 for queries the caller must redo with the row scan
    int32_t* retry_total;  // device [1]: incremented once per flagged query (never reset by the kernels)
    int32_t* retry_total_host;  // the same counter in mapped pinned memory (read by the host without a copy), or nullptr
    int* split_overflow_host;   // split only: mapped pinned twin of split_overflow, or nullptr
    const uint32_t* row_mask;  // optional device bitmask over corpus rows (bit set = row may be returned)
    cudaEvent_t (*ev)[2];  // optional event pairs, one recorded around every kernel launched
    int* ev_kind;          //   kind per pair: 0 = dominant (MAIN) kernel, 1 = sample pass, 2 = auxiliary
    int ev_max;
    int* ev_used;
    int ev_main_only;      // 1: record events only around the dominant (MAIN) kernel
    QueryMasks qmask;      // optional per-query masks of queries [0, nq) (instead of row_mask)
};
constexpr int kMmaMaxQueries = 32768;  // queries per launch_mma_search call (256 chunks of 128; callers slab)
size_t mma_workspace_bytes(const MmaArgs& a);
cudaError_t launch_mma_search(const MmaArgs& a, void* workspace, size_t workspace_bytes,
                              cudaStream_t s, int* launches);
// Threshold search on the tensor cores (tav_range_search): the MAIN kernel without a sample pass, admission
// threshold = the exact dot floor of min_score, so every row whose score passes lands in one of the query's
// n_seg private segments of cap_seg keys (counts keep counting past cap_seg).  Needs a.retry_flags [nq]
// (scratch) and, split, a.split_overflow [2]; a.k is unused.
struct MmaCollect {
    int per_chunk = 0;    // units per query chunk (fixes which rows feed which segment)
    int n_seg = 0;        // segments per query
    uint32_t cap_seg = 0; // keys a segment holds
    size_t ws_bytes = 0;  // workspace of this plan
};
// per_chunk 0: the plan's own; cap_seg is clamped to what a segment can see
MmaCollect mma_collect_plan(const MmaArgs& a, int per_chunk, int64_t cap_seg);
// query prep + MAIN + a count kernel: totals[q] = rows admitted, maxseg[q] = fullest segment (> cap_seg:
// overflowed, its keys incomplete).  With a.ev / a.ev_used: one event pair (kind 0) around MAIN.
cudaError_t launch_mma_collect(const MmaArgs& a, const MmaCollect& c, void* workspace, uint32_t* totals,
                               uint32_t* maxseg, cudaStream_t s, int* launches);
// the keys of every query with dst_off[q] >= 0 (device [nq]), as library keys, to dst + dst_off[q]
cudaError_t launch_mma_gather(const MmaArgs& a, const MmaCollect& c, void* workspace, const int64_t* dst_off,
                              uint64_t* dst, int ties_low, cudaStream_t s);
// verification aid: every raw dot product of the tensor-core path, out[nq, n_corpus] on the device
cudaError_t launch_mma_dump(const MmaArgs& a, void* workspace, size_t workspace_bytes, float* out,
                            cudaStream_t s);

void set_error(const char* fmt, ...);

}  // namespace tav

// library-internal (not in include/tavec.h): device address of the "queries flagged for the exact redo"
// counters of the index's most recent search — `*count` int32 words, 2 words apart — or nullptr when that
// search ran on the row-scan path (nothing to flag).  The sharded search ships their sum with the
// published candidate list so that every rank learns, without a second exchange, whether some rank will
// correct its candidates at finish.
extern "C" const int32_t* tav_internal_retry_totals(tav_index* ix, int* count);
// library-internal: device address of the index's "a corpus value left the fp16 range" flag when its most recent
// search ran the split form (float32 rows as two fp16 planes), else nullptr.  While the flag is set, finish redoes
// every query of such a search, so the sharded search counts all of them in the published tail.
extern "C" const int* tav_internal_split_flag(tav_index* ix);

// library-internal: how tav_remove_rows compacts on this index.  `mode` 0 the default (in place), 1 out of
// place (TAV_ERR_OOM when its allocation fails), 2 in place; `scratch_bytes` bounds the in-place window buffer (0: the
// default).  tav_internal_compact_stats reports the last removal: path 0 nothing moved, 1 out of place,
// 2 in place, and the number of windows.  Tests use them to reach both paths on small indexes.
extern "C" int tav_internal_compact_policy(tav_index* ix, int mode, int64_t scratch_bytes);
extern "C" int tav_internal_compact_stats(tav_index* ix, int* path, int64_t* windows);
// library-internal: the largest allocation tav_rows_stage may make on this index, in bytes (-1: no cap).  A
// stage above it gives TAV_ERR_OOM as a failed cudaMalloc would; tests use it to reach that path.
extern "C" int tav_internal_stage_cap(tav_index* ix, int64_t max_bytes);
// Tests only: tav_set_query_masks fails with TAV_ERR_OOM, as a failed allocation does, for masks of more than
// max_bytes bytes (-1: no cap), so that one rank's mask upload can fail without a device fault.
extern "C" int tav_internal_qmask_cap(tav_index* ix, int64_t max_bytes);
// Tests only: while `on`, every tensor-core search of the index asks cudaMalloc for 2^60 bytes for its bookkeeping
// (a real allocation failure: cudaErrorMemoryAllocation, not sticky) and returns TAV_ERR_OOM, as a search does when
// its buffers do not fit.
extern "C" int tav_internal_search_alloc_fail(tav_index* ix, int on);
// library-internal: bytes of this index's library-owned row allocation and staged block, and bytes held in such row
// blocks by every index of the process.  Tests use it to see that a rebalance frees the block it replaced.
extern "C" int tav_internal_row_bytes(tav_index* ix, int64_t* index_bytes, int64_t* process_bytes);
// library-internal: bytes of this group's range inbox, and bytes held in range inboxes by every group of the process.
// Tests use it to see what a group keeps between threshold searches.
extern "C" int tav_internal_range_bytes(const tav_group* g, int64_t* group_bytes, int64_t* process_bytes);
// Tests only: tav_group_range_reserve fails with TAV_ERR_OOM, as a failed allocation does, for an inbox of more than
// max_bytes bytes (-1: no cap), so that one rank's grow can fail without a device fault.
extern "C" int tav_internal_range_cap(tav_group* g, int64_t max_bytes);

// TAV_REBALANCE_MUTANT (tests only, never set by build.py): 1..3 compile one deliberate defect each into the
// rebalance (tav_rows_stage / tav_rows_commit), so that tests/test_gpu_rebalance.py can show its exact checks catch
// it: 1 the first two pieces of a stage are laid out in swapped order, 2 the fp16 planes of a float32 index are kept
// at commit, 3 the row mask is kept at commit, 4 the old rows are not freed at commit.  No variant reads or writes
// outside an allocation.
#ifndef TAV_REBALANCE_MUTANT
#define TAV_REBALANCE_MUTANT 0
#endif

namespace tav {

}  // namespace tav
