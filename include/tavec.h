/*
 * tavec.h — C ABI of libtavec.so, the H100 (sm_90a) engine behind typeagent's
 * VectorBase top-k lookup.
 *
 * This is the drop-in boundary for ONE path of microsoft/typeagent-py:
 *
 *   src/typeagent/aitools/vectorbase.py:163-201  VectorBase.fuzzy_lookup_embedding
 *   src/typeagent/aitools/vectorbase.py:203-230  VectorBase.fuzzy_lookup_embedding_in_subset
 *   src/typeagent/aitools/vectorbase.py:115-148  add_embedding / add_embeddings  (append)
 *   src/typeagent/aitools/vectorbase.py:253-287  clear / serialize / deserialize (bulk load)
 *   src/typeagent/aitools/vectorbase.py:44-47    cosine_to_score
 *
 * The reference has no FFI of its own (it is pure Python + numpy); these entry points
 * are what a ctypes binding for that path binds (see INTEGRATION.md).  Plain pointers
 * and sizes only; no torch / numpy types.  Every function returns 0 on success or a
 * negative tav_status; tav_last_error() returns a thread-local message for the last
 * failure.  There is no CPU fallback anywhere behind this ABI: without a CUDA device
 * every compute entry point fails with TAV_ERR_CUDA.
 *
 * Threading: calls on one index are serialised by a mutex inside the library (ctypes releases
 * the GIL); different indexes are independent.  Work is enqueued on the
 * caller's stream (`stream`, a cudaStream_t passed as void*; NULL = the CUDA legacy default
 * stream, as everywhere in the CUDA runtime).  Entry points that take host output pointers
 * synchronise that stream before returning; with TAV_OUTPUTS_ON_DEVICE they return as soon
 * as the work is enqueued, ordered after earlier work on the same stream.
 */
#ifndef TAVEC_H
#define TAVEC_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TAV_ABI_VERSION 2

typedef struct tav_index tav_index; /* opaque: device corpus + search workspace */

/* storage / source element types */
enum tav_dtype { TAV_F32 = 0, TAV_BF16 = 1, TAV_F16 = 2 };

enum tav_status {
    TAV_OK = 0,
    TAV_ERR_INVALID = -1, /* bad argument (the Python side maps this to ValueError) */
    TAV_ERR_CUDA = -2,    /* CUDA runtime / driver failure, or no device  (RuntimeError) */
    TAV_ERR_OOM = -3,     /* device or pinned-host allocation failed      (MemoryError) */
    TAV_ERR_RANGE = -4,   /* ordinal out of range                         (IndexError) */
    TAV_ERR_STATE = -5    /* operation not valid in this state (e.g. append to adopted memory) */
};

/* tav_create flags */
enum tav_index_flags {
    /* L2-normalise every appended row (fused into the convert-on-append kernel) and every
     * query (fused into query staging): cosine similarity for un-normalised inputs.  The
     * default (0) is the reference's behaviour: a plain dot product that relies on the
     * caller's unit-norm embeddings (vectorbase.py:176, model_adapters.py:176-184).
     * A row (or query) is first scaled by the power of two of its largest magnitude, which is
     * exact, so rows of any finite scale normalise to within a few float32 ulps of v / ||v||
     * (then one rounding to the storage type).  Edge cases:
     *   - a zero row stays zero and is returned with score 0.5 (dot 0);
     *   - a row with a NaN or +-inf element has NaN dots and is never returned;
     *   - a zero query stays zero and returns every row without NaN or inf at score 0.5. */
    TAV_NORMALIZE = 1
};

/* tav_search flags */
enum tav_search_flags {
    TAV_QUERIES_ON_DEVICE = 1, /* `queries` is a device pointer (float32 [n_queries, dim]) */
    TAV_OUTPUTS_ON_DEVICE = 2, /* out_* are device pointers; no synchronisation */
    TAV_FORCE_SCAN = 4,        /* use the CUDA-core row-scan kernels whatever the shape */
    TAV_FORCE_MMA = 8,         /* use the wgmma tensor-core kernel (needs dim % 8 == 0, no subset) */
    /* Fully asynchronous tensor-core search (needs both ..._ON_DEVICE flags): the check whether
     * some query must be redone by the exact row scan — a host synchronisation — is left to
     * tav_finish_search.  Until then the outputs of such (rare) queries are not final. */
    TAV_DEFER_RETRY = 16,
    /* Predicate / post-filter pushdown (vectorbase.py:191-201, storage/sqlite/messageindex.py:
     * 296-326): only rows whose bit is set in the mask given to tav_set_row_mask may be returned. */
    TAV_USE_ROW_MASK = 32,
    /* Among exactly equal scores return the LOWER row first (the reference's stable sort on its
     * predicate path, vectorbase.py:200); default is higher row first (its argsort path, :184-187).
     * Row-scan kernels only. */
    TAV_TIES_LOW_FIRST = 64,
    /* Do not use the single-launch form of the row scan (one host query, host outputs: the query
     * rides in the kernel parameters and the last CTA merges); tests use it to reach the two-kernel
     * form with one query. */
    TAV_NO_FUSED_SCAN = 128
};

int tav_abi_version(void);
const char* tav_last_error(void);
int tav_device_count(int* out_count);

/* Lifecycle.  `dim` may be 0: adopted from the first append (vectorbase.py:119-121).
 * `reserve_rows` pre-sizes the device buffer (growth is by capacity doubling). */
int tav_create(int device, int dim, int store_dtype, int index_flags, int64_t reserve_rows,
               tav_index** out);
int tav_destroy(tav_index* ix);
int tav_clear(tav_index* ix); /* size -> 0; dim and capacity kept (vectorbase.py:253-256) */
int tav_reserve(tav_index* ix, int64_t rows);

/* Append `n` rows of `dim` elements of `src_dtype` from host (src_on_device = 0) or device
 * memory; converted to the storage dtype with round-to-nearest-even on the GPU. */
int tav_append(tav_index* ix, const void* rows, int64_t n, int dim, int src_dtype,
               int src_on_device, void* stream);

/* Zero-copy: use caller-owned device memory (`n` rows of storage dtype, row-major, dense,
 * 16-byte aligned) as the corpus.  The caller keeps it alive; append is then invalid. */
int tav_adopt_device(tav_index* ix, void* device_rows, int64_t n, int dim);

int64_t tav_size(const tav_index* ix);
int tav_dim(const tav_index* ix);
int tav_store_dtype(const tav_index* ix);
int tav_device(const tav_index* ix);

/* Read rows [first, first+n) back as float32 into host memory (storage -> f32 is exact). */
int tav_read_rows(tav_index* ix, int64_t first, int64_t n, float* out_host, void* stream);

/*
 * The hot path.  For each of `n_queries` query vectors (float32 [n_queries, dim]):
 *   x      = dot(row, query)                       float32 accumulate
 *   score  = clip((x + 1) / 2, 0, 1)               float32, as vectorbase.py:44-47
 *   keep rows with score >= min_score              float32 compare, as :179
 *   return the `k` best, descending by score (equal scores: higher row first)
 * Rows are the whole corpus, or — if `subset` != NULL — the `subset_len` host int64
 * ordinals in `subset` (negative ordinals count from the end like numpy; duplicates are
 * scored and returned once per occurrence; vectorbase.py:217-218).
 *
 *   out_items  [n_queries, k] int64   row ordinal + item_offset (or the subset ordinal)
 *   out_scores [n_queries, k] float32
 *   out_counts [n_queries]    int32   number of valid entries per query (<= k)
 *
 * k must be >= 1 (the caller turns the reference's "max_hits == 0 means everything",
 * quirk Q2, into k = number of rows).  Any k is accepted.  Routing of large k: with host
 * outputs, k >= rows searched and more than 4 * TAV_PASS_K (8192) rows, the search is
 * served by the threshold engine of tav_range_search (one read of the rows) and its
 * result laid out as above; otherwise, above TAV_PASS_K rows per query, the search runs
 * in ceil(k / TAV_PASS_K) passes over the rows.  Both give the same result.
 */
int tav_search(tav_index* ix, const float* queries, int n_queries, int k, float min_score,
               int flags, const int64_t* subset, int64_t subset_len, int64_t item_offset,
               int64_t* out_items, float* out_scores, int32_t* out_counts, void* stream);

/* Threshold (range) search.  Every row whose score >= min_score, per query, in the library's
 * order: score descending, then row descending (row ascending with TAV_TIES_LOW_FIRST).
 * Writes CSR offsets out_offsets[n_queries + 1] (host, or device with TAV_OUTPUTS_ON_DEVICE):
 * query q's hits are [out_offsets[q], out_offsets[q + 1]).  The hits stay in library-owned
 * device memory until the next search on the index; tav_range_fetch copies them out.
 * expected_hits is a capacity hint for the whole batch (0 = library default; the previous
 * search's total is a good one); it never changes the result, only whether queries with more
 * hits than their share get one more pass.  Flags: QUERIES_ON_DEVICE, OUTPUTS_ON_DEVICE,
 * FORCE_SCAN, FORCE_MMA, USE_ROW_MASK, TIES_LOW_FIRST.  Path choice as in tav_search: batches
 * (>= 16 queries, >= 4096 rows, no subset, dim % 8 == 0) or FORCE_MMA on the tensor cores, the row
 * scan otherwise; a float32 value beyond the fp16 range sends the search to the row scan.  Subset
 * and row mask as in tav_search.  NaN min_score, an empty corpus or an empty subset give all-zero
 * offsets; NaN rows are never returned.  Synchronises once: it must learn the total before it can
 * size the result (a tensor-core re-pass adds a second check of its counts).  TAV_ERR_OOM when
 * the hits do not fit in device memory (the index stays usable). */
int tav_range_search(tav_index* ix, const float* queries, int n_queries, float min_score, int flags,
                     const int64_t* subset, int64_t subset_len, int64_t item_offset,
                     int64_t expected_hits, int64_t* out_offsets, void* stream);
/* Copy hits [first, first + n) of the last range search (items = row + item_offset, or the
 * subset ordinal + item_offset; scores float32) to host or device (TAV_OUTPUTS_ON_DEVICE) memory. */
int tav_range_fetch(tav_index* ix, int64_t first, int64_t n, int64_t* out_items, float* out_scores,
                    int flags, void* stream);

/* Completes EVERY outstanding TAV_DEFER_RETRY search of the index: synchronises `stream`, redoes
 * each search's flagged queries exactly into that search's own outputs and reports how many
 * (*redone).  The caller keeps the query and output buffers of deferred searches alive until
 * then.  Up to 64 searches may be outstanding (a 65th finishes the earlier ones first, and the
 * queries redone then are not counted in *redone).  On a TAV_NORMALIZE index each outstanding
 * search keeps its normalised queries in device memory of its own (grown as needed, never by
 * finishing searches early) until this call.  No-op when nothing is pending. */
int tav_finish_search(tav_index* ix, void* stream, int* redone);

/* Row mask for TAV_USE_ROW_MASK: `n_rows` bits (bit r of word r/32 = row r allowed), host or
 * device memory; n_rows must equal tav_size().  Kept on the device until the rows change
 * (tav_clear / tav_adopt_device drop it; appends invalidate it) or n_rows == 0 clears it. */
int tav_set_row_mask(tav_index* ix, const uint32_t* bits, int64_t n_rows, int on_device, void* stream);

/*
 * Merge step of the row-sharded search (SURVEY.md §8e): `n_lists` per-shard results of
 * tav_search (device memory, as an all-gather of each rank's outputs produces) -> the
 * global top-k per query, same order rule.  List g's arrays start at
 *   items + g * items_stride   ([n_queries, k] int64;  stride in int64 elements)
 *   scores + g * scores_stride ([n_queries, k] float32; stride in float elements)
 *   counts + g * counts_stride ([n_queries] int32;      stride in int32 elements)
 * (a stride of 0 means dense: n_queries*k, n_queries*k, n_queries), which lets one packed
 * all-gather buffer per rank be merged in place.  Lists must be in ascending shard (row)
 * order.  All pointers are device pointers on `device`; outputs are [n_queries, k] /
 * [n_queries].
 */
int tav_merge_topk(int device, int n_lists, int n_queries, int k, const int64_t* items,
                   const float* scores, const int32_t* counts, int64_t items_stride,
                   int64_t scores_stride, int64_t counts_stride, int64_t* out_items,
                   float* out_scores, int32_t* out_counts, void* stream);

/*
 * Row-sharded search across the GPUs of one box, one process per GPU (SURVEY.md §8e).  A group is
 * this rank's end of the candidate exchange: an "exchange region" in its HBM which the peers map
 * through a CUDA IPC handle.  Create it on every rank with the same arguments, exchange the handles
 * (tav_group_handle_bytes() bytes each, rank order) by any host-side means, connect, then search:
 *
 *   tav_sharded_search = tav_search on this rank's rows (ordinals shifted by item_offset)
 *                        -> PUBLISH kernel: this rank's [B, k] list stored into every peer's region
 *                           over NVLink, sequence flag released at system scope
 *                        -> MERGE: waits for all ranks' flags, merges the world's lists (same total
 *                           order as one GPU: bit-identical results), acknowledges to the peers.
 *
 * No NCCL call and no host synchronisation on this path.  SPMD: every rank calls it with the same
 * n_queries and k, in the same order.  queries / outputs are device pointers; the merged result is
 * replicated on every rank.  With TAV_DEFER_RETRY in `flags` up to `depth` searches may be
 * outstanding before tav_sharded_finish, which also agrees, across ranks, which of them had a query
 * redone exactly by some rank, and repeats the exchange for exactly those (their output buffers must
 * stay valid until then).
 */
typedef struct tav_group tav_group;
int tav_group_handle_bytes(void);
int tav_group_create(int device, int rank, int world, int max_queries, int max_k, int depth, tav_group** out);
int tav_group_local_handle(tav_group* g, void* handle_out);
int tav_group_connect(tav_group* g, const void* handles /* world x tav_group_handle_bytes() */);
int tav_group_capacity(const tav_group* g, int* max_queries, int* max_k, int* depth);
int tav_group_destroy(tav_group* g);
int tav_sharded_search(tav_index* ix, tav_group* g, const float* queries_device, int n_queries, int k,
                       float min_score, int flags, int64_t item_offset, int64_t* out_items, float* out_scores,
                       int32_t* out_counts, void* stream);
int tav_sharded_finish(tav_index* ix, tav_group* g, void* stream, int* redone_total);

/*
 * Chunk -> message fold of hit lists, on the device, in place (storage/memory/messageindex.py:
 * 185-207 `to_scored_message_ordinals`; the reference folds AFTER the top-k over chunks): walking
 * each query's hits in score order, the first hit of a group keeps its score, later hits of the
 * same group are dropped; items become group ordinals `row_to_group[item - item_offset]` (device
 * int32 [n_rows]); counts are updated, tails padded with -1 / 0.  k <= 8192.
 */
int tav_fold_groups(int device, int n_queries, int k, const int32_t* row_to_group, int64_t n_rows,
                    int64_t item_offset, int64_t* items, float* scores, int32_t* counts, void* stream);

/* Verification aid for the tensor-core path: every raw dot product it computes,
 * out_device[n_queries, size] float32 (device memory); float32 indexes go through their fp16 planes.  `flags` may
 * carry TAV_QUERIES_ON_DEVICE.  On a TAV_NORMALIZE index the queries are normalised first, as a search
 * does.  Synchronises.  Not a hot-path entry point. */
int tav_mma_scores(tav_index* ix, const float* queries, int n_queries, int flags, float* out_device,
                   void* stream);

/* Event timing is off by default (four fewer driver calls per search); enable it before the
 * searches you want timed: 1 = an event pair around every kernel, 2 = only around the dominant
 * kernel and the whole search (the pairs themselves cost ~1-2 us of device time per kernel
 * boundary).  Path and launch count are always recorded. */
int tav_set_timing(tav_index* ix, int enabled);

/* Device time of the last tav_search on this index, measured with CUDA events on the
 * search's stream: `scan_ms` = the dominant kernel (row-scan kernel, or the MAIN launch of the
 * tensor-core kernel; summed over query chunks), `total_ms` = first launch to last result byte on
 * device (both -1 when timing is off); `launches` = kernels launched; `path` = 1 row-scan
 * kernels, 2 tensor-core kernel on bf16/fp16 rows, 3 tensor-core kernel on a float32 index through
 * its two fp16 planes (x = hi + lo/2048, ~2^-22 relative).  Synchronises when timing is on. */
int tav_last_timing(tav_index* ix, float* scan_ms, float* total_ms, int* launches, int* path);

/* Per-kernel durations of the last tav_search, in launch order (up to `capacity` entries;
 * *n = number recorded): kinds[i] = 0 dominant kernel, 1 sample pass, 2 auxiliary kernel. */
int tav_timing_breakdown(tav_index* ix, float* ms, int* kinds, int capacity, int* n);

/* Device times of the last (up to 64, up to `capacity`) timed searches, oldest first: per search
 * the dominant kernel, the sample pass, the auxiliary kernels and first-launch-to-last-byte.
 * Lets a benchmark time its steps back to back and read the per-kernel times of the SAME pass
 * afterwards.  Synchronises on the last search's events. */
int tav_timing_history(tav_index* ix, int capacity, float* main_ms, float* sample_ms, float* aux_ms,
                       float* total_ms, int* n);

#ifdef __cplusplus
}
#endif
#endif /* TAVEC_H */
