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
 * as the work is enqueued.
 * The device work of the calls on one index runs in the order the calls were made, whatever
 * stream each call names: a call on another stream than the previous call's first makes its
 * stream wait (cudaStreamWaitEvent) for the work of the calls before it, and the calls without
 * a stream (tav_clear, tav_adopt_device, tav_reserve) wait for it on the host.  So a search queued
 * before tav_remove_rows / tav_write_rows sees the old rows and one queued after it the new ones,
 * whatever streams they name.  Consecutive
 * calls on one stream add no CUDA call for this.  Hazards in the caller's own buffers stay the
 * caller's: queries or a device row mask written on stream X and passed with stream Y, or
 * outputs read on another stream than the search's.
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
    TAV_ERR_STATE = -5,   /* operation not valid in this state (e.g. append to adopted memory) */
    TAV_ERR_PEER = -6     /* a sharded search failed on another rank (tav_sharded_*)     (RuntimeError) */
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
    TAV_NO_FUSED_SCAN = 128,
    /* With a subset only (otherwise TAV_ERR_INVALID): items are the POSITION of the hit in `subset`
     * (+ item_offset) instead of subset[position] (+ item_offset).  Which rows are scored, their keys and
     * the order are unchanged.  A row-sharded subset search uses it: positions stay distinct when the
     * subset repeats an ordinal, so the ranks' lists can be merged by position (tav_merge_topk_ordered
     * orders 2 / 3, tav_merge_range) and decoded through the caller's list afterwards (tav_map_items). */
    TAV_ITEMS_AS_POSITIONS = 256,
    /* Per-query row masks: query q may return only rows whose bit is set in mask q of
     * tav_set_query_masks.  n_queries must equal the number of masks set (else TAV_ERR_INVALID); with
     * TAV_USE_ROW_MASK or a subset: TAV_ERR_INVALID; without current masks: TAV_ERR_STATE.  Every path
     * (row scan, tensor cores, the exact redo, the threshold search and its re-pass) gives each query
     * exactly what a one-query search with its mask as the row mask gives. */
    TAV_USE_QUERY_MASKS = 512
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

/* Remove rows, as numpy.delete does: `ordinals` (host int64 [n]) may be negative (counted from the end),
 * repeated (one row removed) and in any order.  The surviving rows keep their order: row r becomes row
 * r - #{removed rows < r}.  Every search afterwards equals a search of a fresh index built from the
 * surviving rows.  The rows move on the device (an order-preserving compaction of the rows after the first
 * removed one, which are not written); nothing is re-uploaded.  The compaction runs in place, in
 * ascending windows through a buffer of at most 256 MB (smaller when that does not fit).  Any
 * ordinal out of range: TAV_ERR_RANGE and the index is
 * unchanged.  Adopted memory: TAV_ERR_STATE.  The row mask is dropped (ordinals change meaning); the
 * hits of the last threshold search are results and stay as they were.  Outstanding TAV_DEFER_RETRY
 * searches are finished first (their exact redo reads the rows).  Synchronises `stream` when rows move. */
int tav_remove_rows(tav_index* ix, const int64_t* ordinals, int64_t n, void* stream);

/* Overwrite rows [first, first + n) in place with `n` rows of `dim` elements of `src_dtype` from host
 * (src_on_device = 0) or device memory, converted exactly as tav_append converts (RNE; normalised on a
 * TAV_NORMALIZE index; host sources through the same pinned double buffer).  first + n beyond tav_size():
 * TAV_ERR_RANGE.  Adopted memory: TAV_ERR_STATE.  The row mask stays (ordinals keep their meaning).
 * Outstanding TAV_DEFER_RETRY searches are finished first.  Does not synchronise. */
int tav_write_rows(tav_index* ix, int64_t first, const void* rows, int64_t n, int dim, int src_dtype,
                   int src_on_device, void* stream);

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
 * subset ordinal + item_offset; scores float32) to host or device (TAV_OUTPUTS_ON_DEVICE) memory.
 * After a tav_range_search_into, TAV_ERR_STATE until the next tav_range_search. */
int tav_range_fetch(tav_index* ix, int64_t first, int64_t n, int64_t* out_items, float* out_scores,
                    int flags, void* stream);

/* Threshold search into the caller's device memory, sized on the device: the result of tav_range_search (same
 * order, score map, float32 compare, item_offset, shared subset of host ordinals, masks, NaN rules, path choice
 * and fp16-range fallback) without reading the hit counts back to the host first.
 *   out_offsets [n_queries + 1] int64   the full CSR offsets, also when out_offsets[n_queries] > capacity
 *   out_items   [capacity]      int64   every hit whose CSR position is below capacity; positions at or
 *   out_scores  [capacity]      float32 beyond it are never touched (the written hits are a prefix of the result)
 * Positions between the total and capacity are not written either, with one exception: when a tensor-core
 * re-pass (below) does not count what the first pass counted, the search is redone whole by the row scan, and
 * hits of the first pass may remain between the new total and capacity.  A caller that finds the total above
 * capacity can search again with enough room.  expected_hits sizes the collect regions as in tav_range_search
 * (0 = library default, 16384 per query); device scratch of about 2 x 8 bytes per key of the regions (1.5 x the
 * per-query share + 32, or twice that on the tensor cores) is held by the index.  Flags: QUERIES_ON_DEVICE,
 * FORCE_SCAN, FORCE_MMA, USE_ROW_MASK, USE_QUERY_MASKS, TIES_LOW_FIRST, DEFER_RETRY; any other flag,
 * capacity < 0 or a NULL output that is needed (items / scores with capacity > 0): TAV_ERR_INVALID.
 * A query whose collect region (row scan) or segment (tensor cores) overflowed is flagged and searched again at
 * the finish: all flagged queries of the search together, in one more pass of the collection that flagged them
 * (gathered queries, regions of their counted size; the tensor cores with the same plan, so the re-pass must
 * count what the first pass counted), sorted into these outputs at their offsets.  A split-form (float32 on the
 * tensor cores) search that met a value beyond the fp16 range writes no hits and is searched again whole by the
 * row scan, offsets included, as tav_range_search falls back.  Every search so redone counts its queries in
 * *redone.  Without TAV_DEFER_RETRY the call finishes itself before it returns (like tav_search, with the other
 * outstanding deferred searches): one synchronisation, and three or four when queries are searched again.
 * With TAV_DEFER_RETRY the call makes no host synchronisation (growing a device buffer may allocate; a repeat call
 * of the same shape does not) and joins the deferred searches tav_finish_search completes (at most 64
 * outstanding, shared with tav_search); until then only the flagged queries' outputs (the whole search's, when
 * flagged whole) are not final.  The caller keeps the device queries and the outputs alive until the finish (host
 * queries, normalised queries and the subset are held by the library).  The hits of the last tav_range_search
 * are given up (see tav_range_fetch); a finish never touches them. */
int tav_range_search_into(tav_index* ix, const float* queries, int n_queries, float min_score, int flags,
                          const int64_t* subset, int64_t subset_len, int64_t item_offset,
                          int64_t expected_hits, int64_t capacity,
                          int64_t* out_offsets, int64_t* out_items, float* out_scores, void* stream);

/*
 * Per-query subsets: one batched lookup in which query q scores only its own entries
 * ordinals[offsets[q] .. offsets[q + 1]) (the candidate re-ranking of fuzzy_lookup_embedding_in_subset,
 * vectorbase.py:203-230, for a whole batch).  `offsets` is host int64 [n_queries + 1], starting at 0 and never
 * decreasing, at most 2^32 - 1 in all; `ordinals` is host int64 [offsets[n_queries]].  Row q of the result equals,
 * bit for bit, tav_search (tav_range_search) of query q alone with its entries as the subset: repeated ordinals
 * are scored and returned once per occurrence, negative ordinals wrap like numpy and come back as given, equal
 * scores put the later entry first (the earlier with TAV_TIES_LOW_FIRST), an empty subset, an empty corpus or a
 * NaN min_score give no hits.  With TAV_ITEMS_AS_POSITIONS the item is the hit's flat index into `ordinals`.
 * Other accepted flags: TAV_QUERIES_ON_DEVICE, TAV_OUTPUTS_ON_DEVICE; any other flag, malformed offsets or more
 * than 2^32 - 1 ordinals: TAV_ERR_INVALID; an ordinal outside [-size, size): TAV_ERR_RANGE.  Every check runs on
 * the host before any work.  One gather reads each entry's row once (the row scan's arithmetic, path 1 in
 * tav_last_timing), and each query's hits are sorted by the threshold search's segmented sort; the number of
 * launches does not depend on n_queries.  Both calls synchronise once, to learn the hit counts, and replace the
 * hits of the last range search.
 *
 * tav_search_subsets: out_items / out_scores [n_queries, k], out_counts [n_queries]; count q is at most
 * min(k, entries of q); the slots after it hold item -1, score 0.
 * tav_range_search_subsets: CSR offsets out_offsets [n_queries + 1] of every hit at or above min_score;
 * tav_range_fetch copies the hits out.
 */
int tav_search_subsets(tav_index* ix, const float* queries, int n_queries, int k, float min_score, int flags,
                       const int64_t* offsets, const int64_t* ordinals, int64_t* out_items, float* out_scores,
                       int32_t* out_counts, void* stream);
int tav_range_search_subsets(tav_index* ix, const float* queries, int n_queries, float min_score, int flags,
                             const int64_t* offsets, const int64_t* ordinals, int64_t* out_offsets, void* stream);

/*
 * Per-query subsets from device memory: tav_search_subsets / tav_range_search_subsets for callers whose candidate
 * lists are already on the GPU, checked, planned and searched on the device with no host round trip.  Every pointer
 * is device memory on the index's device: queries float32 [n_queries, dim], offsets int64 [n_queries + 1], ordinals
 * int64 [n_ordinals], and the outputs.  Row q of the result equals, bit for bit, the host form's on the same CSR:
 * the same items, score bits, counts or offsets, order, repeats, negative ordinals returned as given and tie order.
 *
 * Flags: TAV_DEFER_RETRY, TAV_TIES_LOW_FIRST, TAV_ITEMS_AS_POSITIONS; TAV_QUERIES_ON_DEVICE and
 * TAV_OUTPUTS_ON_DEVICE are accepted and change nothing; any other flag: TAV_ERR_INVALID.  Checked on the host
 * before any work (TAV_ERR_INVALID): n_ordinals outside [0, 2^32 - 1], capacity < 0, k < 1, a NULL pointer that is
 * needed.  Checked on the device before any access: the offsets must start at 0, never decrease and end at
 * n_ordinals (else TAV_ERR_INVALID, and no work is planned); every ordinal must lie in [-size, size) (else
 * TAV_ERR_RANGE; the row of an ordinal outside is never read).  A refused search leaves counts 0, items -1 and
 * scores 0 (top-k form), or all offsets 0 with the items and scores untouched (threshold form).  No queries, no
 * entries, an empty index or a NaN min_score give no hits, and the ordinals are not looked at.
 *
 * Without TAV_DEFER_RETRY the call synchronises `stream` once, to read the device checks' status, and returns
 * their error.  With it the call makes no host synchronisation (growing a device buffer may allocate) and joins the
 * deferred searches tav_finish_search completes (at most 64 outstanding, shared with tav_search); the finish reports
 * a refusal after it has completed every other outstanding search, with the first such error.  The caller keeps
 * the queries, offsets, ordinals and outputs alive until then; on a TAV_NORMALIZE index the normalised queries are
 * held by the library.  The calls join the index's call order across streams, replace the hits of the last range
 * search (tav_range_fetch gives TAV_ERR_STATE afterwards, as after tav_range_search_into) and are timed as path 1.
 *
 * tav_search_subsets_into: out_items / out_scores [n_queries, k], out_counts [n_queries], padding item -1 and
 * score 0.  k is not clamped.
 * tav_range_search_subsets_into: the contract of tav_range_search_into's outputs.  out_offsets [n_queries + 1] is
 * always complete; hits at CSR positions >= capacity are not written, and those slots keep what they held.
 */
int tav_search_subsets_into(tav_index* ix, const float* queries, int n_queries, int k, float min_score, int flags,
                            const int64_t* offsets, const int64_t* ordinals, int64_t n_ordinals,
                            int64_t* out_items, float* out_scores, int32_t* out_counts, void* stream);
int tav_range_search_subsets_into(tav_index* ix, const float* queries, int n_queries, float min_score, int flags,
                                  const int64_t* offsets, const int64_t* ordinals, int64_t n_ordinals,
                                  int64_t capacity, int64_t* out_offsets, int64_t* out_items, float* out_scores,
                                  void* stream);

/* Completes EVERY outstanding TAV_DEFER_RETRY search of the index, whatever stream each was issued
 * on: waits until they have run (`stream` first waits for them, then is synchronised), redoes
 * each search's flagged queries exactly on `stream` into that search's own outputs and reports how many
 * (*redone).  The caller keeps the query and output buffers of deferred searches alive until
 * then.  Up to 64 searches may be outstanding (a 65th finishes the earlier ones first, and the
 * queries redone then are not counted in *redone).  On a TAV_NORMALIZE index each outstanding
 * search keeps its normalised queries in device memory of its own (grown as needed, never by
 * finishing searches early) until this call.  Deferred tav_range_search_into searches are completed
 * here too (their flagged queries searched again into their outputs at their offsets).  No-op when
 * nothing is pending. */
int tav_finish_search(tav_index* ix, void* stream, int* redone);

/* Row mask for TAV_USE_ROW_MASK: `n_rows` bits (bit r of word r/32 = row r allowed), host or
 * device memory; n_rows must equal tav_size().  Kept on the device until the rows change
 * (tav_clear / tav_adopt_device / tav_remove_rows drop it; appends invalidate it) or n_rows == 0
 * clears it.  tav_write_rows keeps it. */
int tav_set_row_mask(tav_index* ix, const uint32_t* bits, int64_t n_rows, int on_device, void* stream);

/* Per-query masks for TAV_USE_QUERY_MASKS: mask q is ceil(n_rows / 32) words (the bit order of
 * tav_set_row_mask) starting at bits + q * stride_words, in host or device memory.  n_rows must equal
 * tav_size() and stride_words must be at least ceil(n_rows / 32).  The masks are copied into library-owned
 * device memory, each padded to whole 256-row tiles: about n_queries * n_rows / 8 bytes.  An allocation
 * failure gives TAV_ERR_OOM and leaves the index usable, without masks.  n_queries == 0 clears them.  Same
 * lifecycle and ordering as the row mask: the call joins the index's call order, outstanding TAV_DEFER_RETRY
 * searches are finished first (their exact redo reads the masks they were issued with); tav_clear,
 * tav_adopt_device and tav_remove_rows drop the masks, appends invalidate them, tav_write_rows keeps them. */
int tav_set_query_masks(tav_index* ix, const uint32_t* bits, int n_queries, int64_t n_rows, int64_t stride_words,
                        int on_device, void* stream);

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
 * tav_merge_topk with a choice of the order among equal scores (`order`; anything else: TAV_ERR_INVALID):
 *   0  tav_merge_topk's: later list first, inside a list the earlier slot (higher row first);
 *   1  earlier list first, inside a list the earlier slot: lower row first for lists in ascending row
 *      blocks that were searched with TAV_TIES_LOW_FIRST (the predicate path);
 *   2  the item itself, higher first;  3  the item itself, lower first.  For lists whose items are
 *      distinct and in [0, 2^32), such as global subset positions (TAV_ITEMS_AS_POSITIONS), in any list
 *      order.  The merged items are those keys.
 * Same arguments, layout and limits as tav_merge_topk otherwise.
 */
int tav_merge_topk_ordered(int device, int n_lists, int n_queries, int k, const int64_t* items,
                           const float* scores, const int32_t* counts, int64_t items_stride,
                           int64_t scores_stride, int64_t counts_stride, int order, int64_t* out_items,
                           float* out_scores, int32_t* out_counts, void* stream);

/*
 * Device gather, in place: items[i] = table[items[i]] for every i < n with 0 <= items[i] < table_len;
 * other entries (the -1 padding of a [n_queries, k] result, for one) stay as they are.  `items` (int64 [n])
 * and `table` (int64 [table_len]) are device pointers on `device`; works on [n_queries, k] and CSR results
 * alike.  Enqueued on `stream`, no synchronisation.  n < 0, table_len < 0, or a NULL pointer that is
 * needed: TAV_ERR_INVALID.
 */
int tav_map_items(int device, int64_t n, const int64_t* table, int64_t table_len, int64_t* items, void* stream);

/*
 * Merge step of the row-sharded threshold search: `n_lists` per-shard CSR results of tav_range_search
 * (items already global: item_offset = the shard's first row) -> every hit of every list, per query, in
 * the library's order (score descending, then item descending, or ascending with ties_low_first).  List g:
 *   offsets + g * offsets_stride   [n_queries + 1] int64, starting at 0: query q's hits are
 *   items   + g * items_stride     [offsets[q], offsets[q + 1])  int64
 *   scores  + g * scores_stride                                  float32
 * (strides in elements), so one padded all-gather buffer is merged in place.  Each list must already be
 * in the library's order; items are compared as int64 and must be distinct across lists for the result
 * not to depend on the list order.  Scores are compared as float32 values (tav_range_search's are in
 * [0, 1]); they must not be NaN.  Outputs: out_offsets [n_queries + 1] = the per-query sums of the
 * lists' offsets, out_items / out_scores [out_offsets[n_queries]].  A merge (co-rank tiles spread evenly
 * over the GPU whatever the queries' sizes, each input hit read once), not a sort; no synchronisation
 * (8 * (n_queries + 1) bytes of stream-ordered scratch, cudaMallocAsync).  All pointers are device
 * pointers on `device` and must be non-NULL when n_queries > 0 (the counts live on the device);
 * 1 <= n_lists <= 32; negative strides are invalid; n_queries == 0 does nothing.  Lists with no hits
 * are normal input.
 */
int tav_merge_range(int device, int n_lists, int n_queries, const int64_t* offsets, int64_t offsets_stride,
                    const int64_t* items, int64_t items_stride, const float* scores, int64_t scores_stride,
                    int ties_low_first, int64_t* out_offsets, int64_t* out_items, float* out_scores,
                    void* stream);

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
 * stay valid until then), each merged again in the order it was first merged in.  A deferred search
 * beyond `depth`: TAV_ERR_STATE; a synchronous one finishes the open ones first.
 *
 * tav_sharded_search also takes TAV_USE_ROW_MASK, TAV_USE_QUERY_MASKS (each rank's masks cover its own
 * rows, set with tav_set_row_mask / tav_set_query_masks) and TAV_TIES_LOW_FIRST, which merges with
 * order 1 of tav_merge_topk_ordered (the lists come in rank order, each rank's block in ascending rows).
 *
 * tav_sharded_search_subset: the subset forms.  `subset` holds this rank's BLOCK-LOCAL host ordinals
 * (subset_len of them).  offsets == NULL: one subset shared by every query, searched as tav_search
 * with a subset; otherwise host int64 [n_queries + 1] CSR offsets of per-query subsets (offsets[0] == 0,
 * offsets[n_queries] == subset_len), searched as tav_search_subsets, which synchronises `stream` once.
 * The local search runs with TAV_ITEMS_AS_POSITIONS into this rank's slot, and tav_map_items through
 * `positions_device` (device int64 [subset_len]: where each entry stands in the caller's whole list, or
 * in the concatenation of the per-query lists) makes them global positions before the publish.  The
 * merge is by position, order 2 (3 with TAV_TIES_LOW_FIRST): the outputs are global positions, decoded
 * by the caller (tav_map_items through its list).  A rank without a share passes subset_len 0.  Other
 * accepted flags: TAV_DEFER_RETRY, TAV_FORCE_SCAN (shared subset only).
 *
 * Failures.  A sharded search that fails on a rank's host side (a local error other than TAV_ERR_CUDA:
 * an invalid argument, a missing mask, an allocation) still publishes an empty list with a status word
 * set, and returns that rank's own error; every rank's merge adds up the status words, and every other
 * rank gets TAV_ERR_PEER: on return for a synchronous call, from tav_sharded_finish for a deferred one
 * (which still completes every open search and its repairs).  A local TAV_ERR_CUDA is not published
 * (the device may be unusable): the peers' merges then wait about 4 s and trap.
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
int tav_sharded_search_subset(tav_index* ix, tav_group* g, const float* queries_device, int n_queries, int k,
                              float min_score, int flags, const int64_t* subset, int64_t subset_len,
                              const int64_t* offsets, const int64_t* positions_device, int64_t* out_items,
                              float* out_scores, int32_t* out_counts, void* stream);
int tav_sharded_finish(tav_index* ix, tav_group* g, void* stream, int* redone_total);

/*
 * Row-sharded threshold search through peer memory: every hit at or above min_score over every rank's rows, merged
 * on every rank (the result of tav_range_search over the whole corpus), with no NCCL call.  Its results have sizes
 * known only after the local search, so it uses a second allocation of the group, the RANGE INBOX:
 *
 *   range_arrive[world] u32 | range_ack[world] u32 | hdr[world][max_queries + 2] int64 |
 *   items[world][capacity] int64 | scores[world][capacity] float32
 *
 * Section r (rank r's CSR offsets [B + 1] and a word status | hits-included << 1, then its hits) is written only
 * by rank r, and tav_merge_range merges the world's sections in place.  The host side runs these steps on every
 * rank in lockstep, taking every decision from replicated data:
 *
 *   tav_group_range_reserve   frees this rank's inbox (closing its mappings of the peers' inboxes) and allocates
 *                             one for max_queries queries and `capacity` hits per rank (0, 0: only frees it).
 *                             Collective with _handle and _connect, as tav_group_create / _local_handle / _connect
 *                             are: the ranks quiesce and agree first, reserve, exchange the handles, connect.  The
 *                             new inbox counts its rounds from 0.  An allocation failure gives TAV_ERR_OOM and no
 *                             inbox; the host side then frees the inbox on every rank.
 *   tav_group_range_capacity  max_queries and capacity of the connected inbox (0, 0: none).
 *   tav_sharded_range_search  the local search (tav_range_search over this rank's rows, items + item_offset; with
 *                             TAV_ITEMS_AS_POSITIONS one subset of block-local ordinals, or per-query subsets with
 *                             CSR `offsets` as tav_range_search_subsets takes them, whose hits are mapped through
 *                             `positions` (host int64 [subset_len], copied to the device by the library) as
 *                             tav_sharded_search_subset maps them); it synchronises once, as tav_range_search
 *                             does.  Then round 1: this rank's header, and its hits when they fit in `capacity`,
 *                             stored into every peer's inbox over NVLink with a system-scope release flag; a wait
 *                             for every rank's round, and every rank's header to `world_headers` (host int64
 *                             [world][n_queries + 2]).  A second synchronisation, which sizes the result.
 *                             Flags: TAV_FORCE_SCAN, TAV_FORCE_MMA, TAV_USE_ROW_MASK, TAV_USE_QUERY_MASKS,
 *                             TAV_TIES_LOW_FIRST, TAV_ITEMS_AS_POSITIONS.  queries are host float32.
 *   tav_sharded_range_republish  round 2, when some rank's hits-included bit was 0: after every rank reserved an
 *                             inbox that holds the largest total, every rank publishes its whole list again (the
 *                             index still holds the hits) and waits for the world's.  Synchronises.
 *   tav_sharded_range_merge   tav_merge_range over the inbox into the caller's device outputs (out_offsets [B + 1],
 *                             out_items / out_scores [sum of the totals]), then this rank acknowledges the round to
 *                             its peers (also when the merge fails).  No synchronisation.
 *   tav_sharded_range_abort   closes an open search without a merge: this rank acknowledges its last round, so that
 *                             no peer's next publish waits for it.  For a caller that cannot merge (its output
 *                             buffers could not be allocated, say); its peers merge as usual.  No-op when nothing is
 *                             open.
 *
 * A search stays open from tav_sharded_range_search to its merge or abort: no other range search, and no search on
 * the index that would replace its hits, may run in between (a tav_sharded_range_search finding one open closes it
 * as tav_sharded_range_abort does).  Every rank calls the steps with the same n_queries and flags.
 *
 * Failures.  A threshold search whose local part fails on a rank (an error of the local tav_range_search* other than
 * TAV_ERR_CUDA: an argument it rejects, a missing mask, an allocation; or the allocation of the positions' device
 * copy) still publishes its header, with status 1 and no hits, and returns that rank's own error; every rank adds up
 * the world's status words, and every other rank gets TAV_ERR_PEER from tav_sharded_range_search.  Each rank
 * acknowledges such a round itself and the search is closed.  Not published, so that the peers' waits trap after
 * about 4 s: a local TAV_ERR_CUDA, and the checks tav_sharded_range_search makes before its local search (NULL or
 * malformed arguments, no connected inbox, more queries than it holds).  Those checks see only replicated state and
 * arguments, so a caller that makes every rank's call alike, and checks its arguments on every rank first (as
 * ShardedVectorBase does), never reaches them on one rank alone.
 */
int tav_group_range_reserve(tav_group* g, int max_queries, int64_t capacity);
int tav_group_range_handle(tav_group* g, void* handle_out /* tav_group_handle_bytes() */);
int tav_group_range_connect(tav_group* g, const void* handles /* world x tav_group_handle_bytes() */);
int tav_group_range_capacity(const tav_group* g, int* max_queries, int64_t* capacity);
int tav_sharded_range_search(tav_index* ix, tav_group* g, const float* queries, int n_queries, float min_score,
                             int flags, const int64_t* subset, int64_t subset_len, const int64_t* offsets,
                             const int64_t* positions, int64_t item_offset, int64_t expected_hits,
                             int64_t* world_headers, void* stream);
int tav_sharded_range_republish(tav_group* g, void* stream);
int tav_sharded_range_abort(tav_group* g, void* stream);
int tav_sharded_range_merge(tav_group* g, int ties_low_first, int64_t* out_offsets, int64_t* out_items,
                            float* out_scores, void* stream);

/*
 * Rebalance of row-sharded indexes (ShardedVectorBase.rebalance): every rank's new block is copied from the
 * ranks' current row allocations over CUDA IPC, in the storage dtype, byte for byte, by the copy engines.
 *
 *   tav_rows_export  writes this index's record (tav_rows_handle_bytes() bytes: the IPC handle of its row
 *                    allocation and its row count) to handle_out and the row count to *rows_out, after the
 *                    work queued by earlier calls on the index has run.  An index without rows gives a record
 *                    that no piece may read.  Adopted memory: TAV_ERR_STATE.
 *   tav_rows_stage   allocates this rank's new block (library-owned, capacity = its row count) and copies
 *                    `n_parts` pieces into it in order: piece i is rows [part_first[i], part_first[i] +
 *                    part_rows[i]) of rank part_src_rank[i]'s block, this index's own rows for
 *                    part_src_rank[i] == rank, the peers' through the records in `handles` (world records,
 *                    rank order).  A piece outside its source's rows: TAV_ERR_RANGE; a bad rank, or a source
 *                    whose rows have another width or dtype: TAV_ERR_INVALID; all checked on the host before
 *                    anything is allocated.  With `mirror_out` (host float32
 *                    [rows, dim]; a float32 index without TAV_NORMALIZE only, else TAV_ERR_INVALID) the staged
 *                    rows are also read back into it.  Joins the index's call order, finishes outstanding
 *                    TAV_DEFER_RETRY searches, synchronises `stream` and closes the peers' mappings before it
 *                    returns.  An allocation failure gives TAV_ERR_OOM; on any failure nothing stays staged and
 *                    the index is unchanged.  One staged block at a time: a second stage gives TAV_ERR_STATE.
 *   tav_rows_commit  commit = 1: the staged block becomes the index's rows, the old allocation is freed, the
 *                    row mask and per-query masks are dropped and the fp16 planes of a float32 index are
 *                    rebuilt from row 0 at the next tensor-core search (with their "left the fp16 range" flag).
 *                    Nothing staged: TAV_ERR_STATE.  commit = 0: the staged block is freed, nothing changes.
 *
 * Protocol: every rank exports, the records are exchanged (any host-side means), every rank stages, the ranks
 * agree that all stages succeeded (a rank has finished reading its peers' rows when its stage returns), then
 * every rank commits (or every rank drops).  No rank may change or free its rows between its export and the
 * agreement.
 */
int tav_rows_handle_bytes(void);
int tav_rows_export(tav_index* ix, void* handle_out, int64_t* rows_out);
int tav_rows_stage(tav_index* ix, int world, int rank, const void* handles, int n_parts, const int32_t* part_src_rank,
                   const int64_t* part_first, const int64_t* part_rows, float* mirror_out, void* stream);
int tav_rows_commit(tav_index* ix, int commit);

/*
 * Row-sharded search across the devices of ONE process (VectorBase(devices=[...])).  A tav_multi borrows W shard
 * indexes (1 <= W <= 32, created with tav_create as usual, distinct, any devices, a device may repeat), shard g
 * holding the contiguous block of global rows [starts[g], starts[g + 1]), in ascending block order.  It owns only the
 * workspace of the fan-out and the merge: one non-blocking stream and one event per shard on the shard's device, a
 * stream on `home_device`, and the buffers below.  tav_multi_create enables peer access between the distinct devices
 * where cudaDeviceCanAccessPeer allows it.  Destroy the tav_multi before its shards.  Calls on one tav_multi are
 * serialised by a mutex; every call restores the caller's current device.
 *
 * `starts` (host int64 [W + 1], starts[0] == 0) must match the shards' sizes (else TAV_ERR_INVALID).  Queries are host
 * float32 [n_queries, dim], outputs host memory; both calls synchronise once at the end.  Flags: TAV_FORCE_SCAN,
 * TAV_FORCE_MMA, TAV_USE_ROW_MASK (each shard's block of the mask set on that shard with tav_set_row_mask first; a
 * shard without rows ignores it) and TAV_TIES_LOW_FIRST; any other flag: TAV_ERR_INVALID.  The result equals, bit for
 * bit, the same call on one index holding every row: the per-shard searches are the library's searches of the blocks
 * (ordinals shifted by starts[g]) and the merges keep one index's order.
 *
 *   tav_multi_search        the queries are copied once into pinned memory and to each shard's device; every shard's
 *                           tav_search (both _ON_DEVICE flags, TAV_DEFER_RETRY) is launched before anything waits;
 *                           tav_finish_search completes each (the exact redo runs before the merge); each [B, k] list
 *                           is copied into a slab on the home device (cudaMemcpyPeerAsync), the home stream waits on the
 *                           shards' events and merges with tav_merge_topk_ordered (order 0, 1 with ties-low-first).
 *                           1 <= k <= 8192 (the merge's limit; tav_multi_range_search serves "every hit").
 *   tav_multi_range_search  every hit at or above min_score, CSR offsets out_offsets [n_queries + 1] (host).  Each
 *                           shard runs tav_range_search_into with TAV_DEFER_RETRY into buffers of the tav_multi sized
 *                           from expected_hits (the whole batch's hint, as tav_range_search takes it); after the
 *                           finishes a shard whose total exceeds its room is searched again with room enough.  The
 *                           shards' CSR results are copied to the home device and merged by tav_merge_range.  The hits
 *                           stay in the tav_multi until the next tav_multi_range_search.
 *   tav_multi_range_fetch   copies hits [first, first + n) of the last tav_multi_range_search to host memory
 *                           (TAV_ERR_RANGE beyond its total).
 *
 * Subset: the host ordinals are split by block on the host (negative ordinals wrap against the global row count
 * starts[W]; any ordinal outside [-starts[W], starts[W]): TAV_ERR_RANGE before any work).  Each shard searches its share
 * with block-local ordinals and TAV_ITEMS_AS_POSITIONS (a threshold search of a share runs tav_range_search, which
 * synchronises, then tav_range_fetch), the positions are mapped to positions in the caller's subset, merged by
 * position (top-k order 2, or 3 with ties-low-first) and decoded through the caller's subset (tav_map_items): repeats,
 * negative ordinals and the subset's tie order come back as one index returns them.
 *
 * Errors: a shard that fails fails the call with its status and message; every other shard is still finished and its
 * stream synchronised, so nothing is left outstanding, and the tav_multi and every index stay usable.
 */
typedef struct tav_multi tav_multi;
int tav_multi_create(int home_device, int n_shards, tav_index* const* shards, tav_multi** out);
int tav_multi_destroy(tav_multi* m);
int tav_multi_search(tav_multi* m, const int64_t* starts, const float* queries, int n_queries, int k, float min_score,
                     int flags, const int64_t* subset, int64_t subset_len, int64_t* out_items, float* out_scores,
                     int32_t* out_counts);
int tav_multi_range_search(tav_multi* m, const int64_t* starts, const float* queries, int n_queries, float min_score,
                           int flags, const int64_t* subset, int64_t subset_len, int64_t expected_hits,
                           int64_t* out_offsets);
int tav_multi_range_fetch(tav_multi* m, int64_t first, int64_t n, int64_t* out_items, float* out_scores);

/*
 * Chunk -> message fold of hit lists, on the device, in place (storage/memory/messageindex.py:
 * 185-207 `to_scored_message_ordinals`; the reference folds AFTER the top-k over chunks): walking
 * each query's hits in score order, the first hit of a group keeps its score, later hits of the
 * same group are dropped; items become group ordinals `row_to_group[item - item_offset]` (device
 * int32 [n_rows]); counts are updated, tails padded with -1 / 0.  k <= 8192.
 */
int tav_fold_groups(int device, int n_queries, int k, const int32_t* row_to_group, int64_t n_rows,
                    int64_t item_offset, int64_t* items, float* scores, int32_t* counts, void* stream);

/*
 * Grouped lookups: the k best GROUPS of rows (messages, when rows are their chunks), each group scored by its best
 * row.  Exact, unlike tav_fold_groups after a top-k, which returns fewer than k groups when the best rows of a few
 * groups fill the k slots.  Definition: take query q's hit list of tav_range_search with the same min_score, masks
 * and tie order; a group's LEADER is its first row in that list; the grouped result is the list of leaders in that
 * order (group id, the leader's score, the leader's row).  So groups come by score descending, equal scores with
 * the higher leader row first (the lower with TAV_TIES_LOW_FIRST), a group with no passing row does not appear, and
 * the grouped top-k is the first k entries of the grouped threshold search.
 *
 * tav_set_row_groups: groups[r] (int32 [n_rows], host or device memory) is the group of row r; n_rows must equal
 * tav_size(), and n_rows == 0 clears the map.  Values must lie in [0, 2^31): a negative one gives TAV_ERR_INVALID
 * and leaves the index as it was.  The map is copied into library-owned device memory and checked there by a kernel
 * (one synchronisation).  Lifecycle and call order of the row mask: outstanding TAV_DEFER_RETRY searches are
 * finished first; tav_clear, tav_adopt_device, tav_remove_rows and a rebalance commit drop the map, appends
 * invalidate it, tav_write_rows keeps it.
 *
 * tav_range_search_groups: every group's leader per query, CSR offsets out_offsets [n_queries + 1] (host, or device
 * with TAV_OUTPUTS_ON_DEVICE).  The collection, path choice, sizing, hint, re-pass and fp16-range fallback of
 * tav_range_search, then the leader reduction (each query's keys through an open-addressing table of twice their
 * count), then the segmented sort over the leaders only.  The leaders stay in the index until the next threshold
 * search; tav_range_fetch_groups copies leaders [first, first + n) out (host, or device with TAV_OUTPUTS_ON_DEVICE):
 * out_groups int64, out_scores float32, out_rows int64.  After any other threshold search: TAV_ERR_STATE.
 * Synchronises twice (the hit counts, then the leader counts).
 *
 * tav_search_groups: out_groups / out_scores / out_rows [n_queries, k], out_counts [n_queries]; padding group -1,
 * score 0, row -1.  It runs tav_search for the top kp rows of each query (kp = k times the rows per run of equal
 * group ids in the map, at most 2048 and at least k; the path choice of tav_search), reduces that prefix to its
 * leaders and sorts them.  A prefix's leaders are the first leaders of the whole list, so a query whose prefix is
 * all its hits, or holds k groups, is exact; every other query is redone by the grouped threshold search of that
 * query alone and cut to k, and *redone (may be NULL) reports how many.  When kp covers the rows the grouped
 * threshold search serves the whole call.  Synchronises (to size the leaders and the redo); replaces the hits of
 * the last threshold search.
 *
 * Flags of the three searches: TAV_QUERIES_ON_DEVICE, TAV_OUTPUTS_ON_DEVICE, TAV_FORCE_SCAN, TAV_FORCE_MMA,
 * TAV_USE_ROW_MASK, TAV_USE_QUERY_MASKS, TAV_TIES_LOW_FIRST; any other flag: TAV_ERR_INVALID.  No current map (none
 * set, or set for another row count) on a non-empty index: TAV_ERR_STATE.  An empty index or a NaN min_score gives
 * no hits.
 */
int tav_set_row_groups(tav_index* ix, const int32_t* groups, int64_t n_rows, int on_device, void* stream);
int tav_range_search_groups(tav_index* ix, const float* queries, int n_queries, float min_score, int flags,
                            int64_t expected_hits, int64_t* out_offsets, void* stream);
int tav_range_fetch_groups(tav_index* ix, int64_t first, int64_t n, int64_t* out_groups, float* out_scores,
                           int64_t* out_rows, int flags, void* stream);
int tav_search_groups(tav_index* ix, const float* queries, int n_queries, int k, float min_score, int flags,
                      int64_t* out_groups, float* out_scores, int64_t* out_rows, int32_t* out_counts, void* stream,
                      int* redone);

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
