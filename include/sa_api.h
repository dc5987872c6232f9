/* sa_api.h -- C ABI of the H100-native vector-search engine (libsa_b200.so).
 *
 * This is the drop-in boundary for the one data-parallel path of confluentinc/quickstart-streaming-agents:
 * the Lab2 RAG lookup that the reference runs as Flink SQL inside Confluent Cloud against a MongoDB Atlas
 * vector index.  The reference has no FFI of its own (it is Python glue + Terraform; SURVEY.md section 2.1),
 * so each entry point cites the reference statement / script whose work it takes over.  A Python caller
 * binds these with ctypes (quickstart-streaming-agents_b200/capi.py; INTEGRATION.md shows the stub).
 *
 * Conventions
 *   - every function returns 0 on success, a negative sa_status otherwise; sa_last_error() has the detail;
 *   - "dev" pointers are CUDA device pointers on the engine's device, "host" pointers are ordinary memory;
 *   - the caller owns every data buffer (a torch tensor is just an allocator here); the library owns only
 *     its own scratch, pinned staging and TMA descriptors and never copies the corpus;
 *   - `stream` is a cudaStream_t passed as an integer (0 = the legacy default stream); device entry points
 *     are asynchronous on it, *_host entry points block until their result is in host memory;
 *   - an engine serves one CUDA device and is not re-entrant;
 *   - there is no CPU fallback: on a device that is not sm_90 sa_engine_create fails with SA_ERR_DEVICE.
 */
#ifndef SA_API_H_
#define SA_API_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct sa_engine sa_engine;

typedef enum sa_status {
  SA_OK = 0,
  SA_ERR_CUDA = -1,     /* a CUDA runtime / driver call failed */
  SA_ERR_ARG = -2,      /* bad argument (null, range, alignment, dim % 64 != 0, k > max_k ...) */
  SA_ERR_COMM = -3,     /* NCCL could not be loaded / a collective call failed (sa_comm_*) */
  SA_ERR_CAPACITY = -4, /* append past capacity_rows, batch past max_batch */
  SA_ERR_DEVICE = -5    /* device is not compute capability 9.0 */
} sa_status;

/* Similarity of an index, fixed at creation (Atlas's vector index "similarity": cosine, dotProduct, euclidean).
 * The ranking and the returned score per similarity (all arithmetic over the bf16-rounded values, sums in float64):
 *   SA_SIM_COSINE     cosine desc, row asc;         score = cosine;        all-zero rows are never returned
 *   SA_SIM_DOT        <q,c> desc, row asc;          score = <q,c>;         an all-zero row is a live row (score 0)
 *   SA_SIM_EUCLIDEAN  |q - c| asc, row asc;         score = |q - c| = sqrt(max(0, (|q|^2 - 2<q,c>) + |c|^2));
 *                                                   an all-zero row is a live row (distance |q|)
 * Empty result slots hold row -1 with the worst value: -inf, or +inf for distances. */
#define SA_SIM_COSINE 0
#define SA_SIM_DOT 1
#define SA_SIM_EUCLIDEAN 2

/* Element type of an index, fixed at creation: the type of its rows and of the queries of its device search forms.
 *   SA_ELEM_BF16  rows and queries are bf16 (sa_engine_create, sa_engine_create_sim)
 *   SA_ELEM_INT8  rows and queries are int8 (Atlas's int8 vectors, pre-quantized int8 embeddings).  The definition above
 *                 is evaluated on the integers themselves; every sum is exact, so cosine is <q,c> / sqrt(|q|^2 |c|^2),
 *                 dotProduct the integer <q,c>, and the distance one correctly rounded sqrt of an exact integer.  There
 *                 is no scale factor: scores are in the integers' own units.  fp32 input to an int8 index (the *_f32
 *                 and *_host forms, sa_gather_merge*) is converted by one rule: round to nearest even, saturate to
 *                 [-128, 127], NaN -> 0 (sa_debug_int8_round), so integer-valued floats in range pass unchanged.
 * Pointers documented below as "*_bf16_dev" (the rows of sa_corpus_bind, the queries of sa_search, sa_search_filtered,
 * sa_search_hits*, sa_sharded_search* and sa_debug_tile_dots) point to elements of the engine's type. */
#define SA_ELEM_BF16 0
#define SA_ELEM_INT8 1

/* Largest k of a search.  Candidate lists hold 16 (k <= 16) or 32 entries per tile lane; a "deep" search (28 < k <= 64)
 * keeps the 32-entry lists and runs a scan variant whose shared bounds hold for its k (DESIGN.md section 4.1). */
#define SA_MAX_K 64
/* Largest dim of either element type: the exact fallback scan stages one query row (2 SA_MAX_DIM bytes of bf16) in
 * shared memory, and an int8 |<q,c>| <= dim 2^14 stays inside the int32 accumulators. */
#define SA_MAX_DIM 65536
#define SA_HOST_SLOTS 2 /* host-buffer searches that may be in flight at once (sa_search_host_submit) */

int sa_version(void);
const char* sa_strerror(int rc);
const char* sa_last_error(void); /* thread-local detail of the last failure on this thread */

/* --- engine -------------------------------------------------------------------------------------------
 * Replaces the external vector table + index declaration:
 *   CREATE TABLE documents_vectordb_lab2 (... embedding ARRAY<FLOAT>) WITH ('connector'='mongodb',
 *   'mongodb.index'='vector_index', 'mongodb.embedding_column'='embedding', ...)
 *   (terraform/lab2-vector-search/main.tf:215) and the index definition {numDimensions 1536, similarity cosine}
 *   (assets/pre-setup/MongoDB-Setup.md:72-83, scripts/common/validate.py:56-61,167-180).
 * dim must be a multiple of 64 (1536 and 768 are) and at most SA_MAX_DIM; capacity_rows < 2^31; max_k <= SA_MAX_K.
 * sa_engine_create makes a cosine index; sa_engine_create_sim takes the similarity (SA_SIM_*) and rejects any other value
 * with SA_ERR_ARG before it touches a device.  sa_engine_create_elem also takes the element type (SA_ELEM_*;
 * sa_engine_create_sim is it with SA_ELEM_BF16); an int8 index needs dim to be a multiple of 128.  An unknown elem or
 * such a dim (of either type) is rejected with SA_ERR_ARG before it touches a device. */
int sa_engine_create(sa_engine** out, int device, int dim, int64_t capacity_rows, int max_batch, int max_k);
int sa_engine_create_sim(sa_engine** out, int device, int dim, int64_t capacity_rows, int max_batch, int max_k,
                         int similarity);
int sa_engine_create_elem(sa_engine** out, int device, int dim, int64_t capacity_rows, int max_batch, int max_k,
                          int similarity, int elem);
void sa_engine_destroy(sa_engine* e);

/* Attach caller-owned device storage: rows_bf16 is [capacity_rows x dim] row-major of the engine's element type (bf16
 * or int8; 16-byte aligned), row_term is [capacity_rows] fp32 (16-byte aligned), one term per row that the scan
 * combines with <q,c>:
 *   cosine      1/|c| over the stored values (int8: rounded once from fp64), 0 for an all-zero row or a tombstone
 *   dotProduct  1 for a live row, 0 for a tombstone
 *   euclidean   |c|^2/2 (summed in fp64, rounded once to fp32) for a live row, negative (e.g. -1) for a tombstone
 * A bf16 row holding a NaN or an infinite element is not live under any similarity: ingest gives it the tombstone term
 * (cosine 0, dotProduct 0, euclidean -1), it never enters the norm bound below, and no search returns it.
 * The ingest entry points below write it; a caller that tombstones a row writes the row's term itself (and may zero the
 * row).  n_valid rows are taken as already committed (their terms valid); for dotProduct and euclidean the bound on the
 * rows' norms that the search's certificate uses is recomputed over them. */
int sa_corpus_bind(sa_engine* e, void* rows_bf16_dev, float* row_term_dev, int64_t n_valid);

/* --- pre-filtered search (the "filter" of Atlas's $vectorSearch over an index's {"type": "filter"} fields) ----------
 * Row tags: one caller-owned 64-bit word per row, a device array of [capacity_rows] entries, 16-byte aligned.  A set bit
 * means "this row carries value v of filter field f"; which bit stands for which (field, value) is the caller's mapping
 * (the Python layer's FilterSchema).  Tags of rows at or past the committed row count are never read.  The caller
 * writes a new row's tag before it appends or commits the row, exactly as with the row itself; tags of committed rows
 * may be rewritten between searches.  row_tags_dev == NULL detaches the array. */
int sa_corpus_bind_tags(sa_engine* e, uint64_t* row_tags_dev);

/* The per-query predicate in one fixed normal form.  Row r is eligible for query i iff it is live (as for an unfiltered
 * search) and pass(tags[r], filters[i]):
 *   (t & all_of) == all_of  and  (t & none_of) == 0  and  for each j: any_of[j] == 0 or (t & any_of[j]) != 0
 * All zero matches every row.  The search's answer is then exactly the unfiltered definition over the eligible rows
 * (fewer than k eligible rows: the remaining slots are empty). */
typedef struct sa_filter {
  uint64_t all_of;    /* every bit must be set on the row */
  uint64_t none_of;   /* no bit may be set */
  uint64_t any_of[2]; /* each nonzero word: at least one of its bits must be set; 0 = no constraint */
} sa_filter;          /* all zero = matches every row */

/* --- ingest (the "documents -> documents_embed -> MongoDB sink" half of Lab2, LAB2-Walkthrough.md:41-51,
 *     fed by scripts/publish_docs.py:225-351; embeddings arrive as ARRAY<FLOAT>, main.tf:141,215) ------- */
/* Rows [first_row, first_row+n_new) were written in place (bf16 or int8, the engine's element type) by the caller:
 * compute their row terms and publish them (first_row must equal the current row count). */
int sa_corpus_commit(sa_engine* e, int64_t first_row, int64_t n_new, uintptr_t stream);
/* Convert n_new fp32 rows (device) to the element type (bf16: round-to-nearest-even; int8: see SA_ELEM_INT8), append,
 * compute row terms, publish. */
int sa_corpus_append_f32(sa_engine* e, const float* rows_f32_dev, int64_t n_new, uintptr_t stream);
/* Same from host memory (staged through pinned memory in chunks); blocking. */
int sa_corpus_append_host_f32(sa_engine* e, const float* rows_f32_host, int64_t n_new);
/* Forget all rows -- what scripts/common/clear_mongodb.py:98-158 (delete_many({})) does to the collection.  For
 * dotProduct and euclidean it also clears the norm bound, and then waits for the device. */
int sa_corpus_reset(sa_engine* e);
int64_t sa_corpus_rows(const sa_engine* e);

/* --- search: LATERAL TABLE(VECTOR_SEARCH_AGG(documents_vectordb_lab2, DESCRIPTOR(embedding),
 *     qe.embedding, k))  (terraform/lab2-vector-search/main.tf:292; LAB3-Walkthrough.md:343-350;
 *     LAB4-Walkthrough.md:302-309) for a batch of nq query vectors --------------------------------------
 * Result for query i: out_idx[i*k .. i*k+k) = shard-local rows of the k best committed corpus rows under the
 * engine's similarity (see SA_SIM_*: descending cosine or dot product, ascending distance; ties by ascending row);
 * out_score = their scores (fp32 rounding of the fp64 value); slots past the number of eligible rows hold idx -1 /
 * score -inf (+inf for distances).  Tombstoned rows are never returned, nor all-zero rows under cosine.
 * out_score64 (optional, may be NULL) receives the unrounded scores for a cross-shard merge. */
int sa_search(sa_engine* e, const void* q_bf16_dev, int nq, int k, float* out_score_dev, int32_t* out_idx_dev,
              double* out_score64_dev, uintptr_t stream);
/* Queries as fp32 (the ML_PREDICT output type, terraform/core/main.tf:500,534): converted to the element type first
 * (bf16: round-to-nearest-even; int8: see SA_ELEM_INT8).  The host forms below convert the same way. */
int sa_search_f32(sa_engine* e, const float* q_f32_dev, int nq, int k, float* out_score_dev, int32_t* out_idx_dev,
                  double* out_score64_dev, uintptr_t stream);
/* End-to-end call with HOST buffers: H2D of the queries, search, D2H of the results; blocking. */
int sa_search_host(sa_engine* e, const float* q_f32_host, int nq, int k, float* out_score_host,
                   int32_t* out_idx_host);

/* The same call split in two, so a serving loop can decode / stage batch i+1 while the GPU works on batch i:
 * submit enqueues H2D + search + D2H for `slot` (0 .. SA_HOST_SLOTS-1) and returns at once; wait blocks until that
 * slot's results are in host memory and copies them out.  Searches execute in submission order.  A pageable query
 * buffer may be reused as soon as submit returns; a page-locked one must stay unchanged until the matching wait. */
int sa_search_host_submit(sa_engine* e, int slot, const float* q_f32_host, int nq, int k);
int sa_search_host_wait(sa_engine* e, int slot, float* out_score_host, int32_t* out_idx_host);

/* Filtered twins of the searches above: `filters` holds nq sa_filter entries, device memory for the device forms and
 * host memory for the host forms.  They fail with SA_ERR_ARG when filters is NULL or the engine has no tags bound
 * (sa_corpus_bind_tags).  The host forms stage the filters in the slot's own pinned and device buffers, so the caller
 * may reuse its filter array as soon as the call returns; sa_search_host_wait collects a filtered submit as well. */
int sa_search_filtered(sa_engine* e, const void* q_bf16_dev, const sa_filter* filters_dev, int nq, int k,
                       float* out_score_dev, int32_t* out_idx_dev, double* out_score64_dev, uintptr_t stream);
int sa_search_f32_filtered(sa_engine* e, const float* q_f32_dev, const sa_filter* filters_dev, int nq, int k,
                           float* out_score_dev, int32_t* out_idx_dev, double* out_score64_dev, uintptr_t stream);
int sa_search_host_filtered(sa_engine* e, const float* q_f32_host, const sa_filter* filters_host, int nq, int k,
                            float* out_score_host, int32_t* out_idx_host);
int sa_search_host_submit_filtered(sa_engine* e, int slot, const float* q_f32_host, const sa_filter* filters_host, int nq,
                                   int k);

/* --- multi-GPU (SURVEY.md section 8e): the corpus is row-sharded, every GPU searches its shard with the same single-GPU
 *     path, the per-shard results cross NVLink in ONE all-gather of packed (cosine f64, global row) lists -- nq*k*16 bytes
 *     per rank -- and every rank merges them to the global top-k by (cosine desc, global row asc).  This is the whole of
 *     what the sharded VECTOR_SEARCH_AGG (main.tf:292) needs; there is no all-reduce and no all-to-all. ------------------ */
typedef struct sa_hit {
  double score; /* the returned score, float64: cosine, dot product or Euclidean distance (the engine's similarity) */
  int64_t row;  /* global row = shard-local row + row_offset, -1 = no row */
} sa_hit;

/* This shard's results in exchange format (device buffer [nq x k]), e.g. for a caller-run collective. */
int sa_search_hits(sa_engine* e, const void* q_bf16_dev, int nq, int k, int64_t row_offset, sa_hit* out_hits_dev,
                   uintptr_t stream);
/* Filtered twin (filters_dev: [nq] on the device); each shard filters by its own tags. */
int sa_search_hits_filtered(sa_engine* e, const void* q_bf16_dev, const sa_filter* filters_dev, int nq, int k,
                            int64_t row_offset, sa_hit* out_hits_dev, uintptr_t stream);
/* Merge gathered hit lists [n_shards x nq x k] into the global top-k: out_score [nq x k] fp32, out_row [nq x k] int64.
 * The order is that of e's similarity (ascending for distances). */
int sa_merge_hits(sa_engine* e, const sa_hit* hits_dev, int n_shards, int nq, int k, float* out_score_dev,
                  int64_t* out_row_dev, uintptr_t stream);
/* Older split form of the same merge (separate score / row arrays). */
int sa_merge_shards(sa_engine* e, const double* score64_dev, const int64_t* global_idx_dev, int n_shards, int nq,
                    int k, float* out_score_dev, int64_t* out_idx_dev, uintptr_t stream);

/* Communicator.  NCCL is loaded at run time (dlopen): the copy already loaded in the process if any (e.g. torch's), else
 * the path given to sa_comm_set_library / $SA_NCCL_LIB, else the system libnccl.so.2.  Failures return SA_ERR_COMM. */
#define SA_COMM_ID_BYTES 128
typedef struct sa_comm sa_comm;
int sa_comm_set_library(const char* path);
int sa_comm_nccl_version(int* version, char* path_out, int path_cap);
/* single process driving n_gpus devices (ncclCommInitAll); devices == NULL means 0 .. n_gpus-1 */
int sa_comm_create(sa_comm** out, int n_gpus, const int* devices);
/* one process per GPU: rank 0 calls sa_comm_unique_id, ships the 128 bytes to the others out of band, all call create_rank */
int sa_comm_unique_id(void* id_out_128);
int sa_comm_create_rank(sa_comm** out, int n_ranks, int rank, const void* id_128, int device);
void sa_comm_destroy(sa_comm* c);
int sa_comm_ranks(const sa_comm* c);

/* One process per GPU: this rank's part of a sharded search (collective: every rank must call it with the same nq, k).
 * The first search on a communicator also compares the ranks' similarities (one small all-gather, blocking) and every
 * rank fails with SA_ERR_ARG if they differ; sa_gather_merge* fails the same way if the engines' similarities differ.
 * Device form, asynchronous on `stream`: out_score [nq x k] fp32, out_row [nq x k] int64 global rows, same on all ranks. */
int sa_sharded_search(sa_comm* c, sa_engine* e, const void* q_bf16_dev, int nq, int k, int64_t row_offset,
                      float* out_score_dev, int64_t* out_row_dev, uintptr_t stream);
/* Host-buffer form, split like sa_search_host_submit/_wait (slots 0 .. SA_HOST_SLOTS-1, two batches in flight). */
int sa_sharded_search_host_submit(sa_comm* c, sa_engine* e, int slot, const float* q_f32_host, int nq, int k,
                                  int64_t row_offset);
int sa_sharded_search_host_wait(sa_comm* c, sa_engine* e, int slot, float* out_score_host, int64_t* out_row_host);
/* Filtered twins: every rank passes the same filters; each filters its shard by its own tags. */
int sa_sharded_search_filtered(sa_comm* c, sa_engine* e, const void* q_bf16_dev, const sa_filter* filters_dev, int nq,
                               int k, int64_t row_offset, float* out_score_dev, int64_t* out_row_dev, uintptr_t stream);
int sa_sharded_search_host_submit_filtered(sa_comm* c, sa_engine* e, int slot, const float* q_f32_host,
                                           const sa_filter* filters_host, int nq, int k, int64_t row_offset);

/* Single process, all GPUs of the communicator: host fp32 queries in, merged host results out.  engines[g] lives on the
 * communicator's device g and holds the shard whose first global row is shard_offsets[g].  sa_gather_merge blocks;
 * the _submit/_wait pair keeps two batches in flight. */
int sa_gather_merge(sa_comm* c, sa_engine* const* engines, const float* q_f32_host, int nq, int k,
                    const int64_t* shard_offsets, float* out_score_host, int64_t* out_row_host);
int sa_gather_merge_submit(sa_comm* c, sa_engine* const* engines, int slot, const float* q_f32_host, int nq, int k,
                           const int64_t* shard_offsets);
int sa_gather_merge_wait(sa_comm* c, sa_engine* const* engines, int slot, float* out_score_host, int64_t* out_row_host);
/* Filtered twins (filters_host: [nq] host sa_filter, the same for every shard; every engine needs its tags bound). */
int sa_gather_merge_filtered(sa_comm* c, sa_engine* const* engines, const float* q_f32_host, const sa_filter* filters_host,
                             int nq, int k, const int64_t* shard_offsets, float* out_score_host, int64_t* out_row_host);
int sa_gather_merge_submit_filtered(sa_comm* c, sa_engine* const* engines, int slot, const float* q_f32_host,
                                    const sa_filter* filters_host, int nq, int k, const int64_t* shard_offsets);

/* --- observability ------------------------------------------------------------------------------------
 * CUDA-event times of the most recent search on this engine (synchronises on its last event):
 * scan_ms = sum over its scan-kernel launches, total_ms = first scan start to last merge end,
 * bytes / flops = ALGORITHMIC work of that search (DESIGN.md section 5; rows and queries at 2 bytes per bf16 element,
 * 1 per int8 element; for an int8 engine "flops" are int8 operations, same formula), launches = scan launches,
 * kernels = all kernels the search launched. */
int sa_last_timing(sa_engine* e, float* scan_ms, float* total_ms, double* bytes, double* flops, int* launches,
                   int* kernels);
/* Mean scan / total milliseconds over the most recent min(n, 16) searches (a ring of CUDA events is kept, so
 * back-to-back searches can be timed without a host synchronisation between them). */
int sa_timing_mean(sa_engine* e, int n, float* scan_ms_mean, float* total_ms_mean, int* n_used);
/* Options: "cta_group" = 0 (auto) | 1 | 2;  "max_launch_qblocks" = cap on query blocks per scan launch;
 * drift control between query blocks that share corpus tiles (keeps a shared tile L2-resident so it crosses HBM
 * once): "max_drift" = unpaced lead in tiles (-1 auto), "pace_gain" = delay cycles per K-slice per extra tile
 * of lead (-1 auto, 0 off), "pace_max" = cap of that delay (-1 auto);
 * "share_thresholds" = 1 | 0 (tile lanes exchange per-query top-k thresholds; default 1), "list_len" = 0 (auto) | 16 | 32
 * (16 serves k <= 16, 32 every k <= SA_MAX_K),
 * "window_bound" = 1 | 0 (with >= 16 tile lanes, a lane also bounds its threshold by the (list_len/2)-th largest of 16
 * lanes' second-best scores -- list_len rows in all -- which is far tighter while the lists are young; a deep search, k > 28,
 * takes the 14th largest of their 5th-best scores, 70 rows; default 1),
 * "presample" = S (a pre-pass over every S-th tile seeds those thresholds, so the order of the rows cannot hurt; 0 off, -1 auto),
 * "unit_map" = 0 | 1 (CTA -> (query block, tile lane) mapping), "record_times" = 0 | 1 (per-CTA timestamps),
 * "profile" = 0 | 1 (run the scan's profiling build: per-CTA role wait/busy cycle counters, see sa_scan_profile),
 * "force_fix" = 0 | 1 (test hook: route every (query, tile lane) through the exact fallback scan),
 * "count_fix" = 0 | 1 (record how many (query, lane) pairs the last search sent to the fallback; costs a host sync). */
int sa_set_option(sa_engine* e, const char* name, int64_t value);
/* "num_sms", "dim", "capacity", "n_rows", "max_batch", "max_k", "last_grid", "last_fix_entries" (with "count_fix"),
 * "eps_rel_e12" (the certificate's relative error bound, times 1e12; int8: a constant, DESIGN.md section 4.2),
 * "similarity" (SA_SIM_*), "elem" (SA_ELEM_*), "cmax_bits" (fp32 bits of
 * the device-side upper bound on the committed rows' norms; dotProduct and euclidean only, 0 for cosine; synchronous),
 * "has_tags" (1 when a row tag array is bound, sa_corpus_bind_tags). */
int sa_get_info(const sa_engine* e, const char* name, int64_t* value);
/* Per-CTA profile records of the last scan launch run with "profile" = 1 (synchronises the device): out_host receives
 * n_ctas x 8 int64 {TMA producer wait for a free slot, MMA issuer wait for data, MMA issuer wait for the epilogue,
 * epilogue wait for the MMA, epilogue busy, epilogue 32-column chunks on the insertion path, CTA lifetime, tiles}, SM cycles. */
int sa_scan_profile(sa_engine* e, int64_t* out_host, int max_ctas, int* n_ctas);

/* Test hook: raw fp32 Q.C^T accumulators (int8: the exact int32 accumulators rounded to fp32) of one 256-row corpus tile
 * for the first nq queries (of the engine's element type),
 * out_dots_dev is [ceil(nq/(128*cg))*128*cg x 256].  Runs the scan kernel's debug instantiation. */
int sa_debug_tile_dots(sa_engine* e, const void* q_bf16_dev, int nq, int tile, int cta_group, float* out_dots_dev,
                       uintptr_t stream);

/* Test hook (pure host logic, no GPU needed): how a batch of nq queries is split into scan launches on a device
 * with num_sms SMs.  out receives up to max_out rows of {first query, queries, query blocks, tile lanes}. */
int sa_debug_plan(int num_sms, int nq, int cta_group, int num_tiles, int max_launch_qblocks, int* out, int max_out,
                  int* n_launches);

/* Test hooks over the kernels' pure helper functions, compiled for the host (no GPU needed): the order-preserving
 * score keys of the shared thresholds, the fp32 -> bf16 rounding of the ingest path, the (score, row) merge keys, and
 * the epilogue's list rule fed exactly as the kernel feeds it, in chunks of 32 consecutive values (floor_after[i], if
 * given and > -inf, is a shared bound that becomes visible at the start of the chunk holding value i); out_drop (optional)
 * receives the "dropped" bound: the largest score the list saw and does not hold. */
int sa_debug_float_keys(const float* x, int n, uint32_t* key, float* back, float* below);
int sa_debug_bf16_round(const float* x, int n, uint16_t* bits, float* back);
/* The fp32 -> int8 conversion of an int8 index (SA_ELEM_INT8): round to nearest even, saturate, NaN -> 0. */
int sa_debug_int8_round(const float* x, int n, int8_t* out);
int sa_debug_merge_keys(const float* score, const int32_t* row, int n, uint64_t* key, int32_t* row_back);
int sa_debug_list_insert(const float* score, const int32_t* row, int n, int list_len, const float* floor_after,
                         float* out_score, int32_t* out_row, float* out_drop);
/* The window bound of the scan's epilogue: for each of n_windows groups of 16 keys (16 tile lanes' second-best scores of
 * one query as order-preserving keys, 0 = not published yet) the (list_len/2)-th largest key (0 = no bound yet);
 * out_sorted (optional) receives each window sorted descending by the kernel's 16-input network. */
int sa_debug_window_bound(const uint32_t* keys, int n_windows, int list_len, uint32_t* out_bound, uint32_t* out_sorted);
/* The deep search's window bound (28 < k <= 64): for each group of 16 keys (16 tile lanes' 5th-best scores of one query,
 * 0 = not published yet) the 14th largest key -- 70 rows in all (0 = no bound yet). */
int sa_debug_window_bound_deep(const uint32_t* keys, int n_windows, uint32_t* out_bound);
/* The filter predicate (sa_filter) exactly as the scan and the fallback scan evaluate it: out[i] = pass(tags[i], *f). */
int sa_debug_filter_pass(const uint64_t* tags, int n, const sa_filter* f, uint8_t* out);

/* Pinned host memory for callers that want truly asynchronous staging. */
int sa_host_alloc(void** out, uint64_t bytes);
int sa_host_free(void* p);

#ifdef __cplusplus
}
#endif
#endif /* SA_API_H_ */
