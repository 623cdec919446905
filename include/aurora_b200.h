/*
 * aurora_b200.h -- C ABI of the H100-native retrieval engine behind Aurora's
 * knowledge-base RAG path.
 *
 * The reference (Arvo-AI/aurora) has no FFI for this path: its boundary is the Python
 * module server/routes/knowledge_base/weaviate_client.py, which forwards every call
 * over gRPC to a Weaviate 1.27.6 server (vector index) and, through it, to the
 * t2v-transformers container (text -> vector).  This header is what a ctypes binding in
 * that module binds instead (see INTEGRATION.md); each entry point cites the reference
 * interface it replaces.  Plain pointers and sizes only; no torch / CUDA types.
 *
 * Conventions
 *   - every function returns AUR_OK (0) or a negative aur_status; on failure no output
 *     buffer has been written and aur_last_error() (thread-local) describes why;
 *   - "host" entry points take host pointers and include the H2D / D2H copies;
 *     "_dev" entry points take device pointers on the index's device and a cudaStream_t
 *     passed as void* (NULL = the index's own stream; pass cudaStreamLegacy, (void*)1, for
 *     the legacy default stream) and do not synchronise;
 *   - vectors are row-major [n, dim]; dtype is fixed per index (AUR_BF16: raw uint16
 *     bfloat16 bits; AUR_F32: IEEE float);
 *   - ids are caller-chosen int64 (>= 0), unique per index; adding an existing id
 *     replaces the old row (reference: deterministic uuid5 upsert,
 *     weaviate_client.py:172);
 *   - scores are cosine similarity (= 1 - Weaviate cosine distance, cf.
 *     server/routes/incident_feedback/weaviate_client.py:296-297), NOT clamped;
 *     results are ordered (score desc, id asc); missing results are padded with
 *     id -1 / score -INFINITY;
 *   - all entry points are thread-safe and never touch the Python GIL.  The shard is append-only
 *     with a published row count: a search scans exactly the rows that were published when it was
 *     enqueued (a consistent prefix) and never waits for a writer; several searches may be in
 *     flight at once, each with its own scratch (see aur_search_ex); writers are serialised among
 *     themselves; aur_compact / aur_export are exclusive.
 */
#ifndef AURORA_B200_H_
#define AURORA_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AUR_ABI_VERSION 3

typedef enum aur_status {
  AUR_OK = 0,
  AUR_ERR_INVALID = -1,     /* bad argument                                   */
  AUR_ERR_CUDA = -2,        /* CUDA runtime / driver error                    */
  AUR_ERR_NOMEM = -3,       /* capacity exceeded or allocation failure        */
  AUR_ERR_UNSUPPORTED = -4, /* shape / dtype not supported by the chosen path */
  AUR_ERR_NO_DEVICE = -5    /* no CUDA device (the library has no CPU path)   */
} aur_status;

typedef enum aur_dtype { AUR_BF16 = 0, AUR_F32 = 1 } aur_dtype;

/* Which similarity kernel serves a search (aur_set_option "kernel"). */
typedef enum aur_kernel {
  AUR_KERNEL_AUTO = 0,   /* tensor-core path when the shape allows it, else SIMT      */
  AUR_KERNEL_SIMT = 1,   /* generic CUDA-core path (any dim / dtype / filter)     */
  AUR_KERNEL_TC1 = 2,    /* wgmma, single CTAs                                    */
  AUR_KERNEL_TC2 = 3,    /* wgmma, two-CTA clusters sharing tiles by TMA multicast */
  AUR_KERNEL_LIST = 4    /* per-query list gather (aur_search_lists only; not an option value) */
} aur_kernel;

typedef struct aur_index aur_index; /* opaque: one corpus shard resident on one GPU */

typedef struct aur_config {
  int32_t device;     /* CUDA ordinal                                               */
  int32_t dim;        /* vector dimension                                           */
  int32_t dtype;      /* aur_dtype                                                  */
  int32_t reserved;
  int64_t capacity;   /* rows of HBM to reserve for this shard (grow = reopen)      */
} aur_config;

typedef struct aur_stats {
  int64_t rows;          /* rows ever appended (including tombstones)               */
  int64_t live;          /* rows visible to search                                  */
  int64_t capacity;
  int32_t dim, dtype;
  int32_t last_kernel;   /* aur_kernel actually used by the last search             */
  int32_t last_launches; /* kernels launched by the last search                     */
  float   last_kernel_ms;/* device time of the dominant kernel of the last search   */
  float   last_total_ms; /* device time of the whole last search                    */
  float   last_finalize_ms; /* from the end of the (first) similarity kernel to the end of the last exact
                               re-rank kernel (for nq > 256 this spans the later query blocks too)         */
  float   last_merge_ms; /* aur_search_exchange_dev: delivery wait + cross-shard merge; else ~0           */
  int64_t last_candidates;     /* candidate keys the last search's exact re-rank read, summed over its queries */
  int32_t last_candidates_max; /* the most any one query of the last search carried into the re-rank          */
  int32_t last_tile_n;   /* corpus rows per tile of the last search's tensor-core kernel (64, 128; 0: none) */
} aur_stats;

int aur_abi_version(void);
const char* aur_last_error(void);
int aur_device_count(void);

/* Lifecycle.  Replaces weaviate.connect_to_local / _ensure_collection
 * (weaviate_client.py:35-133): the "collection" is this shard. */
int aur_open(const aur_config* cfg, aur_index** out);
int aur_close(aur_index* ix);
int aur_get_stats(aur_index* ix, aur_stats* out);
/* Options: "kernel" (aur_kernel), "tc_tile" (corpus rows per tensor-core tile: 0 = auto, 64 or 128;
 * a search the 128-row layout does not fit fails); bring-up only: "dbg_flags", and "dbg_epoch" (1 .. 2^31 - 1), which
 * sets the tensor-core kernel's launch counter of every search context of the index, e.g. just before it wraps. */
int aur_set_option(aur_index* ix, const char* key, int64_t value);
int aur_sync(aur_index* ix);

/* Ingest.  Replaces collection.batch.dynamic()/add_object (weaviate_client.py:167-186)
 * for already-embedded chunks: appends n rows, computes their inverse L2 norms on the
 * device (Weaviate normalises at import for cosine).  user_codes / org_codes carry the
 * tenant scope used by weaviate_client.py:244-249 as int32 codes (org -1 = none); both
 * may be NULL (all rows get user 0, org -1). */
int aur_add(aur_index* ix, const void* rows_host, const int64_t* ids,
            const int32_t* user_codes, const int32_t* org_codes, int64_t n);
int aur_add_dev(aur_index* ix, const void* rows_dev, const int64_t* ids_host,
                const int32_t* user_codes_host, const int32_t* org_codes_host,
                int64_t n, void* stream);

/* Snapshot.  Replaces the Weaviate data volume (docker-compose.yaml:477-478) as the durable copy of
 * the shard: copies all n = aur_stats.rows appended rows (tombstones included, live_out[i] = 0 for
 * them) back to the host in append order.  Restore = aur_open + aur_add of the live rows, which also
 * compacts the tombstones away.  user_out / org_out may be NULL. */
int aur_export(aur_index* ix, void* rows_out, int64_t* ids_out, int32_t* user_out,
               int32_t* org_out, uint8_t* live_out, int64_t n);

/* Reads back rows [row0, row0 + n) of the published prefix (append order, tombstones included) with their ids:
 * a partial aur_export, e.g. to snapshot only what was appended since the last snapshot. */
int aur_read_rows(aur_index* ix, int64_t row0, int64_t n, void* rows_out, int64_t* ids_out);

/* Reclaims the tombstones left by upserts and deletes (the reference's prediscovery job deletes and
 * re-inserts its chunks periodically, weaviate_client.py:374-394): live rows move down in append order,
 * aur_stats.rows drops to aur_stats.live.  Exclusive: waits for in-flight searches.  *reclaimed
 * (nullable) receives the number of rows freed. */
int aur_compact(aur_index* ix, int64_t* reclaimed);

/* Deletes.  Replaces collection.data.delete_many(where=...) (weaviate_client.py:309,
 * :336, :387): the Python layer resolves the filter to ids; rows become tombstones.
 * *removed receives how many ids were live. */
int aur_remove(aur_index* ix, const int64_t* ids, int64_t n, int64_t* removed);

/* Search.  Replaces the dense leg of collection.query.hybrid (weaviate_client.py:252-259)
 * and collection.query.near_text (incident_feedback/weaviate_client.py:286-291), batched:
 * nq queries at once, top-k each.  q_user / q_org: per-query tenant codes (NULL q_user =
 * unfiltered; q_org may be NULL or hold -1 for "no org").  When every query of the batch
 * carries the same scope (the reference's call pattern) the tensor-core kernel serves it;
 * a batch with up to 32 distinct scopes rides on the same kernel through per-row bit masks,
 * more fall back to the generic kernel.
 * scores_out [nq*k] float, ids_out [nq*k] int64.  When both are page-locked (cudaHostAlloc /
 * cudaHostRegister / torch pin_memory) the results are written into them by the device itself,
 * without device-to-host copies; pageable buffers work the same, one staging copy slower. */
int aur_search(aur_index* ix, const void* queries_host, int32_t nq, int32_t k,
               const int32_t* q_user, const int32_t* q_org,
               float* scores_out, int64_t* ids_out);
/* Same call, additionally reporting the snapshot it answered from: *snapshot_rows_out = number of
 * appended rows (tombstones included) that were visible to this search.  With a writer appending
 * concurrently (the reference: Celery ingest workers next to gunicorn search threads,
 * docker-compose.yaml:191,283-285) the answer is the top-k of exactly that prefix. */
int aur_search_ex(aur_index* ix, const void* queries_host, int32_t nq, int32_t k,
                  const int32_t* q_user, const int32_t* q_org,
                  float* scores_out, int64_t* ids_out, int64_t* snapshot_rows_out);
/* Search restricted to the rows whose ids are listed: a metadata pre-filter the Python layer has
 * resolved to ids, e.g. `org_id == o AND document_id LIKE "discovery:*"`
 * (server/chat/background/rca_prompt_builder.py:286-298) or Aurora Learn's org scope
 * (server/routes/incident_feedback/weaviate_client.py:279-291).  Weaviate pre-filters the same way
 * (allow-list, then vector search).  Unknown ids are ignored; n_allow = 0 returns only padding. */
int aur_search_subset(aur_index* ix, const void* queries_host, int32_t nq, int32_t k,
                      const int64_t* allow_ids, int64_t n_allow,
                      float* scores_out, int64_t* ids_out);
/* Search with a pre-filter per query: query q sees only the rows whose ids are in list q_list[q], list l being
 * list_ids[list_offsets[l] .. list_offsets[l + 1]).  Several queries may name the same list.  Unknown ids, tombstoned ids
 * and ids appended after the search's snapshot are ignored; an id listed twice counts once; an empty list yields padding.
 * Cost grows with the listed rows, not the shard.  bf16 indexes (any dim the index accepts); 1 <= k <= 128.
 * Many tenants' pre-filtered requests (Aurora Learn's org or user scope, incident_knowledge.py:128-133; the
 * prediscovery `org_id AND document_id LIKE "discovery:*"` filter, rca_prompt_builder.py:286-298) share one call.
 * Threading, snapshot (*snapshot_rows_out, nullable) and page-locked outputs as for aur_search_ex; aur_stats reports
 * last_kernel = AUR_KERNEL_LIST.  The "kernel" option does not apply. */
int aur_search_lists(aur_index* ix, const void* queries_host, int32_t nq, int32_t k,
                     const int64_t* list_ids, const int64_t* list_offsets, int32_t n_lists, const int32_t* q_list,
                     float* scores_out, int64_t* ids_out, int64_t* snapshot_rows_out);
/* Attribute columns and device-evaluated pre-filters.
 *
 * A shard carries up to 16 int32 attribute columns, numbered 2 .. 17 (columns 0 and 1 are the tenant user / org codes
 * of aur_add).  A column is allocated on its first aur_set_attrs with every row absent (-1); rows appended later, the new
 * row of an upsert and the rows compaction frees start absent too.  aur_set_attrs writes codes by id (unknown ids are
 * ignored) and is serialised with the other writers.  A search sees a row's codes as they were when its filter kernel read
 * them: a caller that must never answer from a row without its codes sets them before it lets searches name them.
 *
 * A filter program is a postfix sequence of tokens, 4 int32 each: {AUR_FILTER_LEAF, column, bitmap offset, bitmap length}
 * or {AUR_FILTER_AND | AUR_FILTER_OR, 0, 0, 0}.  Offsets and lengths count bits of `bitmap` (bitmap_words uint32 words,
 * bit i = word i / 32, bit i % 32).  A leaf is true for a row whose code c in that column has bit c + 1 of its slice set
 * (bit 0: absent), so the tenant scope of aur_search, row_user == u OR (o >= 0 AND row_org == o), is the program
 * [leaf(0, bit u + 1), leaf(1, bit o + 1), OR].  At most 32 leaves per program; only live rows of the search's snapshot
 * match.  Malformed programs (stack underflow, not exactly one value left, more than 32 leaves, unknown token, a column
 * out of range or never set, a slice outside the bitmap) are AUR_ERR_INVALID. */
#define AUR_FILTER_LEAF 0
#define AUR_FILTER_AND 1
#define AUR_FILTER_OR 2
int aur_set_attrs(aur_index* ix, int32_t col, const int64_t* ids, const int32_t* codes, int64_t n);
/* aur_search_lists with every list given as a filter program evaluated on the device: program p
 * (tokens prog[4 * prog_offsets[p] .. 4 * prog_offsets[p + 1]), 1 <= n_programs <= 1024) selects the rows query q searches
 * when q_program[q] = p.  The matching rows never leave the device, and no id is resolved on the host.  The programs are
 * counted first, 32 per pass over the rows, with one small read-back for all passes; a call with one program whose matching rows exceed max_list_rows runs the masked
 * full scan of aur_search_subset (aur_stats.last_kernel = the tensor-core or SIMT kernel), every other call the list kernels
 * of aur_search_lists (AUR_KERNEL_LIST).  Either way the answer is bit for bit that of the corresponding host-resolved call
 * over the matching ids.  matched_out [n_programs] (nullable) receives each program's matching rows.  bf16 indexes;
 * threading, snapshot and page-locked outputs as for aur_search_lists. */
int aur_search_filtered(aur_index* ix, const void* queries_host, int32_t nq, int32_t k, const int32_t* prog,
                        const int32_t* prog_offsets, int32_t n_programs, const uint32_t* bitmap, int64_t bitmap_words,
                        const int32_t* q_program, int64_t max_list_rows, float* scores_out, int64_t* ids_out,
                        int64_t* matched_out, int64_t* snapshot_rows_out);
/* The ids of the live rows one program (n_tokens tokens) matches, in row order: the first min(*n_out, cap) go to ids_out,
 * *n_out receives how many there are (call again with a larger cap when it exceeds cap). */
int aur_filter_ids(aur_index* ix, const int32_t* prog, int32_t n_tokens, const uint32_t* bitmap, int64_t bitmap_words,
                   int64_t* ids_out, int64_t cap, int64_t* n_out);
/* Device variant: everything in HBM; scores64_dev (nullable) additionally receives the
 * fp64 ranking keys needed for an exact cross-shard merge. */
int aur_search_dev(aur_index* ix, const void* queries_dev, int32_t nq, int32_t k,
                   const int32_t* q_user_dev, const int32_t* q_org_dev,
                   float* scores_dev, int64_t* ids_dev, double* scores64_dev,
                   void* stream);

/* Cross-shard merge (row-sharded corpus over <= 8 GPUs): after an all-gather of each
 * shard's (fp64 score, id) top-k, keep the best k per query on the device.
 * in_scores64 / in_ids: [n_shards, nq, k]; out: [nq, k]. */
int aur_merge_topk_dev(int32_t device, const double* in_scores64, const int64_t* in_ids,
                       int32_t n_shards, int32_t nq, int32_t k,
                       float* out_scores, int64_t* out_ids, double* out_scores64,
                       void* stream);

/* Same merge over ONE gathered buffer: each shard contributes a block of 2*nq*k 8-byte words, plane 0
 * its fp64 scores [nq,k], plane 1 its int64 ids [nq,k] (pass scores64_dev = block, ids_dev = block +
 * nq*k to aur_search_dev), so the exchange is a single all-gather.  packed: [n_shards][2][nq][k]. */
int aur_merge_topk_packed_dev(int32_t device, const void* packed, int32_t n_shards, int32_t nq,
                              int32_t k, float* out_scores, int64_t* out_ids,
                              double* out_scores64, void* stream);

/* Host-side k-way merge of per-shard lists for a single owner process that holds one shard per GPU (each shard
 * answered through aur_search from its own host thread): scores / ids are [n_lists][nq][k_in], each list sorted by
 * (score desc, id asc) with id < 0 padding at its end; out is [nq][k_out] in the same order.  n_lists <= 64.
 * Stands in for the coordinator-side merge of a multi-shard Weaviate class (weaviate_client.py:252-259 call site). */
int aur_merge_topk_host(const float* scores, const int64_t* ids, int32_t n_lists, int32_t nq, int32_t k_in,
                        int32_t k_out, float* out_scores, int64_t* out_ids);
/* The same merge on fp64 scores (the keyword stores' exact BM25 scores, aur_kw_search_multi); padding -INFINITY / -1. */
int aur_merge_topk_host_f64(const double* scores, const int64_t* ids, int32_t n_lists, int32_t nq, int32_t k_in,
                            int32_t k_out, double* out_scores, int64_t* out_ids);

/* Fused exchange (SURVEY.md 2c C1, "fused variant"): instead of a local top-k array + ncclAllGather + merge, the
 * kernel that produces a shard's exact top-k stores it straight into EVERY rank's exchange buffer over NVLink
 * (peer-mapped through CUDA IPC) as 8-byte words that each carry 4 bytes of payload and a 4-byte sequence tag, and the
 * merge kernel that follows polls those words until the tags match -- no flag, fence or collective on the path.  One
 * process per GPU:
 *   1. every rank:  aur_exchange_create(...)      -> its 64-byte IPC handle
 *   2. all-gather the handles (any host transport: torch.distributed, MPI, a file)
 *   3. every rank:  aur_exchange_connect(ex, all_handles)
 *   4. per batch, every rank, in lock step: aur_search_exchange_dev(ix, ex, queries, ...) -- on return of the
 *      stream's work scores_dev / ids_dev hold the GLOBAL top-k on every rank (ids must be globally unique).
 * All ranks must call step 4 the same number of times; barrier before aur_exchange_close. */
typedef struct aur_exchange aur_exchange;
int aur_exchange_create(int32_t device, int32_t rank, int32_t world, int32_t nq_max, int32_t k_max,
                        aur_exchange** out, uint8_t* handle_out /* [64] */);
int aur_exchange_connect(aur_exchange* ex, const uint8_t* all_handles /* [world][64] */);
int aur_exchange_close(aur_exchange* ex);
/* exchanges completed on this rank; *status != 0: a peer did not deliver within the kernel's time-out */
int aur_exchange_status(aur_exchange* ex, int64_t* exchanges_done, int32_t* status);
int aur_search_exchange_dev(aur_index* ix, aur_exchange* ex, const void* queries_dev, int32_t nq,
                            int32_t k, float* scores_dev, int64_t* ids_dev, void* stream);

/* Pairwise cosine of row i of a with row i of b (host buffers, fp32 in, fp64 out).
 * Replaces SimilarityStrategy._cosine_similarity
 * (server/services/correlation/strategies/similarity.py:84-98); clamp != 0 applies its
 * [0,1] clamp (:98). */
int aur_cosine_pairs(int32_t device, const float* a_host, const float* b_host,
                     int64_t n, int32_t dim, int32_t clamp, double* out_host);

/* Raw device buffers for callers without a CUDA runtime of their own (ctypes tests, the
 * benchmark's host-side staging).  Synchronous. */
int aur_dev_malloc(int32_t device, uint64_t bytes, void** out);
int aur_dev_free(int32_t device, void* p);
int aur_memcpy_h2d(int32_t device, void* dst_dev, const void* src_host, uint64_t bytes);
int aur_memcpy_d2h(int32_t device, void* dst_host, const void* src_dev, uint64_t bytes);

/* ------------------------------------------------------------------ BM25 keyword store
 * Replaces the BM25 leg of collection.query.hybrid (weaviate_client.py:252-259), which Weaviate runs on its own host
 * cores next to the vector leg.  A standalone store on one GPU, keyed by the same caller ids and tenant codes as an
 * aur_index: a forward index of (term id, tf) postings per document, term ids chosen by the caller (aurora_b200.bm25
 * keeps the vocabulary).  Scores are bm25.BM25Index.search's loop path bit for bit: k1 = 1.2, b = 0.75,
 * idf = log(1 + (N - df + 0.5) / (df + 0.5)), avgdl = total_len / N (1 when total_len is 0), N / df / total_len over
 * every live document of the store, a document's score summed in the order its query lists the terms, fp64.  Results are
 * ordered (score desc, id asc), only documents with a matching term appear, padding is id -1 / score -INFINITY.
 * Append-only with a published prefix like aur_index; a search scores exactly the prefix whose statistics it took
 * (*snapshot_rows_out).  Upserts of existing ids, removes, posting growth and compaction wait for searches in flight. */
typedef struct aur_kw aur_kw;

typedef struct aur_kw_stats {
  int64_t docs;               /* rows ever appended (including tombstones)          */
  int64_t live;               /* documents visible to search (N)                    */
  int64_t capacity;           /* document rows reserved at open                     */
  int64_t postings_used;      /* postings of the appended rows                      */
  int64_t postings_allocated; /* posting slots in HBM (grows on demand)             */
  int64_t total_len;          /* tokens over the live documents                     */
  int32_t last_launches;      /* kernels launched by the last search                */
  float   last_ms;            /* device time of the last search (uploads included)  */
  int32_t last_terms;         /* most distinct live terms one launch of it scored   */
  int32_t last_spilled;       /* its launches whose per-warp term table did not fit shared
                                 memory and lived in global memory instead          */
} aur_kw_stats;

/* Lifecycle; the keyword half of _ensure_collection (weaviate_client.py:35-133).  postings_capacity 0 = 2^20 to start
 * with.  Without a device: AUR_ERR_NO_DEVICE. */
int aur_kw_open(int32_t device, int64_t doc_capacity, int64_t postings_capacity, aur_kw** out);
int aur_kw_close(aur_kw* kw);
/* Upsert n documents (the text side of add_object, weaviate_client.py:167-186): document i has postings
 * [offsets[i], offsets[i + 1]) of term_ids / tfs, term ids strictly increasing (0 .. 2^28 - 1), tf >= 1; an existing id
 * loses its old row (weaviate_client.py:172).  user_codes / org_codes as for aur_add (NULL: user 0, org -1). */
int aur_kw_add(aur_kw* kw, const int64_t* ids, const int32_t* user_codes, const int32_t* org_codes,
               const int32_t* term_ids, const int32_t* tfs, const int64_t* offsets, int64_t n);
/* Deletes (collection.data.delete_many, weaviate_client.py:309): *removed (nullable) = ids that were live. */
int aur_kw_remove(aur_kw* kw, const int64_t* ids, int64_t n, int64_t* removed);
/* Stable compaction of the tombstones, as aur_compact; *reclaimed (nullable) = rows freed. */
int aur_kw_compact(aur_kw* kw, int64_t* reclaimed);
int aur_kw_get_stats(aur_kw* kw, aur_kw_stats* out);
/* The BM25 leg of collection.query.hybrid (weaviate_client.py:252-259), batched: query q's term ids are
 * q_terms[q_offsets[q] .. q_offsets[q + 1]) in summation order (repeats and unknown ids are ignored); top-k each,
 * 1 <= k <= 128 (larger: AUR_ERR_UNSUPPORTED).  q_user / q_org: per-query tenant scope as in aur_search
 * (weaviate_client.py:244-249; NULL q_user = unscoped).  allow_ids (n_allow of them) restrict every query of the batch to
 * those documents, as aur_search_subset; NULL = no restriction, n_allow = 0 with a non-NULL pointer = nothing.
 * scores_out / ids_out [nq * k]; *snapshot_rows_out (nullable) = appended rows the search saw. */
int aur_kw_search(aur_kw* kw, const int32_t* q_terms, const int64_t* q_offsets, int32_t nq, int32_t k,
                  const int32_t* q_user, const int32_t* q_org, const int64_t* allow_ids, int64_t n_allow,
                  double* scores_out, int64_t* ids_out, int64_t* snapshot_rows_out);
/* aur_kw_search over n_stores (1 .. 64) stores taken as ONE corpus, e.g. one store per GPU of the host with documents
 * placed by id mod n_stores; ids must be unique across the stores (the caller's placement keeps them so).  The answer
 * equals aur_kw_search on a single store holding the union of every store's snapshot prefix: ids exact, fp64 scores
 * bit-identical, padding (-1, -INFINITY).  N, df and total_len are summed over the stores' snapshots and idf / avgdl
 * computed once from the sums; every store scores its own prefix on its own device with them, all stores at once, and
 * the per-store lists are merged on the host by (score desc, id asc).  Every store's shared lock is held for the whole
 * call, taken in address order.  q_user / q_org / allow_ids as for aur_kw_search (each store resolves allow_ids against
 * its own documents).  snapshot_rows_out [n_stores] (nullable): the prefix store s scanned; each store's
 * aur_kw_stats.last_* describe its part of the search.  NULL entries and a store listed twice: AUR_ERR_INVALID. */
int aur_kw_search_multi(aur_kw* const* stores, int32_t n_stores, const int32_t* q_terms, const int64_t* q_offsets,
                        int32_t nq, int32_t k, const int32_t* q_user, const int32_t* q_org, const int64_t* allow_ids,
                        int64_t n_allow, double* scores_out, int64_t* ids_out, int64_t* snapshot_rows_out);

/* ------------------------------------------------------------------ hybrid query
 * collection.query.hybrid (weaviate_client.py:252-259) in one call: the dense leg (aur_search_ex of queries_host over
 * ix, top-fetch cosines) and the keyword leg (aur_kw_search of q_terms / q_offsets over kw, top-fetch BM25 scores) run
 * on the GPU, both enqueued before either is waited on, with the same per-query tenant scope q_user / q_org (as in
 * aur_search; NULL = unscoped); each leg's answer is the one those calls give for the snapshot it reports.  A kernel
 * then fuses query q's two lists with weights w_dense[q] / w_sparse[q] (finite; a leg whose weight is <= 0 takes no
 * part, so with w_dense <= 0 the dense leg is searched but ignored) and one copy returns the best k_out entries by
 * (fused score desc, id asc):
 *   AUR_FUSION_RANKED          Weaviate's rankedFusion: an entry at 0-based rank r of a leg adds w / (r + 60);
 *   AUR_FUSION_RELATIVE_SCORE  relativeScoreFusion: an entry with score s adds w * (s - lo) / (hi - lo), lo / hi the
 *                              min / max score of its leg's list (w when hi == lo), cosines taken as fp64;
 * summed in fp64 from 0.0, dense part first -- bit for bit aurora_b200.bm25.ranked_fusion / relative_score_fusion.
 * scores_out [nq * k_out] fp64 fused scores, ids_out [nq * k_out], cosine_out [nq * k_out] the dense leg's fp32 cosine
 * of the id (NaN when the id is not in the dense list); padding (-INFINITY, -1, NaN).  snapshot_rows_out [2] (nullable):
 * the prefix the dense and the keyword leg saw.  1 <= fetch <= 128, 1 <= k_out <= 2 * fetch; a bf16 index and a
 * keyword store on its device (else AUR_ERR_UNSUPPORTED / AUR_ERR_INVALID).  aur_stats.last_* and aur_kw_stats.last_*
 * describe the two legs. */
#define AUR_FUSION_RANKED 0
#define AUR_FUSION_RELATIVE_SCORE 1
int aur_hybrid_search(aur_index* ix, aur_kw* kw, const void* queries_host, int32_t nq, int32_t fetch,
                      const int32_t* q_terms, const int64_t* q_offsets, const int32_t* q_user, const int32_t* q_org,
                      const double* w_dense, const double* w_sparse, int32_t fusion, int32_t k_out,
                      double* scores_out, int64_t* ids_out, float* cosine_out, int64_t* snapshot_rows_out);
/* aur_hybrid_search over n (1 .. 64) vector shards and n keyword stores taken as one corpus, e.g. one shard and one store
 * per GPU of the host with documents placed by id mod n (engine.MultiIndex + engine.MultiKeywordIndex); shard s and
 * store s must be on the same device, shards bf16, ids unique across the shards.  Every shard's dense leg and every
 * store's keyword leg (the stores scored with corpus-wide statistics, as aur_kw_search_multi) run on their own devices,
 * all enqueued before any is waited on; the lists of shards 1 .. n-1 are copied to shard 0's device (peer copies;
 * peer access is neither required nor enabled), where one kernel merges each leg's lists into its global top-fetch and
 * fuses the two as aur_hybrid_search does.  Each leg's merged list is exactly the host merge's: aur_merge_topk_host on
 * the shards' fp32 cosines (engine.MultiIndex.search), aur_merge_topk_host_f64 on the stores' fp64 scores
 * (aur_kw_search_multi) -- best head first by (score desc, id asc, list asc), a list ending at its first id < 0.
 * snapshot_rows_out [2n] (nullable): entries 0 .. n-1 the prefix each shard's dense leg saw, n .. 2n-1 the prefix each
 * store's keyword leg saw.  Each shard's aur_stats.last_* and each store's aur_kw_stats.last_* describe its own part.
 * NULL entries, a shard or a store listed twice, n out of range: AUR_ERR_INVALID; an f32 shard: AUR_ERR_UNSUPPORTED; a
 * store on another device than its shard: AUR_ERR_INVALID; the other arguments as for aur_hybrid_search.  Every
 * rejection happens before any device work.  aur_hybrid_search is this call with n = 1. */
int aur_hybrid_search_multi(aur_index* const* shards, aur_kw* const* stores, int32_t n, const void* queries_host,
                            int32_t nq, int32_t fetch, const int32_t* q_terms, const int64_t* q_offsets,
                            const int32_t* q_user, const int32_t* q_org, const double* w_dense, const double* w_sparse,
                            int32_t fusion, int32_t k_out, double* scores_out, int64_t* ids_out, float* cosine_out,
                            int64_t* snapshot_rows_out /* [2n] */);

/* ------------------------------------------------------------------ text encoder
 * Replaces the text2vec-transformers sidecar: EmbeddingClient.embed / embed_batch
 * (server/services/correlation/embedding_client.py:39-78, POST {base}/vectors) and the
 * server-side vectorisation Weaviate performs on insert and on hybrid / near_text queries
 * (server/routes/knowledge_base/weaviate_client.py:113-126, :252-259).  A BERT-family encoder
 * forward (embeddings, L x [QKV GEMM, attention, out-proj + LayerNorm, FFN + LayerNorm],
 * pooling) in bf16 with fp32 accumulation.  Input is WordPiece token ids, packed:
 * tokens [total] and cu_seqlens [n_seq + 1] (sequence i = tokens[cu[i] : cu[i+1]], each
 * 1..max_pos long, [CLS] / [SEP] included by the caller). */
typedef struct aur_encoder aur_encoder;

typedef enum aur_pool { AUR_POOL_CLS = 0, AUR_POOL_MEAN = 1 } aur_pool;

typedef struct aur_encoder_config {
  int32_t device;
  int32_t hidden, layers, heads, inter;   /* head dim (hidden / heads) 64, or 32 (zero-padded) */
  int32_t vocab, max_pos, type_vocab;     /* max_pos <= 512                               */
  int32_t pool;                           /* aur_pool                                     */
  int32_t normalize;                      /* != 0: L2-normalise the pooled vector         */
  int32_t max_tokens;                     /* packed tokens per aur_encode call (workspace)*/
  int32_t max_seqs;                       /* sequences per call                           */
  float   ln_eps;
  int32_t reserved;                       /* 0; (1 = single-CTA GEMM tiles, bring-up only) */
} aur_encoder_config;

typedef struct aur_encoder_stats {
  int64_t tokens, seqs;      /* of the last call                                          */
  int32_t launches;          /* kernels launched by the last call                         */
  float   total_ms;          /* device time of the last forward (embeddings .. pooling)   */
  float   gemm_ms, attn_ms;  /* thereof: wgmma GEMMs, attention                          */
  double  gemm_flops;        /* 2*M*N*K summed over the GEMMs, M = real (unpadded) tokens  */
  double  attn_flops;        /* 4 * len^2 * hidden per sequence and layer                  */
} aur_encoder_stats;

int aur_encoder_open(const aur_encoder_config* cfg, aur_encoder** out);
int aur_encoder_close(aur_encoder* enc);
/* Upload one parameter tensor (host fp32; matrices are stored as bf16 on the device).  Names:
 * word_emb [vocab,H], pos_emb [max_pos,H], type_emb [type_vocab,H], emb_ln_g/emb_ln_b [H], and per
 * layer l: l{l}.wqkv [3H,H] (query, key, value rows stacked), l{l}.bqkv [3H], l{l}.wo [H,H],
 * l{l}.bo, l{l}.ln1_g, l{l}.ln1_b, l{l}.wi [I,H], l{l}.bi [I], l{l}.wo2 [H,I], l{l}.bo2,
 * l{l}.ln2_g, l{l}.ln2_b -- all [out_features, in_features] like torch.nn.Linear. */
int aur_encoder_load(aur_encoder* enc, const char* name, const float* data, int64_t count);
/* Host in / host out.  out_f32 [n_seq, hidden] and/or out_bf16 [n_seq, hidden] (either may be
 * NULL).  Fails with AUR_ERR_INVALID until every parameter has been loaded. */
int aur_encode(aur_encoder* enc, const int32_t* tokens, const int32_t* cu_seqlens, int32_t n_seq,
               float* out_f32, uint16_t* out_bf16);
/* Fused ingest: encode the chunks and append the pooled bf16 vectors to the shard without
 * leaving the device (insert_chunks, weaviate_client.py:136-212, minus the text handling). */
int aur_encode_append(aur_encoder* enc, aur_index* ix, const int32_t* tokens,
                      const int32_t* cu_seqlens, int32_t n_seq, const int64_t* ids,
                      const int32_t* user_codes, const int32_t* org_codes);
int aur_encoder_get_stats(aur_encoder* enc, aur_encoder_stats* out);

/* ------------------------------------------------------------------ WordPiece tokenizer
 * Text -> token ids on the host cores, multi-threaded.  In the reference this step is inside the t2v sidecar
 * (raw text is posted to it, embedding_client.py:52-59); semantics = transformers.BertTokenizer (the `tokenizers`
 * BertNormalizer + BertPreTokenizer + WordPiece): see csrc/tokenizer.cpp.  Texts travel as one UTF-8 buffer plus
 * offsets [n_texts + 1]. */
typedef struct aur_tokenizer aur_tokenizer;
int aur_tokenizer_open(const char* vocab_path, int32_t lower_case, aur_tokenizer** out);       /* vocab.txt, one piece per line */
int aur_tokenizer_open_mem(const char* vocab_utf8, int64_t nbytes, int32_t lower_case, aur_tokenizer** out);
int aur_tokenizer_close(aur_tokenizer* t);
int aur_tokenizer_info(aur_tokenizer* t, int32_t* vocab_size, int32_t* unk_id, int32_t* cls_id, int32_t* sep_id);
/* Every text -> [CLS] pieces [SEP] truncated to max_len ids, packed: tokens_out (capacity tokens_cap; n_texts * max_len
 * always suffices) and cu_seqlens_out [n_texts + 1].  n_threads 0 = all host cores.  tokens_out = NULL with
 * tokens_cap = 0 asks for the lengths only (cu_seqlens_out is filled, no ids are written). */
int aur_tokenize(aur_tokenizer* t, const char* texts_utf8, const int64_t* offsets, int32_t n_texts, int32_t max_len,
                 int32_t* tokens_out, int64_t tokens_cap, int32_t* cu_seqlens_out, int32_t n_threads);
/* Text in, rows in the shard: tokenise, encoder forward, append -- insert_chunks (weaviate_client.py:136-212) without
 * Python on the path.  Batches are cut to max_tokens_per_call / max_seqs_per_call (the encoder's workspace). */
int aur_encode_text_append(aur_encoder* enc, aur_tokenizer* tok, aur_index* ix, const char* texts_utf8,
                           const int64_t* offsets, int32_t n_texts, int32_t max_len, int32_t max_tokens_per_call,
                           int32_t max_seqs_per_call, const int64_t* ids, const int32_t* user_codes,
                           const int32_t* org_codes, int32_t n_threads);

/* Bring-up / test hooks (not part of the drop-in surface). */
/* out[M,N] = epi(A[M,K] . W[N,K]^T + bias) through the encoder's wgmma GEMM; host buffers,
 * bf16 bits; epi 0 = bias, 1 = bias + GELU, 2 = bias + resid[M,N]; cta_group 1 or 2 (CTAs per tile). */
int aur_debug_gemm(int32_t device, const uint16_t* a, const uint16_t* w, const float* bias,
                   const uint16_t* resid, int32_t m, int32_t n, int32_t k, int32_t epi,
                   int32_t cta_group, uint16_t* out, float* ms_out);
/* ctx[T,H] = self-attention over packed qkv[T,3H] (bf16 bits, host buffers). */
int aur_debug_attention(int32_t device, const uint16_t* qkv, const int32_t* cu_seqlens,
                        int32_t n_seq, int32_t heads, int32_t hidden, uint16_t* ctx,
                        float* ms_out);
/* Final hidden states [tokens, hidden] (bf16 bits) of the last aur_encode call. */
int aur_debug_encoder_hidden(aur_encoder* enc, uint16_t* out, int64_t count);
int aur_debug_tc_scores(aur_index* ix, const void* queries_dev, int32_t nq,
                        int32_t cta_group, float* out_dev /* [n_ctas,64,64] */,
                        int32_t* n_ctas_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* AURORA_B200_H_ */
