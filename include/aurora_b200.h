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
 *   - a device or page-locked allocation that fails is AUR_ERR_NOMEM, any other CUDA failure
 *     AUR_ERR_CUDA;
 *   - "host" entry points take host pointers and include the H2D / D2H copies;
 *     "_dev" entry points take device pointers on the index's device and a cudaStream_t
 *     passed as void* (NULL = the index's own stream; pass cudaStreamLegacy, (void*)1, for
 *     the legacy default stream) and do not synchronise;
 *   - vectors are row-major [n, dim]; dtype is fixed per index (AUR_BF16: raw uint16
 *     bfloat16 bits; AUR_F32: IEEE float; AUR_I8: rows are stored as int8, see aur_dtype);
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

/* AUR_I8: rows are stored as int8 [capacity, dim] (dim % 16 == 0), half the memory of bf16.  Rows and queries go in
 * as bf16 bits, as for AUR_BF16; each row is quantized on the device when it is added:
 * q = rint(x * 127 / max|x|) in fp64 (half to even), a zero row stays zero, and a row holding a NaN or +-inf is stored
 * as zeros and never returned by a search (as in a bf16 shard).  Cosine ignores the per-row scale, so scores are exact
 * cosines against the stored int8 rows.  aur_export / aur_read_rows return the int8 rows.  The tensor-core kernel
 * serves int8 shards with dim % 128 == 0 and dim <= 1024 (wgmma s8 over a two-byte query image); "tc_qregs" does not
 * apply to them. */
typedef enum aur_dtype { AUR_BF16 = 0, AUR_F32 = 1, AUR_I8 = 2 } aur_dtype;

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
  int64_t capacity;   /* rows to map in HBM when the shard opens; aur_reserve grows it */
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
 * a search the 128-row layout does not fit fails), "tc_stages" (cap on the tensor-core kernel's TMA ring: 0 = the
 * deepest that fits, 2 .. 12), "tc_qregs" (query k-blocks a 128-row launch holds in registers: -1 = auto, 0 = none, or
 * the depth the library is built with where dim / 64 reaches it); bring-up only: "dbg_flags", and "dbg_epoch" (1 .. 2^31 - 1), which
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
 * compacts the tombstones away.  user_out / org_out may be NULL.  AUR_I8: live_out[i] = 2 for a live row stored from a
 * row holding a NaN or +-inf (zeros that no search returns); a restore re-adds it as a row holding a NaN. */
int aur_export(aur_index* ix, void* rows_out, int64_t* ids_out, int32_t* user_out,
               int32_t* org_out, uint8_t* live_out, int64_t n);

/* Reads back rows [row0, row0 + n) of the published prefix (append order, tombstones included) with their ids:
 * a partial aur_export, e.g. to snapshot only what was appended since the last snapshot. */
int aur_read_rows(aur_index* ix, int64_t row0, int64_t n, void* rows_out, int64_t* ids_out);

/* Incremental snapshots.  Published rows never change, a delete only tombstones a row, and growth moves nothing, so a
 * snapshot needs only the rows appended since the last one plus one liveness bit per row; aur_compact is the only call
 * that renumbers rows.
 *
 * aur_live_bits: under the shard's shared lock and its writers' lock (ordered after every aur_add / aur_remove that has
 * returned; searches go on), *rows_out = aur_stats.rows and one kernel on the low-priority ingest stream packs rows
 * [0, rows) into words: bit r % 32 of live_out[r / 32] = row r is live (its inverse norm is not NaN), of
 * nonfinite_out[r / 32] = aur_export would report it live = 2 (AUR_I8 only; zero words for bf16 and f32, where
 * nonfinite_out may be NULL).  Bits past rows are 0.  One copy back and a wait for that stream; no device-wide sync.
 * *compactions_out (nullable) = aur_compact calls over the shard's life: rows kept their numbers between two captures
 * with the same count.  words < ceil(rows / 32): AUR_ERR_INVALID before anything is launched.
 *
 * aur_export_rows: rows [row0, row0 + n) of the published prefix (tombstones included) with their ids and tenant codes
 * (user_out / org_out nullable), as aur_export gives them, but under the shared lock only: searches and appends go on.
 * The copy runs on the ingest stream through page-locked staging in bounded chunks.  A range outside the published
 * prefix: AUR_ERR_INVALID, as in aur_read_rows. */
int aur_live_bits(aur_index* ix, uint32_t* live_out, uint32_t* nonfinite_out, int64_t words, int64_t* rows_out,
                  int64_t* compactions_out);
int aur_export_rows(aur_index* ix, int64_t row0, int64_t n, void* rows_out, int64_t* ids_out, int32_t* user_out,
                    int32_t* org_out);

/* Reclaims the tombstones left by upserts and deletes (the reference's prediscovery job deletes and
 * re-inserts its chunks periodically, weaviate_client.py:374-394): live rows move down in append order,
 * aur_stats.rows drops to aur_stats.live.  Exclusive: waits for in-flight searches.  *reclaimed
 * (nullable) receives the number of rows freed. */
int aur_compact(aur_index* ix, int64_t* reclaimed);

/* Grows the shard to at least `capacity` rows, in place.  Existing rows, ids, tenant codes, attribute codes and
 * tombstones stay where they are.  No device pointer of the shard changes, and neither a search in flight nor a
 * captured CUDA graph is affected.  New rows start absent in every attribute column.
 *   capacity <= current: AUR_OK, nothing done.
 *   > 0x7FFFFFC0 (the int32 row limit aur_open enforces), or null: AUR_ERR_INVALID.
 *   Out of device memory: AUR_ERR_NOMEM, and the shard is unchanged and still serving.
 * Every per-row array of a shard lives on a CUDA virtual-memory mapping whose address range, reserved at aur_open,
 * could hold as many rows as the device's memory; growth maps more physical memory at its end.  Serialised with the
 * writers; searches go on meanwhile.  aur_stats.capacity reports the new value.  aur_add still fails when full. */
int aur_reserve(aur_index* ix, int64_t capacity);

/* Deletes by id: the rows of the live ids among ids[0, n) become tombstones (one upload of their rows, one kernel
 * launch).  *removed receives how many ids were live.  aur_remove_filtered deletes by filter without naming ids. */
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
 * docker-compose.yaml:191,283-285) the answer is the top-k of exactly that prefix.
 * A search whose context cannot grow its scratch fails with AUR_ERR_NOMEM, as does every other call on a shard that
 * runs out of device memory (aur_search_dev, aur_remove, the filter calls and the debug dumps included); earlier
 * releases reported these allocation failures as AUR_ERR_CUDA. */
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
/* The number of live rows one program matches in the published prefix: the count pass of aur_filter_ids alone, no row
 * or id leaves the device.  Replaces collection.aggregate.over_all(filters=...) (weaviate_client.py:366). */
int aur_filter_count(aur_index* ix, const int32_t* prog, int32_t n_tokens, const uint32_t* bitmap, int64_t bitmap_words,
                     int64_t* n_out);
/* Deletes by filter.  Replaces collection.data.delete_many(where=...) (weaviate_client.py:309, :336, :387): every live
 * row one program matches becomes a tombstone (one kernel launch over the matching rows), its id leaves the shard, and
 * the removed ids go to ids_out in row order; *n_out receives how many.  Holds the writer lock throughout, as aur_remove
 * does, so the rows removed are exactly the rows published when the call began that matched.  When there are more than
 * cap, nothing is removed and *n_out receives how many there are: call again with a larger cap.  A malformed program or
 * an attribute column never set is rejected (AUR_ERR_INVALID) with nothing removed and the outputs untouched. */
int aur_remove_filtered(aur_index* ix, const int32_t* prog, int32_t n_tokens, const uint32_t* bitmap, int64_t bitmap_words,
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
  int64_t capacity;           /* document rows reserved (at open, then aur_kw_reserve) */
  int64_t postings_used;      /* postings of the appended rows                      */
  int64_t postings_allocated; /* posting slots in HBM (grows on demand)             */
  int64_t total_len;          /* tokens over the live documents                     */
  int32_t last_launches;      /* kernels launched by the last search                */
  float   last_ms;            /* device time of the last search (uploads included)  */
  int32_t last_terms;         /* most distinct live terms one launch of it scored   */
  int32_t last_spilled;       /* its launches whose per-warp term table did not fit shared
                                 memory and lived in global memory instead          */
} aur_kw_stats;

/* Lifecycle; the keyword half of _ensure_collection (weaviate_client.py:35-133).  doc_capacity: document rows to start
 * with (aur_kw_reserve grows them); postings_capacity 0 = 2^20 to start with.  Without a device: AUR_ERR_NO_DEVICE. */
int aur_kw_open(int32_t device, int64_t doc_capacity, int64_t postings_capacity, aur_kw** out);
int aur_kw_close(aur_kw* kw);
/* aur_reserve's contract, for documents: grows the store to at least doc_capacity documents.  Its per-document arrays
 * are copied into larger ones under the exclusive lock, as posting growth is, so it waits for searches in flight; rows,
 * postings, the term-major index and the BM25 statistics are unchanged.  aur_kw_add still fails when full. */
int aur_kw_reserve(aur_kw* kw, int64_t doc_capacity);
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
/* Attribute columns of the keyword store, exactly as aur_set_attrs for an aur_index: columns 2 .. 17 (0 and 1 are the
 * store's user / org codes of aur_kw_add), allocated on first use at the store's capacity with every row absent (-1);
 * codes are written by id (unknown ids are ignored); rows appended later, the new row of an upsert and the rows compaction
 * frees start absent, and compaction carries every row's codes with it.  Serialised with the store's other writers.  A
 * search sees a row's codes as they were when its filter kernel read them: a caller that must never answer from a row
 * without its codes sets them before it lets searches name them.  Read by aur_hybrid_search_filtered's programs. */
int aur_kw_set_attrs(aur_kw* kw, int32_t col, const int64_t* ids, const int32_t* codes, int64_t n);
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

/* Term-major index (DESIGN.md section 10): besides its forward postings, a store holds an index of its first R rows
 * (the indexed prefix), every term's (row, tf) list, from which a search reads only its own terms' postings; rows
 * [R, rows) are scanned forward.  Answers are bit-identical whichever way a row is scored.  The index is built on the
 * store's stream by aur_kw_reindex, by aur_kw_add once the unindexed rows hold more than 1/8 of the indexed postings
 * (a build that fails there leaves the previous index in place; the add still succeeds), and by aur_kw_compact.  A
 * build runs beside searches and waits for those in flight before it is published; it takes 8 B per indexed posting
 * plus 8 B per term id, twice that while the old index is still held. */
typedef struct aur_kw_index_stats {
  int64_t indexed_rows;       /* R                                                   */
  int64_t index_postings;     /* postings in the index (those of rows [0, R))        */
  int64_t index_bytes;        /* HBM the index holds                                 */
  int64_t builds;             /* builds published since open                         */
  float   last_build_ms;      /* host time of the last one, device work included     */
  int32_t last_path;          /* the last search's AUR_KW_PATH_* bits (0: it scored nothing) */
  int64_t last_postings;      /* postings the last search read: its terms' lists in the index, every posting of
                                 the rows it scanned forward                         */
} aur_kw_index_stats;
#define AUR_KW_PATH_FORWARD 1  /* some rows scanned forward */
#define AUR_KW_PATH_INDEX 2    /* some rows scored from the index */
/* Index every appended row now (the writers' serialisation is held while it builds). */
int aur_kw_reindex(aur_kw* kw);
/* "kw_path": 0 auto (the cost rule picks per launch), 1 forward scan only, 2 the index wherever it can serve (a launch
 * whose queries have more than 64 terms is still scanned forward).  For tests and A/B runs: answers do not change.
 * Unknown names and values: AUR_ERR_INVALID. */
int aur_kw_set_option(aur_kw* kw, const char* name, int64_t value);
int aur_kw_get_index_stats(aur_kw* kw, aur_kw_index_stats* out);

/* Reads back the forward rows [row0, row0 + n) of the published prefix (append order, tombstones included), the keyword
 * counterpart of aur_read_rows: ids_out [n] (nullable), offsets_out [n + 1] from 0, and row i's postings
 * term_ids_out / tfs_out [offsets_out[i] .. offsets_out[i + 1]) (term id ascending).  *postings_out = the rows'
 * postings; when term_ids_out or tfs_out is NULL or cap is smaller, only ids and offsets are written (count mode). */
int aur_kw_read_rows(aur_kw* kw, int64_t row0, int64_t n, int64_t* ids_out, int64_t* offsets_out, int32_t* term_ids_out,
                     int32_t* tfs_out, int64_t cap, int64_t* postings_out);

/* Keyword analysis on the device (DESIGN.md section 10, "Text analysis"): the vocabulary (word -> term id, grow-only,
 * at most 2^28 words) lives in HBM on one device, and aur_kw_add_text turns UTF-8 text into keyword-store rows there.
 * Words are Python's re.findall(r"[0-9a-z]+", text.lower()) on the bytes: ASCII letters (lowered) and digits are word
 * characters, E2 84 AA (U+212A KELVIN SIGN) is "k" inside a word, C4 B0 (U+0130) is "i" followed by a break, every
 * other byte (NUL, other non-ASCII, stray or truncated sequences) is a break.  A word the vocabulary has never seen gets
 * the next free id in order of its first occurrence in the batch (document order, then position); each document's row
 * lists (term id ascending, tf).  For the same texts in the same order the ids and rows equal bm25.build_csr's. */
typedef struct aur_kw_vocab aur_kw_vocab;
/* Without a device: AUR_ERR_NO_DEVICE. */
int aur_kw_vocab_open(int32_t device, aur_kw_vocab** out);
int aur_kw_vocab_close(aur_kw_vocab* v);
/* words (nullable) = words held, bytes (nullable) = their bytes. */
int aur_kw_vocab_size(aur_kw_vocab* v, int64_t* words, int64_t* bytes);
/* The words with ids [id0, id0 + n), concatenated into bytes_out, word i at [offsets_out[i], offsets_out[i + 1]) (from
 * 0).  bytes_out NULL: only the offsets are written (count mode, as aur_tokenize); bytes_cap too small: AUR_ERR_INVALID
 * and nothing is written. */
int aur_kw_vocab_read(aur_kw_vocab* v, int64_t id0, int64_t n, char* bytes_out, int64_t bytes_cap, int64_t* offsets_out);
/* "hash_bits" (1 .. 64, default 64): a test hook that truncates the word hash to that many bits so that distinct words
 * collide; equality is always decided on the bytes, so results do not change.  Only on an empty vocabulary.  Unknown
 * names and values: AUR_ERR_INVALID. */
int aur_kw_vocab_set_option(aur_kw_vocab* v, const char* name, int64_t value);
/* aur_kw_add of n texts analysed on v's device: document i (bytes texts_utf8[text_offsets[i] .. text_offsets[i + 1]),
 * text_offsets[0] = 0)
 * goes to store ids[i] mod n_stores, as engine.MultiKeywordIndex places it, an id repeated in the batch keeps its last
 * occurrence, user_codes / org_codes as for aur_kw_add.  Stores may live on other devices than v; their rows are
 * peer-copied (cudaMemcpyPeerAsync; peer access is neither required nor enabled).  The argument checks, every store's
 * capacity and the 2^28 word limit are checked before anything is written: such a failure leaves the stores and the
 * vocabulary unchanged.  A later failure (out of memory growing the postings, say) may leave new words in the
 * vocabulary, as bm25.build_csr does, but never a partial row in a store.  Batches larger than 64 MB of text are
 * analysed in slices of whole documents, each published before the next: the word limit of a later slice is checked
 * when it is reached.  Writers serialise as for aur_kw_add: every store's writer lock in address order, then the
 * vocabulary's.  NULL or repeated stores and n_stores outside 1 .. 64: AUR_ERR_INVALID. */
int aur_kw_add_text(aur_kw* const* stores, int32_t n_stores, aur_kw_vocab* v, const int64_t* ids,
                    const int32_t* user_codes, const int32_t* org_codes, const char* texts_utf8,
                    const int64_t* text_offsets, int64_t n);

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
/* aur_hybrid_search_multi with every query's scope given as a filter program instead of q_user / q_org: query q sees
 * the rows program q_program[q] matches (programs, bitmap and 1 <= n_programs <= 1024 as for aur_search_filtered; the
 * tenant scope is the program [leaf(0, bit u + 1), leaf(1, bit o + 1), OR]).  n = 1 is the single-shard call.
 *   dense leg of shard s   exactly aur_search_filtered on that shard with max_list_rows / n as its bound;
 *   keyword leg of store s exactly aur_kw_search_multi with, for query q, the allow-list of the store's live rows whose
 *                          codes (tenant codes and aur_kw_set_attrs columns) satisfy program q_program[q]; idf and
 *                          avgdl stay corpus-wide, unaffected by the filter.
 * The programs are evaluated on every store's device and the match bits read in place by its scoring kernel (a row that
 * matches no program of a launch is skipped before its postings are read), so the keyword legs need no host sync.  The
 * keyword legs are enqueued first, then every shard's count pass; their small read-back (the list planning needs it) is
 * the call's only host sync before the final copy.  The lists are then merged and fused as aur_hybrid_search_multi does.
 * A column a leaf names must have been set on every shard and every store; q_program [nq] must name programs and
 * max_list_rows be >= 0; every other argument as for aur_hybrid_search_multi (all AUR_ERR_INVALID / _UNSUPPORTED before
 * any device work, the outputs untouched).  snapshot_rows_out [2n] as for aur_hybrid_search_multi. */
int aur_hybrid_search_filtered(aur_index* const* shards, aur_kw* const* stores, int32_t n, const void* queries_host,
                               int32_t nq, int32_t fetch, const int32_t* q_terms, const int64_t* q_offsets,
                               const int32_t* prog, const int32_t* prog_offsets, int32_t n_programs, const uint32_t* bitmap,
                               int64_t bitmap_words, const int32_t* q_program, int64_t max_list_rows,
                               const double* w_dense, const double* w_sparse, int32_t fusion, int32_t k_out,
                               double* scores_out, int64_t* ids_out, float* cosine_out,
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

/* Out of device memory (aur_encoder_open, aur_encoder_load, aur_encoder_replicate): AUR_ERR_NOMEM; earlier releases
 * reported it as AUR_ERR_CUDA. */
int aur_encoder_open(const aur_encoder_config* cfg, aur_encoder** out);
int aur_encoder_close(aur_encoder* enc);
/* Upload one parameter tensor (host fp32; matrices are stored as bf16 on the device).  Names:
 * word_emb [vocab,H], pos_emb [max_pos,H], type_emb [type_vocab,H], emb_ln_g/emb_ln_b [H], and per
 * layer l: l{l}.wqkv [3H,H] (query, key, value rows stacked), l{l}.bqkv [3H], l{l}.wo [H,H],
 * l{l}.bo, l{l}.ln1_g, l{l}.ln1_b, l{l}.wi [I,H], l{l}.bi [I], l{l}.wo2 [H,I], l{l}.bo2,
 * l{l}.ln2_g, l{l}.ln2_b -- all [out_features, in_features] like torch.nn.Linear. */
int aur_encoder_load(aur_encoder* enc, const char* name, const float* data, int64_t count);
/* Host in / host out, one batch of the workspace: aur_encode_texts with one window per text, so out_f32 [n_seq, hidden]
 * and/or out_bf16 [n_seq, hidden] (either may be NULL) hold each sequence's pooled vector and are written only on
 * success.  Checked first, in this order, before any device work: a parameter not loaded yet, tokens or cu_seqlens NULL
 * or n_seq <= 0 (AUR_ERR_INVALID); n_seq > max_seqs (AUR_ERR_NOMEM); cu_seqlens[0] != 0 (AUR_ERR_INVALID);
 * cu_seqlens[n_seq] > max_tokens (AUR_ERR_NOMEM); then aur_encode_texts' checks of the sequences. */
int aur_encode(aur_encoder* enc, const int32_t* tokens, const int32_t* cu_seqlens, int32_t n_seq,
               float* out_f32, uint16_t* out_bf16);
/* Fused ingest: encode the chunks and append the pooled bf16 vectors to the shard without
 * leaving the device (insert_chunks, weaviate_client.py:136-212, minus the text handling).
 * ids NULL (AUR_ERR_INVALID) and aur_encode's one-batch checks first, then aur_encode_append_multi with n = 1 on the
 * caller's thread: every check of that call, a shard without room for the n_seq rows (AUR_ERR_NOMEM), an id < 0 or a
 * shard on another device than the encoder (AUR_ERR_INVALID) among them, is made before any device work, so a rejected
 * call leaves the shard and the encoder's stats untouched.  The one-batch checks come before the shard's: a call over
 * max_seqs or max_tokens gets AUR_ERR_NOMEM even when its shard is f32 or of another dim. */
int aur_encode_append(aur_encoder* enc, aur_index* ix, const int32_t* tokens,
                      const int32_t* cu_seqlens, int32_t n_seq, const int64_t* ids,
                      const int32_t* user_codes, const int32_t* org_codes);
/* A new encoder on `device` (src's own device too) with src's configuration and src's parameters, copied device to device
 * as stored (the head-dim-32 layouts included; cudaMemcpyPeerAsync, peer access neither required nor enabled), so its
 * forward is src's bit for bit.  It has its own workspace, stream, tensor maps, lock and stats and outlives src.  src with
 * a parameter still missing (named as aur_encode names it), device out of range or out NULL: AUR_ERR_INVALID before
 * anything is allocated. */
int aur_encoder_replicate(aur_encoder* src, int32_t device, aur_encoder** out);
/* aur_encode_append over n (1 .. 64) shards taken as one corpus placed by id mod n (engine.MultiIndex): sequence i is
 * encoded by encs[ids[i] mod n] and appended to shards[ids[i] mod n].  encs[s] must be on shards[s]'s device; entries of
 * encs may repeat (shards on one device may share an encoder, which then serves them one batch at a time).  Each shard's
 * share keeps input order and is cut greedily into batches of at most max_tokens_per_call tokens and max_seqs_per_call
 * sequences (0: the encoder's max_tokens / max_seqs), appended in that order, so an id repeated in the call keeps its
 * last occurrence as successive aur_encode_append calls would.  The pooled bf16 rows go into aur_add_dev on the
 * encoder's stream and never leave the device.  Every shard's share runs on its own host thread, all at once; writers of
 * one shard are serialised as aur_add_dev serialises them, and searches are never blocked.  Checked before any device
 * work, leaving every shard and encoder untouched: NULL arguments, n out of range, a NULL or repeated shard, encoders
 * whose configurations (all but the device) differ or with a parameter missing, an encoder on another device than its
 * shard, an f32 shard or one whose dim is not the hidden size, per-call limits outside 0 .. the workspace, an id < 0, a
 * sequence of length outside 1 .. max_pos, a token id outside the vocabulary (AUR_ERR_INVALID); a sequence longer than
 * one call's token budget, a shard without room for its share (rows appended + share > the capacity at the call) (AUR_ERR_NOMEM).  A
 * concurrent writer of the same shard may still use up its room: that shard's append then fails as aur_add_dev fails.
 * A failure after device work has started (a CUDA error) may leave a prefix of some shards' shares appended, whole
 * batches each; aur_last_error names the first failing shard.  aur_encode_append is this call with n = 1 after its
 * one-batch checks, and aur_encode_text_append this call with n = 1 after tokenising. */
int aur_encode_append_multi(aur_encoder* const* encs, aur_index* const* shards, int32_t n, const int32_t* tokens,
                            const int32_t* cu_seqlens, int32_t n_seq, const int64_t* ids, const int32_t* user_codes,
                            const int32_t* org_codes, int32_t max_tokens_per_call, int32_t max_seqs_per_call);
/* Texts of any length in, one vector per text out.  A text is windows cu_texts[j] .. cu_texts[j+1]-1 of the packed
 * sequences (aur_tokenize_windows' layout): cu_texts [n_texts + 1] starts at 0, rises by at least 1 per text and ends at
 * n_seq.  The windows go through the workspace in greedy batches, in order; a text's windows may span batches, its fp32
 * running sum then stays on the device from one batch to the next (the encoder is held for that long).  A text of one
 * window gets its window's pooled vector, bit for bit, whatever else its batch holds; aur_encode is this call with one
 * window per text on one batch.  A text of w >= 2 windows with pooled vectors v_1 .. v_w (each normalised when the
 * encoder normalises) gets, per component and never fused:
 *   s = fl32(..fl32(v_1 + v_2) .. + v_w), m = fl32(s / w);
 *   normalize: q = sum of the exact fp64 squares m_i^2, summed in fp64 as lane sums r_c = m_c^2 + m_{c+32}^2 + .. (in
 *   increasing i) for c = 0 .. 31, then r_0 + r_1 + .. + r_31; out_i = fl32(m_i / sqrt(q)) in fp64 when q > 0, else m;
 *   without normalize, out = m.  The bf16 row rounds out to nearest even (oracle/window_mean.py restates this).
 * out_f32 / out_bf16 [n_texts, hidden] (either may be NULL) are written only on success.  Checked before any device
 * work: the checks of aur_encode_append_multi that apply, and cu_texts (AUR_ERR_INVALID). */
int aur_encode_texts(aur_encoder* enc, const int32_t* tokens, const int32_t* cu_seqlens, int32_t n_seq,
                     const int32_t* cu_texts, int32_t n_texts, float* out_f32, uint16_t* out_bf16);
/* Texts in (aur_encode_texts' packed windows), cosines of text pairs out: pair p is (pair_a[p], pair_b[p]), indices
 * into the n_texts texts.  cos_out [n_pairs] fp64; vec_out [n_texts, hidden] fp32 (nullable).  vec_out is
 * aur_encode_texts' out_f32 for the same inputs, bit for bit, and cos_out[p] is what aur_cosine_pairs returns for rows
 * pair_a[p] and pair_b[p] of it with the same clamp, bit for bit (0.0 for a zero norm; clamp = 1 applies the [0, 1]
 * clamp of similarity.py:98).  The texts go through the workspace as aur_encode_texts runs them; their vectors stay on
 * the device until one gather launch has scored every pair, and one copy brings the cosines back (and one the vectors).
 * Outputs are written only on success.  Checked before any device work, leaving the outputs and the encoder's stats
 * untouched: every check of aur_encode_texts, n_pairs < 0, pair_a, pair_b or cos_out NULL while n_pairs > 0, a pair
 * index outside 0 .. n_texts - 1, clamp not 0 or 1 (AUR_ERR_INVALID).  A failed allocation of the call's device
 * buffers (the text vectors, the pairs, the cosines) is AUR_ERR_NOMEM. */
int aur_encode_pair_cosines(aur_encoder* enc, const int32_t* tokens, const int32_t* cu_seqlens, int32_t n_seq,
                            const int32_t* cu_texts, int32_t n_texts, const int32_t* pair_a, const int32_t* pair_b,
                            int64_t n_pairs, int32_t clamp, double* cos_out, float* vec_out);
/* aur_encode_append_multi with texts as the unit: text j (its windows, cu_texts as for aur_encode_texts) is encoded by
 * encs[ids[j] mod n] into the vector aur_encode_texts gives it and appended, as bf16, to shards[ids[j] mod n]; each
 * shard's rows are appended in input order; room is counted in texts; ids, user_codes and org_codes are [n_texts].  The
 * checks, threads and failure behaviour are aur_encode_append_multi's, plus a malformed cu_texts (AUR_ERR_INVALID).
 * aur_encode_append_multi is this call with one window per text. */
int aur_encode_append_texts_multi(aur_encoder* const* encs, aur_index* const* shards, int32_t n, const int32_t* tokens,
                                  const int32_t* cu_seqlens, int32_t n_seq, const int32_t* cu_texts, int32_t n_texts,
                                  const int64_t* ids, const int32_t* user_codes, const int32_t* org_codes,
                                  int32_t max_tokens_per_call, int32_t max_seqs_per_call);
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
/* Every text as the windows of its whole tokenisation [CLS] b [SEP] for a position table of max_len (>= 3): one window,
 * aur_tokenize's output, when 2 + |b| <= max_len; otherwise [CLS] b[i : i + max_len - 2] [SEP] for i = 0, max_len - 2,
 * .. < |b|.  Packed: tokens_out (capacity tokens_cap ids), cu_seqlens_out [windows + 1] over windows (capacity seqs_cap
 * windows) and cu_texts_out [n_texts + 1] (text j = windows cu_texts[j] .. cu_texts[j+1]-1).  totals_out [2] (may be
 * NULL) receives the windows and tokens needed.  tokens_out = cu_seqlens_out = NULL with both capacities 0 is count mode
 * (cu_texts_out and totals_out only); capacities too small: AUR_ERR_NOMEM, with cu_texts_out and totals_out written. */
int aur_tokenize_windows(aur_tokenizer* t, const char* texts_utf8, const int64_t* offsets, int32_t n_texts, int32_t max_len,
                         int32_t* tokens_out, int64_t tokens_cap, int32_t* cu_seqlens_out, int32_t seqs_cap,
                         int32_t* cu_texts_out, int64_t* totals_out, int32_t n_threads);
/* Text in, rows in the shard: tokenise, encoder forward, append -- insert_chunks (weaviate_client.py:136-212) without
 * Python on the path.  Every text is tokenised by aur_tokenize, truncated to max_len ids (a longer text loses its tail:
 * aur_tokenize_windows + aur_encode_append_texts_multi keep it), then the texts go, one sequence each, through
 * aur_encode_append_multi(&enc, &ix, 1, ..., max_tokens_per_call, max_seqs_per_call): batches are cut to those limits,
 * and every check of that call (a limit above the encoder's workspace, AUR_ERR_INVALID, among them) is made before any
 * device work, so a rejected call appends nothing.  Checked first: NULL enc, tok, ix or ids (AUR_ERR_INVALID); then
 * n_texts <= 0 returns AUR_OK with nothing done; then max_len outside 2 .. 512, max_tokens_per_call < max_len or
 * max_seqs_per_call < 1 (AUR_ERR_INVALID). */
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
/* The tensor-core similarity kernel's first pass, before any selection: nq <= 128 queries (device bf16) against the
 * published rows, launched with the index's tc_tile / tc_qregs options (an unset tc_tile means 64-row tiles here).  Every
 * CTA writes the whole first corpus tile of its tile set, unscaled by |q|: out_dev [n_ctas, 64 queries, tile_n rows].
 * For int8 rows a score is q16 . c times the row's inverse norm, q16 the kernel's 16-bit query image.  out_cap: floats
 * out_dev holds; too few for n_ctas * 64 * tile_n fails with AUR_ERR_INVALID before anything runs. */
int aur_debug_tc_scores(aur_index* ix, const void* queries_dev, int32_t nq, int32_t cta_group, float* out_dev,
                        int64_t out_cap, int32_t* n_ctas_out, int32_t* tile_n_out, void* stream);
/* The generic kernel's first-pass scores of nq <= 1024 queries (host, as aur_search) over every published row, launched
 * as aur_search launches it (q_user / q_org: tenant codes as aur_search, nullable): out_host [nq, n_rows] row-major,
 * -inf where a row is invisible, NaN where the kernel wrote nothing.  *n_rows_out = the rows; out_cap as above. */
int aur_debug_simt_scores(aur_index* ix, const void* queries_host, int32_t nq, const int32_t* q_user,
                          const int32_t* q_org, float* out_host, int64_t out_cap, int64_t* n_rows_out);
/* The list kernel's first-pass scores of aur_search_lists(ix, queries_host, nq, ., list_ids, list_offsets, n_lists,
 * q_list, ...): out_host [nq, n_rows], the score of query q against every row of its list, NaN elsewhere. */
int aur_debug_list_scores(aur_index* ix, const void* queries_host, int32_t nq, const int64_t* list_ids,
                          const int64_t* list_offsets, int32_t n_lists, const int32_t* q_list, float* out_host,
                          int64_t out_cap, int64_t* n_rows_out);

#ifdef __cplusplus
}
#endif
#endif /* AURORA_B200_H_ */
