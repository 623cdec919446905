// Internal declarations shared by the kernels and the C-ABI host runtime.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdlib.h>

#include <functional>
#include <vector>

struct aur_index;
struct aur_kw;

namespace aur {

// ---------------------------------------------------------------- candidate keys
// A candidate is one uint64: high word = order-preserving image of the fp32 score, low
// word = ~row so that, for equal scores, the LOWER row index compares GREATER.  Sorting
// keys in descending order therefore yields (score desc, row asc).
constexpr uint64_t kKeyEmpty = 0x007FFFFF00000000ull;  // score -inf, row -1
__host__ __device__ __forceinline__ uint32_t f32_to_ord(float f) {
#ifdef __CUDA_ARCH__
  uint32_t u = __float_as_uint(f);
#else
  union { float f; uint32_t u; } c; c.f = f; uint32_t u = c.u;
#endif
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float ord_to_f32(uint32_t o) {
  uint32_t u = (o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o;
#ifdef __CUDA_ARCH__
  return __uint_as_float(u);
#else
  union { float f; uint32_t u; } c; c.u = u; return c.f;
#endif
}
__host__ __device__ __forceinline__ uint64_t make_key(float score, int32_t row) {
  return (static_cast<uint64_t>(f32_to_ord(score)) << 32) | static_cast<uint32_t>(~row);
}
__host__ __device__ __forceinline__ int32_t key_row(uint64_t k) { return static_cast<int32_t>(~static_cast<uint32_t>(k)); }
__host__ __device__ __forceinline__ float key_score(uint64_t k) { return ord_to_f32(static_cast<uint32_t>(k >> 32)); }
#ifdef __CUDACC__
// Candidate order wherever keys are compared, kept or evicted: (approximate score desc, id asc) -- the order of the
// final ranking and of the cross-shard merge, so a group of tied rows cut anywhere keeps its lowest ids.  The key
// carries the row (needed to fetch the vector); equal scores load ids[row], so only ties pay.  Keys without a row
// (empty slots, sort padding) and equal ids fall back to the raw key: a strict total order on distinct keys.
__device__ __forceinline__ bool key_before(uint64_t a, uint64_t b, const int64_t* __restrict__ ids) {
  if ((a ^ b) >> 32) return a > b;
  const int32_t ra = key_row(a), rb = key_row(b);
  if ((ra | rb) < 0 || ra == rb) return a > b;
  const int64_t ia = __ldg(ids + ra), ib = __ldg(ids + rb);
  return ia != ib ? ia < ib : a > b;
}
#endif

// ---------------------------------------------------------------- wgmma similarity kernel
constexpr int kTcTileN = 64;       // corpus rows per tile  (MMA N); the bring-up score dump keeps this width
constexpr int kTcTileWide = 128;   // the wide tile (wgmma m64n128), picked per launch when its layout fits
constexpr int kTcWideMinStages = 4;   // with three 16 KB stages the wide tile measured no faster than the 64-row one
constexpr int kTcKBlock = 64;      // bf16 per 128-byte swizzled smem row (one pipeline stage)
constexpr int kTcQRows = 64;       // queries per CTA (MMA M of one warpgroup)
constexpr int kTcChunk = 16;       // scores examined per threshold test
constexpr int kTcListMin = 64;     // list slots per query: max(ksel, this) so a whole first tile appends
constexpr int kTcMaxStages = 12;
constexpr int kTcMaxDim = 1024;    // largest dim served by the tensor-core path (the query block stays in shared memory)
constexpr int kTcFifoRecs = 16;    // parked 4-score groups per thread before the deferred slow path runs
constexpr int kTcFifoMaxKsel = 64; // (the FIFO shares shared memory with the candidate lists)
constexpr int kSlack = 8;          // extra candidates kept for the exact re-rank
constexpr int kMaxK = 128;

struct TcParams {
  const __nv_bfloat16* q;   // [nq, dim] queries of this launch (<= 64 * n_qblocks)
  const float* inv_norm;    // [n_rows]   1/|c_j|, 0 for zero rows, NaN for tombstones
  const uint32_t* row_mask; // nullable [n_rows]: bit s = tenant scope s of this batch may see the row (per-query scopes)
  const int32_t* q_scope;   // with row_mask: [nq] scope index (0..31) of every query
  const int64_t* ids;       // [n_rows] external ids: break ties between candidate keys (key_before)
  uint64_t* cand;          // [64 * n_qblocks, n_lists * ksel] candidate keys, compacted per
                            // query: only keys that pass the final threshold are appended
  uint32_t* cand_count;     // [64 * n_qblocks] appended keys per query (zero on entry)
  float* dbg_scores;        // optional [grid, 64, 64]: first tile's scores of every CTA
  uint64_t* pub;            // cross-CTA threshold exchange, entries (epoch << 32 | score bits):
                            // [n_qblocks, 64, n_lists (even)] each CTA's m-th best per query,
                            // then [n_qblocks, 64] the served thresholds
  int64_t n_rows;
  uint32_t epoch;           // launch counter: pub entries of other launches are ignored (kSearchEpochMax)
  const uint32_t* epoch_ptr;// when set, the counter lives in device memory (bumped by the finalize kernel)
  int nq, dim, ksel, n_lists, n_qblocks, num_stages, n_tiles;
  int dbg_flags;            // bring-up only (timing decomposition; results are wrong with 1..32): 1 = epilogue neither
                            // reads nor examines the accumulator, 2 = no MMAs issued, 4 = accumulator read but not
                            // examined, 8 = scaled + maxima but no threshold test, 16 = no per-tile threshold read,
                            // 32 = no inverse-norm prefetch, 64 = per-thread counters into dbg_scores
};
constexpr int kTcPubMax = 74;      // published values a thread folds into its threshold
// Searches tag their exchange entries with the device-resident counter, which runs 1 .. kSearchEpochMax and wraps back
// to 1; the bring-up entry point (aur_debug_tc_scores) tags from the disjoint upper half, so neither ever reads the
// other's entries as its own.  0 is never a tag: it marks a zeroed table.
constexpr uint32_t kSearchEpochMax = 0x7FFFFFFFu;

// tile_n: corpus rows per tile, kTcTileN or kTcTileWide; mask: a kMask launch (row_mask set).
size_t tc_smem_bytes(int num_stages, int ksel, int dim, int tile_n, bool mask);
int tc_pick_stages(int ksel, int dim, size_t smem_limit, int tile_n, bool mask);
// Launches the fused similarity + top-k kernel; cta_group 2 = two-CTA clusters sharing every corpus tile by TMA
// multicast.  tmap: CUtensorMap over the corpus with a {64, tile_n / cta_group} box and 128-byte swizzle.
cudaError_t tc_launch(int cta_group, int tile_n, int grid, const void* tmap, const TcParams& p, size_t smem, cudaStream_t s);

// ---------------------------------------------------------------- SIMT kernels
struct FilterArgs {
  const int32_t* row_user;  // [n_rows]
  const int32_t* row_org;   // [n_rows]
  const int32_t* q_user;    // [nq]   (nullptr = unfiltered)
  const int32_t* q_org;     // [nq]   (nullptr = none)
};

cudaError_t launch_row_inv_norms(const void* rows, int dtype, int dim, int64_t n, float* inv_norm, cudaStream_t s);
// Generic path: scores of a chunk of rows for all queries, then per-segment selection.
constexpr int kSimtSeg = 2048;    // corpus rows per selection segment (one candidate list)
cudaError_t launch_simt_scores(const void* q, const void* rows, int dtype, int dim, int nq, int64_t row0,
                               int64_t nrows_chunk, int64_t n_rows, const float* inv_norm, FilterArgs f,
                               float* scores /* [nq, nrows_chunk] */, cudaStream_t s);
cudaError_t launch_simt_select(const float* scores, int nq, int64_t row0, int64_t nrows_chunk, int ksel,
                               const int64_t* ids, uint64_t* cand, int n_lists, int list0, cudaStream_t s);
// [nq, n_lists, ksel] -> [nq, ceil(n_lists/group), ksel]; group*ksel <= 4096
cudaError_t launch_reduce_lists(const uint64_t* in, int nq, int n_lists, int ksel, int group, const int64_t* ids,
                                uint64_t* out, cudaStream_t s);
// Final stage: best ksel of n_lists*ksel (<= 4096) keys, exact fp64 cosine re-rank,
// (score desc, id asc) order, top-k out.
struct FinalizeArgs {
  const uint64_t* cand; int n_lists; int ksel;
  uint32_t* counts;  // nullable: per-query number of valid keys at the front of its cand row
                     // (reset to 0 by the kernel); null = all n_lists * ksel slots are keys
  uint32_t* epoch_bump;  // nullable: the tensor-core kernel's device-resident launch counter, advanced here (never 0)
  uint32_t* cand_read;   // nullable: per query, the number of candidate keys the re-rank read (aur_stats.last_candidates)
  const void* q; const void* rows; int dtype; int dim; int nq; int k;
  const int64_t* ids;
  float* out_scores; int64_t* out_ids; double* out_scores64;   // (out_scores / out_ids nullable in exchange mode)
  int sort_cap;      // set by launch_finalize: keys the shared sort buffer holds
  // Fused cross-shard exchange (ExchangeOut.n_peers > 0): the exact (fp64 score, id) rows of this shard are stored
  // straight into every rank's exchange buffer over NVLink instead of a local array + all-gather.  Every 8-byte word
  // that crosses carries 4 bytes of payload and a 4-byte tag (the exchange's sequence number), so a word is valid the
  // moment its tag matches: 8-byte stores are single-copy atomic, the receiver polls the words themselves, and no
  // flag, fence or counter sits on the critical path (the layout NCCL's LL protocol uses).  An entry = 4 words:
  // score lo, score hi, id lo, id hi.
  struct ExchangeOut {
    uint64_t* slot[8];          // per destination rank: base of THIS rank's slot in that rank's buffer (parity 0)
    int n_peers;                // 0 = off
    const uint64_t* seq;        // device word: exchanges completed so far (this one is *seq + 1; parity = its low bit)
    size_t parity_stride;       // 8-byte words between the two parities of a buffer
    int q0;                     // first query of this launch inside the batch
  } ex;
};
// Cross-shard merge fed by the peer stores above: poll the tagged words of all ranks' slots, keep the best k.
struct ExchangeParams {
  uint64_t* slots;              // this rank's buffer: [2 parity][world][nq_max * k_max entries][4 words]
  uint64_t* seq;                // device word, bumped by the last block
  uint32_t* done;               // block counter (self-resetting)
  uint32_t* status;             // != 0: a peer did not deliver in time
  int world, rank, nq, k;
  size_t parity_stride, slot_stride;   // in words
  float* out_scores; int64_t* out_ids;
};
cudaError_t launch_exchange_merge(const ExchangeParams& p, cudaStream_t s);
cudaError_t launch_finalize(const FinalizeArgs& a, cudaStream_t s);
// shard_stride: elements between consecutive shards' blocks in in_s / in_ids
cudaError_t launch_merge_topk(const double* in_s, const int64_t* in_ids, size_t shard_stride, int n_shards, int nq, int k,
                              float* out_s, int64_t* out_ids, double* out_s64, cudaStream_t s);
cudaError_t launch_cosine_pairs(const float* a, const float* b, int64_t n, int dim, int clamp, double* out,
                                cudaStream_t s);
cudaError_t launch_fill_f32(float* p, float v, int64_t n, cudaStream_t s);
// out[i] = OR over the batch's distinct tenant scopes s < n_scopes of (visible(row i, scope s) << s); scopes = {user, org} pairs
cudaError_t launch_row_scope_mask(const int32_t* row_user, const int32_t* row_org, const int32_t* scopes, int n_scopes, int64_t n,
                                  uint32_t* out, cudaStream_t s);
// out[i] = visible(user u, org o) ? inv[i] : NaN  -- lets the tensor-core kernel serve a batch whose queries all
// carry the same tenant scope
cudaError_t launch_mask_inv_norm(const float* inv, const int32_t* row_user, const int32_t* row_org, int32_t u, int32_t o,
                                 int64_t n, float* out, cudaStream_t s);

// ---------------------------------------------------------------- per-query pre-filter lists (listsearch.cu)
constexpr int kListQMax = 64;     // queries of one work item (four m16 MMA row blocks)
// One work item: rows list_rows[row0 .. row0 + n_rows) (n_rows <= kSimtSeg, segment `seg` of the list) against the
// queries qidx[q0 .. q0 + nq) (nq <= kListQMax); their scores go to rows out .. out + nq of the score scratch.
struct ListItem { int32_t row0, n_rows, seg, q0, nq, out; };
struct ListParams {
  const __nv_bfloat16* q;      // [nq of the query block, dim]
  const __nv_bfloat16* rows;   // the shard's rows
  const float* inv_norm;       // NaN = tombstone
  const int64_t* ids;
  const ListItem* items; int n_items;
  const int32_t* list_rows;    // resolved rows of every list, each list sorted and without repeats
  const int32_t* qidx;         // query (position in the block) of every item slot
  float* scores;               // scratch [sum of the items' nq][kSimtSeg]
  uint64_t* cand;              // [queries of the block, n_lists, ksel] candidate keys (slots no item writes: zero)
  int dim, ksel, n_lists;
};
// Scores and per-segment selection of n_items work items; max_nq = the largest nq among them.
cudaError_t launch_list_search(const ListParams& p, int max_nq, cudaStream_t s);

// ---------------------------------------------------------------- metadata pre-filters (filter.cu)
constexpr int kFiltAttrCols = 16;             // attribute columns per shard
constexpr int kFiltCols = 2 + kFiltAttrCols;  // program columns: 0 = tenant user codes, 1 = org codes, 2.. attributes
constexpr int kFiltMaxLeaves = 32;            // leaves per program (its evaluation stack is one 32-bit word)
constexpr int kFiltMaxPrograms = 32;          // programs per pass (bit p of a row's match mask)
constexpr int kFiltCallPrograms = 1024;       // programs per call, evaluated in passes of kFiltMaxPrograms
constexpr int kFiltBlockRows = 2048;          // rows per CTA of the count and write kernels
enum { kFiltLeaf = 0, kFiltAnd = 1, kFiltOr = 2 };
struct FiltToken { int32_t kind, col, bm_off, bm_len; };   // bm_off / bm_len in bits; AND / OR ignore the rest
struct FiltParams {
  const int32_t* cols[kFiltCols];   // [n_rows] codes per column (only the columns the programs name are read)
  const FiltToken* tok;             // every program's tokens, postfix
  const int32_t* prog_off;          // [n_programs + 1] program q = tok[prog_off[q] .. prog_off[q + 1])
  const uint32_t* bitmap;           // leaf bitmaps
  const float* inv_norm;            // NaN = tombstone (never matches)
  int64_t n_rows;                   // the search's snapshot
  int n_programs;
};
int filter_blocks(int64_t n_rows);
// mask [n_rows] (bit q = program q), block_counts [n_programs][filter_blocks(n_rows)], totals [32] (zeroed here)
cudaError_t launch_filter_count(const FiltParams& p, uint32_t* mask, uint32_t* block_counts, uint32_t* totals, cudaStream_t s);
// rows_out [sum of totals]: program q's matching rows, ascending, after those of programs < q; ids_out (nullable) their ids.
// Scans block_counts in place.
cudaError_t launch_filter_write(const uint32_t* mask, uint32_t* block_counts, const uint32_t* totals, int n_programs, int64_t n_rows,
                                const int64_t* ids, int32_t* rows_out, int64_t* ids_out, cudaStream_t s);
// out[i] = (mask[i] & 1) ? inv[i] : NaN
cudaError_t launch_mask_match(const float* inv, const uint32_t* mask, int64_t n, float* out, cudaStream_t s);
// col[pairs[2i]] = pairs[2i + 1]
cudaError_t launch_scatter_codes(const int32_t* pairs, int64_t n, int32_t* col, cudaStream_t s);
// out[i] = src[map[i]] (compaction of an attribute column)
cudaError_t launch_gather_i32(const int32_t* src, const int32_t* map, int64_t n, int32_t* out, cudaStream_t s);

// out[rows[i]] = inv[rows[i]] for the listed rows (out pre-filled with NaN): a resolved id subset as a row mask
cudaError_t launch_scatter_inv_norm(const float* inv, const int32_t* rows, int64_t n, int64_t n_rows, float* out, cudaStream_t s);
// compaction: rows map[0..n) (and their side arrays) -> bounce buffers
cudaError_t launch_gather_rows(const void* rows, const float* inv, const int64_t* ids, const int32_t* user, const int32_t* org,
                               const int32_t* map, int64_t n, int row_bytes, void* o_rows, float* o_inv, int64_t* o_ids,
                               int32_t* o_user, int32_t* o_org, cudaStream_t s);

// ---------------------------------------------------------------- encoder (BERT-family forward)
// out = epi(A . W^T + bias): A [m_tiles*128, K] bf16 (TMA box {64,128}), W [N, K] bf16 (TMA box {64,BN/cta_group}).
enum { kEpiBias = 0, kEpiBiasGelu = 1, kEpiBiasResid = 2 };
struct GemmParams {
  const float* bias;            // [N]
  const __nv_bfloat16* resid;   // [rows, ldr] (kEpiBiasResid only)
  int ldr;
  __nv_bfloat16* out;           // [m_tiles * 128 * cta_group, ldo]
  int ldo;
  int m_tiles, n_tiles, k_blocks;   // (128 * cta_group)-row tiles, BN-column tiles, 64-wide k-blocks
};
cudaError_t gemm_tc_launch(int cta_group, int bn, int epi, int sm_count, const void* tmap_a, const void* tmap_b,
                           const GemmParams& p, cudaStream_t s);

// Self-attention over packed variable-length sequences (<= 512 tokens each), head dim 64.
// One work item = (sequence, 128-query block); every item runs for all heads.
struct AttnItem { int32_t tok0, len, q0, pad; };   // first token row, length, first query of the block
struct AttnParams {
  const AttnItem* items; int n_items; int heads; int hidden;
  __nv_bfloat16* ctx; int ld_ctx;     // [tokens, hidden] context output
  float scale_log2e;                  // log2(e) / sqrt(head_dim)
};
// tmap_qkv: CUtensorMap over the packed [tokens, 3*hidden] projections, box {64, 128}, SWIZZLE_128B.
cudaError_t attn_tc_launch(const void* tmap_qkv, const AttnParams& p, cudaStream_t s);

cudaError_t launch_embed_ln(const int32_t* tok, const int32_t* pos, int n_tok, int n_rows_pad,
                            const __nv_bfloat16* word, const __nv_bfloat16* pos_emb, const __nv_bfloat16* type_emb,
                            const float* g, const float* b, float eps, int hidden, __nv_bfloat16* out, cudaStream_t s);
cudaError_t launch_layernorm(const __nv_bfloat16* in, const float* g, const float* b, float eps, int n_rows, int hidden,
                             __nv_bfloat16* out, cudaStream_t s);
// pool_mode 0 = first token (CLS), 1 = mean over the sequence; optional L2 normalisation.
cudaError_t launch_pool(const __nv_bfloat16* x, const int32_t* cu, int n_seq, int hidden, int pool_mode, int normalize,
                        float* out_f32, __nv_bfloat16* out_bf16, cudaStream_t s);
cudaError_t launch_f32_to_bf16(const float* in, __nv_bfloat16* out, int64_t n, cudaStream_t s);

// Launch with programmatic dependent launch enabled (and an optional cluster size): the kernel may
// start its prologue while the previous kernel of the stream drains; it must call
// ptx::grid_dep_wait() before touching that kernel's output.
template <typename... KArgs, typename... Args>
cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, int cluster,
                       Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
  cudaLaunchAttribute attr[2];
  int n = 0;
  attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[n].val.programmaticStreamSerializationAllowed = 1;
  ++n;
  if (cluster > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster; attr[n].val.clusterDim.y = 1; attr[n].val.clusterDim.z = 1;
    ++n;
  }
  cfg.attrs = attr; cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

template <typename T>
struct DevBuf {   // grow-only device scratch
  T* p = nullptr; size_t n = 0;
  cudaError_t reserve(size_t want) {
    if (want <= n) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr; n = 0;
    cudaError_t e = cudaMalloc(&p, want * sizeof(T));
    if (e == cudaSuccess) n = want;
    return e;
  }
  void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
};

// ---------------------------------------------------------------- the two legs of a hybrid query (hybrid.cu)
// Dense leg: the search aur_search_ex runs for these host queries and per-query tenant codes (same scope handling, same
// kernels, same answer), enqueued on stream s of `device` over the prefix published now, into the device arrays
// scores / ids [nq * k].  Nothing waits; *snapshot_rows receives the prefix.  A bf16 index on `device` only
// (else AUR_ERR_UNSUPPORTED / AUR_ERR_INVALID).  The leg's aur_stats.last_* are the index's last search.  (capi.cu)
int dense_leg(aur_index* ix, int device, cudaStream_t s, const void* queries_host, int32_t nq, int32_t k, const int32_t* q_user,
              const int32_t* q_org, float* scores, int64_t* ids, int64_t* snapshot_rows);
int index_device(const aur_index* ix);
int index_is_bf16(const aur_index* ix);
// Keyword legs: aur_kw_search_multi's search (no allow-list) over stores[0 .. n) (distinct, non-NULL, 1 <= n <= 64)
// taken as one corpus, each store's part enqueued on its own context and stream; then then(legs) runs with every
// store's (device, stream, top-k lists, snapshot) -- device arrays [nq * k], valid once the stream reaches them,
// sorted by (fp64 score desc, id asc) -- while every store's shared lock and every context are held.  Each store's
// aur_kw_stats.last_* are published after then() returns AUR_OK.  The query arguments are checked by kw_check.  (keyword.cu)
struct KwLeg { int device; cudaStream_t stream; const double* scores; const int64_t* ids; int64_t snapshot_rows; };
using KwLegsThen = std::function<int(const std::vector<KwLeg>& legs)>;
int kw_legs(aur_kw* const* stores, int n, const int32_t* q_terms, const int64_t* q_offsets, int32_t nq, int32_t k,
            const int32_t* q_user, const int32_t* q_org, const KwLegsThen& then);
int kw_check(const int32_t* q_terms, const int64_t* q_offsets, int32_t nq, int32_t k);   // aur_kw_search's query checks
int kw_device(const aur_kw* kw);

// Error reporting shared by the translation units behind the C ABI (thread-local message).
int report_error(int code, const char* fmt, ...);
// 2-D bf16 tensor map, 128-byte swizzle; returns 0 or a CUresult.
int encode_tmap_2d_bf16(void* tmap, const void* base, uint64_t cols, uint64_t rows, uint64_t row_stride_bytes,
                        uint32_t box_cols, uint32_t box_rows);

}  // namespace aur
