// Internal declarations shared by the kernels and the C-ABI host runtime.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdlib.h>

#include <algorithm>
#include <functional>
#include <memory>
#include <mutex>
#include <vector>

#include "../../include/aurora_b200.h"

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
constexpr int kTcKBlockI8 = 128;   // int8 per 128-byte swizzled smem row (a stage of an int8 shard: twice the dimensions)
// Leading query k-blocks a 128-row launch keeps in the MMA warpgroup's registers (16 registers a thread each) when
// dim / 64 has that many, instead of 8 KB shared-memory tiles: every two of them buy one more 16 KB ring stage.
constexpr int kTcQRegs = 6;   // 4 measured slower (six ring stages at dim 768 / top-32 against seven), 8 spills
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
  float* dbg_scores;        // optional [grid, 64, tile_n]: the whole first tile's scores of every CTA
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

// tile_n: corpus rows per tile, kTcTileN or kTcTileWide; mask: a kMask launch (row_mask set); qregs: leading query
// k-blocks held in registers, which take no shared memory (0 or kTcQRegs, the latter with 128-row tiles only).
size_t tc_smem_bytes(int num_stages, int ksel, int dim, int tile_n, bool mask, int qregs = 0);
int tc_pick_stages(int ksel, int dim, size_t smem_limit, int tile_n, bool mask, int qregs = 0);
// Launches the fused similarity + top-k kernel; cta_group 2 = two-CTA clusters sharing every corpus tile by TMA
// multicast.  tmap: CUtensorMap over the corpus with a {64, tile_n / cta_group} box (i8: int8 rows, a {128, ...} UINT8
// box, p.q the query image of launch_query_image_i8) and 128-byte swizzle.
cudaError_t tc_launch(int cta_group, int tile_n, int qregs, bool i8, int grid, const void* tmap, const TcParams& p, size_t smem,
                      cudaStream_t s);

// ---------------------------------------------------------------- SIMT kernels
struct FilterArgs {
  const int32_t* row_user;  // [n_rows]
  const int32_t* row_org;   // [n_rows]
  const int32_t* q_user;    // [nq]   (nullptr = unfiltered)
  const int32_t* q_org;     // [nq]   (nullptr = none)
};

cudaError_t launch_row_inv_norms(const void* rows, int dtype, int dim, int64_t n, float* inv_norm, cudaStream_t s);
// The tensor-core kernel's query operand for int8 rows: per bf16 query q16 = rint(q * 32512 / max|q|) (0 for a zero query)
// split as q16 = 256 hi + lo, hi = (q16 + 128) >> 8, both int8; written [nq][dim / 128][hi 128 B | lo 128 B].
cudaError_t launch_query_image_i8(const __nv_bfloat16* q, int dim, int nq, int8_t* out, cudaStream_t s);
// Ingest into an int8 shard: bf16 rows in -> int8 rows and their inverse norms out (oracle/quantize.py's rule).
cudaError_t launch_quantize_rows_i8(const __nv_bfloat16* in, int dim, int64_t n, int8_t* out, float* inv_norm, cudaStream_t s);
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
  const void* q; const void* rows; int dtype; int dim; int nq; int k;   // q: bf16 for bf16 and int8 rows, f32 for f32
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
// out[p] = the cosine launch_cosine_pairs gives rows pa[p] and pb[p] of vecs [*, dim], bit for bit.
cudaError_t launch_cosine_gather(const float* vecs, const int32_t* pa, const int32_t* pb, int64_t n, int dim, int clamp,
                                 double* out, cudaStream_t s);
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
  const void* rows;            // the shard's rows: bf16, or int8 when rows_i8 (converted exactly to bf16 on the gather)
  const float* inv_norm;       // NaN = tombstone
  const int64_t* ids;
  const ListItem* items; int n_items;
  const int32_t* list_rows;    // resolved rows of every list, each list sorted and without repeats
  const int32_t* qidx;         // query (position in the block) of every item slot
  float* scores;               // scratch [sum of the items' nq][kSimtSeg]
  uint64_t* cand;              // [queries of the block, n_lists, ksel] candidate keys (slots no item writes: zero)
  int dim, ksel, n_lists;
  bool rows_i8;
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
  const float* inv_norm;            // a vector shard's rows: NaN = tombstone (never matches)
  const uint8_t* live;              // a keyword store's rows (launch_filter_mask): 0 = tombstone (never matches)
  int64_t n_rows;                   // the search's snapshot
  int n_programs;
};
int filter_blocks(int64_t n_rows);
// Passes of kFiltMaxPrograms programs a call of n_programs takes, and the programs of pass ps.
inline int filter_passes(int32_t n_programs) { return (n_programs + kFiltMaxPrograms - 1) / kFiltMaxPrograms; }
inline int filter_pass_programs(int32_t n_programs, int ps) { return std::min(kFiltMaxPrograms, n_programs - ps * kFiltMaxPrograms); }
// mask [n_rows] (bit q = program q), block_counts [n_programs][filter_blocks(n_rows)], totals [32] (zeroed here)
cudaError_t launch_filter_count(const FiltParams& p, uint32_t* mask, uint32_t* block_counts, uint32_t* totals, cudaStream_t s);
// The same pass over a keyword store's rows (liveness from p.live): mask [n_rows] only, no counts, nothing read back.
cudaError_t launch_filter_mask(const FiltParams& p, uint32_t* mask, cudaStream_t s);
// The programs of one call (aur_search_filtered, aur_hybrid_search_filtered), as the C ABI takes them; q_program [nq].
struct FiltProgs {
  const int32_t* prog; const int32_t* prog_off; int32_t n_programs;
  const uint32_t* bitmap; int64_t bitmap_words;
  const int32_t* q_program;
};
// fp's structure (n_programs, offsets, tokens, depth, leaves, column range, bitmap slices), then a call's q_program
// [nq] and max_list_rows.  Whether the columns are set is AttrColumns::check, per holder.
int filter_check_programs(const FiltProgs& fp);
int filter_check_queries(const FiltProgs& fp, int32_t nq, int64_t max_list_rows);
// rows_out [sum of totals]: program q's matching rows, ascending, after those of programs < q; ids_out (nullable) their ids.
// Scans block_counts in place.
cudaError_t launch_filter_write(const uint32_t* mask, uint32_t* block_counts, const uint32_t* totals, int n_programs, int64_t n_rows,
                                const int64_t* ids, int32_t* rows_out, int64_t* ids_out, cudaStream_t s);
// out[i] = (mask[i] & 1) ? inv[i] : NaN
cudaError_t launch_mask_match(const float* inv, const uint32_t* mask, int64_t n, float* out, cudaStream_t s);

// out[rows[i]] = inv[rows[i]] for the listed rows (out pre-filled with NaN): a resolved id subset as a row mask
cudaError_t launch_scatter_inv_norm(const float* inv, const int32_t* rows, int64_t n, int64_t n_rows, float* out, cudaStream_t s);
// deletes: inv[rows[i]] = NaN (the tombstone) for the listed rows, one launch
cudaError_t launch_tombstone_rows(const int32_t* rows, int64_t n, float* inv, cudaStream_t s);
// checkpoints: bit r % 32 of word r / 32 of live = row r's inverse norm is not NaN, of nonfinite (i8 only) = it is
// infinite, for rows [0, n); one warp per word, every word of ceil(n / 32) written
cudaError_t launch_live_bits(const float* inv, int64_t n, int i8, uint32_t* live, uint32_t* nonfinite, cudaStream_t s);
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
// One text's share of a batch for window_fold_kernel: pooled rows [first, end) are its windows in this batch; windows is
// its window count over all batches; kFoldCarryIn: the running sum of its earlier windows is in carry_in;
// kFoldOpen: its windows continue in the next batch (the sum goes to carry_out, no output).  Item i writes row i.  One
// batch may finish a carried text and leave another open, so carry_in and carry_out are two rows.
struct FoldItem { int32_t first, end, windows, flags; };
constexpr int32_t kFoldCarryIn = 1, kFoldOpen = 2;
// pool_f32 [n, hidden] window vectors -> out_f32 / out_bf16 [item, hidden] text vectors; carry rows [hidden] fp32.
cudaError_t launch_window_fold(const float* pool_f32, const FoldItem* items, int n_items, int hidden, int normalize,
                               const float* carry_in, float* carry_out, float* out_f32, __nv_bfloat16* out_bf16, cudaStream_t s);

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

// ---------------------------------------------------------------- owners of CUDA resources
// Move-only; the destructor frees.  An owner is destroyed with its own device current (every close sets it first).
// None has static storage: cudart is linked statically, so a destructor run at process exit may find it torn down.
template <typename T>
struct DevBuf {   // grow-only device scratch
  T* p = nullptr; size_t n = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), n(o.n) { o.p = nullptr; o.n = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) { release(); p = o.p; n = o.n; o.p = nullptr; o.n = 0; }
    return *this;
  }
  ~DevBuf() { release(); }
  cudaError_t reserve(size_t want) {
    if (want <= n) return cudaSuccess;
    release();
    cudaError_t e = cudaMalloc(&p, want * sizeof(T));
    if (e == cudaSuccess) n = want; else { p = nullptr; cudaGetLastError(); }   // not left behind for a later launch check
    return e;
  }
  // Grows to max(need, 2 n) elements keeping the first `used`, copied on s and waited for.
  cudaError_t grow_keep(size_t need, size_t used, cudaStream_t s) {
    if (need <= n) return cudaSuccess;
    DevBuf<T> nb;
    cudaError_t e = nb.reserve(std::max(need, 2 * n));
    if (e == cudaSuccess && used) e = cudaMemcpyAsync(nb.p, p, used * sizeof(T), cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e == cudaSuccess) *this = std::move(nb);
    return e;
  }
  void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
};
// A device array that grows without moving (CUDA virtual memory management): open() reserves an address range for the
// most bytes it may ever hold and maps physical memory over its first `bytes`; grow() maps more at the end.  Every
// growth is one physical allocation, so shrink_to() a size the range had before unmaps exactly the later ones.  Only
// the owning device has access; the range is never exported or peer-mapped.  Failures come back as cudaError_t
// (cudaErrorMemoryAllocation when the device or the reserved range has no room) and leave the range as it was.
class VmmRange {
 public:
  VmmRange() = default;
  VmmRange(const VmmRange&) = delete;
  VmmRange& operator=(const VmmRange&) = delete;
  VmmRange(VmmRange&& o) noexcept { *this = std::move(o); }
  VmmRange& operator=(VmmRange&& o) noexcept {
    if (this != &o) {
      release();
      base_ = o.base_; reserved_ = o.reserved_; mapped_ = o.mapped_; gran_ = o.gran_; device_ = o.device_;
      chunks_ = std::move(o.chunks_);
      o.base_ = 0; o.reserved_ = o.mapped_ = 0; o.chunks_.clear();
    }
    return *this;
  }
  ~VmmRange() { release(); }
  cudaError_t open(int device, size_t max_bytes, size_t bytes);
  cudaError_t grow(size_t bytes);        // to at least `bytes` mapped
  void shrink_to(size_t bytes);          // back to a mapped size the range had before
  void* base() const { return reinterpret_cast<void*>(base_); }
  size_t mapped() const { return mapped_; }
 private:
  void release();
  unsigned long long base_ = 0;
  size_t reserved_ = 0, mapped_ = 0, gran_ = 0;
  int device_ = 0;
  struct Chunk { unsigned long long handle; size_t offset, bytes; };
  std::vector<Chunk> chunks_;            // in address order
};
constexpr int64_t kMaxRows = 0x7FFFFFC0ll;   // rows of a shard or keyword store: every row index fits an int32
// The most rows of row_bytes each that the current device's memory could hold, at most kMaxRows: the address room of a
// per-row array, so that it can grow as far as the device lets it without moving.
cudaError_t vmm_max_rows(size_t row_bytes, size_t* out);
// A per-row array on a VmmRange: n elements mapped at p, which never changes once open() succeeded.
template <typename T>
struct VmmBuf {
  T* p = nullptr; size_t n = 0;
  VmmRange r;
  VmmBuf() = default;
  VmmBuf(VmmBuf&& o) noexcept : p(o.p), n(o.n), r(std::move(o.r)) { o.p = nullptr; o.n = 0; }
  VmmBuf& operator=(VmmBuf&& o) noexcept {
    if (this != &o) { r = std::move(o.r); p = o.p; n = o.n; o.p = nullptr; o.n = 0; }
    return *this;
  }
  // row_elems elements a row; address room for vmm_max_rows of them, `rows` mapped.  The device is current.
  cudaError_t open(int device, size_t row_elems, size_t rows) {
    const size_t rb = row_elems * sizeof(T);
    size_t max_rows = 0;
    cudaError_t e = vmm_max_rows(rb, &max_rows);
    if (e == cudaSuccess) e = r.open(device, std::max(max_rows, rows) * rb, rows * rb);
    if (e == cudaSuccess) { p = static_cast<T*>(r.base()); n = r.mapped() / sizeof(T); }
    return e;
  }
  cudaError_t grow(size_t want) {   // to at least `want` elements
    const cudaError_t e = r.grow(want * sizeof(T));
    n = r.mapped() / sizeof(T);
    return e;
  }
  void shrink_to_bytes(size_t bytes) { r.shrink_to(bytes); n = r.mapped() / sizeof(T); }
};

template <typename T>
struct HostBuf {  // grow-only page-locked host buffer; flags: cudaHostAlloc's, per call site
  T* p = nullptr; size_t n = 0;
  HostBuf() = default;
  HostBuf(const HostBuf&) = delete;
  HostBuf& operator=(const HostBuf&) = delete;
  HostBuf(HostBuf&& o) noexcept : p(o.p), n(o.n) { o.p = nullptr; o.n = 0; }
  HostBuf& operator=(HostBuf&& o) noexcept {
    if (this != &o) { release(); p = o.p; n = o.n; o.p = nullptr; o.n = 0; }
    return *this;
  }
  ~HostBuf() { release(); }
  cudaError_t reserve(size_t want, unsigned flags) {
    if (want <= n) return cudaSuccess;
    release();
    cudaError_t e = cudaHostAlloc(reinterpret_cast<void**>(&p), want * sizeof(T), flags);
    if (e == cudaSuccess) n = want; else { p = nullptr; cudaGetLastError(); }
    return e;
  }
  void release() { if (p) cudaFreeHost(p); p = nullptr; n = 0; }
};
struct Stream {
  cudaStream_t s = nullptr;
  Stream() = default;
  Stream(const Stream&) = delete;
  Stream& operator=(const Stream&) = delete;
  Stream(Stream&& o) noexcept : s(o.s) { o.s = nullptr; }
  Stream& operator=(Stream&& o) noexcept { std::swap(s, o.s); return *this; }
  ~Stream() { if (s) cudaStreamDestroy(s); }
  cudaError_t create(unsigned flags, int priority = 0) {
    const cudaError_t e = cudaStreamCreateWithPriority(&s, flags, priority);
    if (e != cudaSuccess) { s = nullptr; cudaGetLastError(); }
    return e;
  }
  operator cudaStream_t() const { return s; }
};
struct Event {
  cudaEvent_t ev = nullptr;
  Event() = default;
  Event(const Event&) = delete;
  Event& operator=(const Event&) = delete;
  Event(Event&& o) noexcept : ev(o.ev) { o.ev = nullptr; }
  Event& operator=(Event&& o) noexcept { std::swap(ev, o.ev); return *this; }
  ~Event() { if (ev) cudaEventDestroy(ev); }
  cudaError_t create(unsigned flags = cudaEventDefault) {
    const cudaError_t e = cudaEventCreateWithFlags(&ev, flags);
    if (e != cudaSuccess) { ev = nullptr; cudaGetLastError(); }
    return e;
  }
  operator cudaEvent_t() const { return ev; }
};
// Returns expr's cudaError_t from the enclosing function unless it is cudaSuccess.
#define AUR_CU_RET(expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) return e_; } while (0)
// Returns from the enclosing C-ABI function unless expr is cudaSuccess: AUR_ERR_NOMEM for a failed allocation, else
// AUR_ERR_CUDA, with the expression, the error and where it failed as the message.
#define AUR_TRY(expr)                                                                                                    \
  do {                                                                                                                   \
    cudaError_t e_ = (expr);                                                                                             \
    if (e_ != cudaSuccess)                                                                                               \
      return ::aur::report_error(e_ == cudaErrorMemoryAllocation ? AUR_ERR_NOMEM : AUR_ERR_CUDA, "%s: %s (%s:%d)", #expr, \
                                 cudaGetErrorString(e_), __FILE__, __LINE__);                                            \
  } while (0)

// Per-call contexts (stream, events, grow-only scratch) of one device, pooled so that calls on several host threads
// each run on their own.  lease() hands out an idle context, or builds one with T::init(device) (which reports its own
// error) when none is idle.  Every context lives as long as the pool; T has a `stream`.
template <typename T> class CtxPool;
// One context taken from a pool for one call.  Its destructor makes the pool's device current, waits for the context's
// stream and only then gives the context back, so a context is never reused while work that reads its scratch is still
// in flight, on success or on an error.  A lease declared after the lock the call holds (a shard's or store's shared
// lock) is destroyed before that lock: the stream is idle before the lock is released.
template <typename T>
class CtxLease {
 public:
  CtxLease() = default;
  CtxLease(const CtxLease&) = delete;
  CtxLease& operator=(const CtxLease&) = delete;
  ~CtxLease() {
    if (!c_) return;
    cudaSetDevice(pool_->device);
    cudaStreamSynchronize(c_->stream);
    pool_->give_back(c_);
  }
  T* operator->() const { return c_; }
  operator T*() const { return c_; }
 private:
  friend class CtxPool<T>;
  CtxPool<T>* pool_ = nullptr;
  T* c_ = nullptr;
};
template <typename T>
class CtxPool {
 public:
  int device = 0;   // set before the first lease
  // An idle context or a new one into *out (empty); AUR_OK or T::init's error.
  int lease(CtxLease<T>* out) {
    out->pool_ = this;
    {
      std::lock_guard<std::mutex> lk(mu_);
      if (!idle_.empty()) { out->c_ = idle_.back(); idle_.pop_back(); return AUR_OK; }
    }
    std::unique_ptr<T> c(new T());
    const int rc = c->init(device);
    if (rc != AUR_OK) return rc;
    std::lock_guard<std::mutex> lk(mu_);
    out->c_ = c.get();
    all_.push_back(std::move(c));
    return AUR_OK;
  }
  std::vector<T*> contexts() {   // every context made so far, leased or idle
    std::lock_guard<std::mutex> lk(mu_);
    std::vector<T*> v;
    for (auto& c : all_) v.push_back(c.get());
    return v;
  }
 private:
  friend class CtxLease<T>;
  void give_back(T* c) {
    std::lock_guard<std::mutex> lk(mu_);
    idle_.push_back(c);
  }
  std::mutex mu_;
  std::vector<std::unique_ptr<T>> all_;
  std::vector<T*> idle_;
};

// ---------------------------------------------------------------- filter columns and uploads, host side (filter.cu)
// The attribute columns of a vector shard or a keyword store (program columns 2..): `rows` int32 codes each, -1 =
// absent.  A column only goes from unallocated to allocated, and grows in place (VmmBuf): its address never changes.
// write, any, grow, gather and clear are the holder's writes, serialised by its writers' lock; mu guards the columns
// write stores against check and fill.
class AttrColumns {
 public:
  // pairs (row, code) into column col (2 .. kFiltCols - 1), waited for; the first write allocates it, all -1.
  int write(int32_t col, const std::vector<int32_t>& pairs, int64_t rows, cudaStream_t s);
  bool any();
  // Every set column from old_rows to rows, the new rows -1, waited for; on a failure every column is as it was.
  cudaError_t grow(int64_t old_rows, int64_t rows, cudaStream_t s);
  // Compaction, every set column: rows map[0 .. m) to rows [dst0, dst0 + m) through bounce [m]; rows [r0, r1) to -1.
  cudaError_t gather(const int32_t* map, int64_t m, int64_t dst0, int32_t* bounce, cudaStream_t s);
  cudaError_t clear(int64_t r0, int64_t r1, cudaStream_t s);
  int check(const FiltProgs& fp, const char* holder);   // every column fp (structure checked) names is set
  void fill(FiltParams* p);                             // p->cols[2 ..]
 private:
  std::mutex mu;
  VmmBuf<int32_t> d_attr[kFiltAttrCols];
  DevBuf<int32_t> stage;
};
// Checked programs into stage on s in one upload (pageable: staged on return), and *p reading them over the holder's
// tenant codes and attribute columns.  *p spans every program: launch filter_pass(*p, ps), liveness and n_rows set.
cudaError_t filter_upload(const FiltProgs& fp, const int32_t* user, const int32_t* org, AttrColumns& attrs,
                          DevBuf<int32_t>& stage, cudaStream_t s, FiltParams* p);
inline FiltParams filter_pass(FiltParams p, int ps) { p.n_programs = filter_pass_programs(p.n_programs, ps); p.prog_off += ps * kFiltMaxPrograms; return p; }
// ---------------------------------------------------------------- the two legs of a hybrid query (hybrid.cu)
// Dense legs: every host search of a vector shard (aur_search, aur_search_ex, aur_search_subset, aur_search_lists,
// aur_search_filtered and the hybrid query's dense legs) over shards[0 .. n) (distinct, arguments checked), each shard's
// part on a search context leased from its shard's pool and that context's stream, over the prefix published when the
// part began.  q holds the host queries and at most one scope: tenant codes (nullable), allow-ids or per-query lists
// (n = 1 only), or checked programs with max_list_rows applied per shard.  Every shard's shared lock is taken in address
// order; with programs every shard's count pass is enqueued before any is waited on, and their read-back is the only
// host sync.  Then every shard's search is enqueued and then(legs) runs with every shard's (device, stream, top-k lists
// [nq * k] in device memory, valid once the stream reaches them, snapshot, matching rows per program) while the shards'
// shared locks and leases are held; each lease (CtxLease) drains its stream before its shard's lock is released, also
// on an error, so the streams are idle again before this returns.  aur_stats.last_* of each shard describe its part.
// scores_host / ids_host (n = 1, nullable): the caller's host outputs; when both are page-locked and mapped, the search
// writes its lists straight into them (DenseLeg.direct) instead of into device staging.  (capi.cu)
struct DenseQuery {
  const void* queries; int32_t nq, k;
  const int32_t* q_user = nullptr; const int32_t* q_org = nullptr;        // tenant codes [nq]
  const int64_t* allow_ids = nullptr; int64_t n_allow = -1;               // allow-ids (n_allow >= 0)
  const int64_t* list_ids = nullptr; const int64_t* list_offsets = nullptr; int32_t n_lists = 0;
  const int32_t* q_list = nullptr;                                        // per-query lists (q_list non-NULL)
  const FiltProgs* fp = nullptr; int64_t max_list_rows = 0;               // programs (fp non-NULL)
};
struct DenseLeg { int device; cudaStream_t stream; const float* scores; const int64_t* ids; int64_t snapshot_rows;
                  const std::vector<int64_t>* matched; bool direct; };
using DenseLegsThen = std::function<int(const std::vector<DenseLeg>& legs)>;
int dense_legs(aur_index* const* shards, int n, const DenseQuery& q, const DenseLegsThen& then, float* scores_host = nullptr,
               int64_t* ids_host = nullptr);
int index_device(const aur_index* ix);
int index_bf16_queries(const aur_index* ix);   // the index takes bf16 queries: bf16 or int8 rows
AttrColumns& index_attrs(aur_index* ix);
// Keyword legs: aur_kw_search_multi's search over stores[0 .. n) (distinct, non-NULL, 1 <= n <= 64) taken as one
// corpus, each store's part enqueued on its own context and stream; fp (nullable; programs checked, their columns set on
// every store) restricts query q to the live rows program fp->q_program[q] matches on each store, evaluated there
// (no allow-list, no read-back).  then(legs) runs with every
// store's (device, stream, top-k lists, snapshot) -- device arrays [nq * k], valid once the stream reaches them,
// sorted by (fp64 score desc, id asc) -- while every store's shared lock and every context are held.  Each store's
// aur_kw_stats.last_* are published after then() returns AUR_OK.  The query arguments are checked by kw_check.  (keyword.cu)
struct KwLeg { int device; cudaStream_t stream; const double* scores; const int64_t* ids; int64_t snapshot_rows; };
using KwLegsThen = std::function<int(const std::vector<KwLeg>& legs)>;
int kw_legs(aur_kw* const* stores, int n, const int32_t* q_terms, const int64_t* q_offsets, int32_t nq, int32_t k,
            const int32_t* q_user, const int32_t* q_org, const FiltProgs* fp, const KwLegsThen& then);
int kw_check(const int32_t* q_terms, const int64_t* q_offsets, int32_t nq, int32_t k);   // aur_kw_search's query checks
int kw_device(const aur_kw* kw);
AttrColumns& kw_attrs(aur_kw* kw);
// The store side of a text add (kw_text.cu): the rows of one batch as aur_kw_add publishes them.  Callers hold the
// store's mu_write (kw_write_mutex) and have checked the arguments and the room (kw_check_room).  land(dst, stream)
// enqueues the copy of the rows' total postings (term id, tf) to the store's device memory dst on the store's stream.
struct KwRows {
  const int64_t* ids; const int32_t* user; const int32_t* org;   // [n]; user / org nullable (0 / -1)
  const int64_t* offsets;    // [n + 1] from 0: row i's postings
  const int32_t* term_ids;   // [total] host copy of the postings' term ids (df)
  const int32_t* len;        // [n] document lengths (sum of tf)
  int64_t n, total; int32_t max_term;
};
using KwLand = std::function<cudaError_t(uint2* dst, cudaStream_t s)>;
int kw_check_room(aur_kw* kw, int64_t n);                         // AUR_ERR_NOMEM when n more rows do not fit
int kw_append_rows(aur_kw* kw, const KwRows& r, const KwLand& land);
void kw_after_append(aur_kw* kw, int rc);                         // the writer's index rebuild rule (index_due)
std::mutex& kw_write_mutex(aur_kw* kw);
int64_t kw_rows_appended(const aur_kw* kw);

// Opt kernel `kern` in to at least `smem` bytes of dynamic shared memory on the current device.  The limit is one
// setting per kernel and device, shared by every thread that launches it there: it is only ever raised, under a lock,
// so a launch asking for less never lowers it under a concurrent launch that needs more, and a kernel first launched
// on one device is still opted in on every other.  (capi.cu)
cudaError_t raise_smem_limit(const void* kern, size_t smem);

// Error reporting shared by the translation units behind the C ABI (thread-local message).
int report_error(int code, const char* fmt, ...);
// 2-D bf16 tensor map, 128-byte swizzle; returns 0 or a CUresult.
int encode_tmap_2d_bf16(void* tmap, const void* base, uint64_t cols, uint64_t rows, uint64_t row_stride_bytes,
                        uint32_t box_cols, uint32_t box_rows);
// The same over uint8 elements (an int8 shard's rows).
int encode_tmap_2d_u8(void* tmap, const void* base, uint64_t cols, uint64_t rows, uint64_t row_stride_bytes,
                      uint32_t box_cols, uint32_t box_rows);

}  // namespace aur
