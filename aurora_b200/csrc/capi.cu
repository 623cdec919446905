// Host runtime + C ABI (include/aurora_b200.h).  Owns one corpus shard in HBM:
//   rows      [capacity, dim]  bf16 or f32, row-major (K-major for the MMA, 128-bit
//                              coalesced for everything else)
//   inv_norm  [capacity] f32   1/|row|; 0 for zero rows; NaN marks a tombstone
//   ids       [capacity] i64   caller ids;  user / org [capacity] i32 tenant codes
//   attr      up to 16 x [capacity] i32 attribute codes for device-evaluated filters (allocated on first aur_set_attrs)
// plus grow-only scratch for candidate lists.  No CPU compute path exists here: without
// a CUDA device every entry point fails with AUR_ERR_NO_DEVICE.
//
// Concurrency (BASELINE config 5: streaming ingest while queries run; the reference's callers are 8 gunicorn
// threads + 4 Celery children, docker-compose.yaml:191,283-285).  The shard is append-only with a PUBLISHED row
// count: a writer copies rows / ids / tenant codes / inverse norms into [rows_pub, rows_pub + n) on the ingest
// stream, waits for them to land, and only then stores rows_pub + n (release).  A search loads rows_pub once
// (acquire) when it is enqueued and scans exactly that prefix -- rows behind it are masked by the kernels' own
// n_rows bound -- so every answer is the top-k of a consistent prefix, which it can report
// (aur_search_ex).  Searches never take the writers' lock; each in-flight search owns a SearchCtx (candidate
// lists, threshold-exchange table, staging buffers, events, stream), so several can be enqueued at once.
// Compaction and export are the only exclusive operations.
#include <cuda.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <atomic>
#include <memory>
#include <mutex>
#include <shared_mutex>
#include <string>
#include <unordered_map>
#include <algorithm>
#include <vector>

#include "../../include/aurora_b200.h"
#include "internal.h"

using namespace aur;

namespace {

thread_local std::string g_err;

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

}  // namespace

namespace aur {
int report_error(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
  g_err = buf;
  return code;
}
int encode_tmap_2d_bf16(void* tmap, const void* base, uint64_t cols, uint64_t rows, uint64_t row_stride_bytes,
                        uint32_t box_cols, uint32_t box_rows) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return -1;
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {row_stride_bytes};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  return static_cast<int>(enc(static_cast<CUtensorMap*>(tmap), CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
                              const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                              CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE));
}
}  // namespace aur

namespace {
int (&fail)(int, const char*, ...) = report_error;
#define CU_TRY(expr)                                                                               \
  do {                                                                                             \
    cudaError_t e_ = (expr);                                                                       \
    if (e_ != cudaSuccess) return fail(AUR_ERR_CUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(e_), \
                                       __FILE__, __LINE__);                                        \
  } while (0)
}  // namespace

// Scratch and bookkeeping of ONE in-flight search.  Device-pointer searches are bound to the caller's stream
// (same stream -> same context -> stream order protects the scratch); host-buffer searches take a context from a
// pool and run on its own stream, so N threads can search at once.
struct SearchCtx {
  std::mutex mu;                  // one enqueue at a time
  cudaStream_t own_stream = nullptr;
  cudaStream_t bound = nullptr;   // caller stream this context serves (nullptr = pool context)
  cudaEvent_t ev_begin = nullptr, ev_k0 = nullptr, ev_k1 = nullptr, ev_fin = nullptr, ev_end = nullptr;
  bool have_timing = false;
  int last_kernel = 0, last_launches = 0, last_nq = 0;
  int last_tile_n = 0;             // corpus rows per tile of the last tensor-core launch (0: none)
  int64_t snapshot_rows = 0;
  uint32_t epoch = 0;
  DevBuf<uint64_t> cand_a, cand_b;
  DevBuf<uint64_t> pub;          // tensor-core kernel's cross-CTA threshold exchange
  DevBuf<uint32_t> cand_count;   // compacted candidates per query (self-resetting)
  DevBuf<uint32_t> d_epoch;      // the tensor-core kernel's launch counter, device resident (CUDA-graph replays advance it)
  DevBuf<uint32_t> cand_read;    // per query of the last search: candidate keys its exact re-rank read
  DevBuf<float> score_chunk;
  DevBuf<float> masked_inv;      // inverse norms with the invisible rows turned into NaN (tenant scope / id subset)
  DevBuf<int32_t> allow_rows;    // subset search: rows that stay visible
  DevBuf<uint32_t> row_mask;     // per-query tenant scopes on the tensor path: bit s = scope s of the batch sees the row
  DevBuf<int32_t> scope_tab, q_scope;   // the batch's distinct {user, org} scopes (<= 32) and every query's scope index
  DevBuf<uint8_t> stage_q;       // host-entry staging: queries
  DevBuf<int32_t> stage_quser, stage_qorg;
  DevBuf<float> stage_scores;
  DevBuf<int64_t> stage_ids;
  DevBuf<int32_t> list_stage;    // list search: work items, their queries and the lists' resolved rows (one upload)
  DevBuf<float> list_scores;     // list search: scores of a batch of work items, [slots][kSimtSeg]
  DevBuf<int32_t> filt_stage;    // filtered search: the programs' tokens, offsets and bitmaps (one upload)
  DevBuf<uint32_t> filt_mask;    // filtered search: per row, bit q = program q matches
  DevBuf<uint32_t> filt_counts;  // filtered search: [32] totals, then [n_programs][blocks] counts (scanned into offsets)
  DevBuf<int32_t> filt_rows;     // filtered search: every program's matching rows, ascending, program after program
  DevBuf<int64_t> filt_ids;      // aur_filter_ids: their ids
  void release() {
    cand_a.release(); cand_b.release(); pub.release(); cand_count.release(); d_epoch.release(); cand_read.release(); score_chunk.release(); masked_inv.release();
    allow_rows.release(); row_mask.release(); scope_tab.release(); q_scope.release(); stage_q.release(); stage_quser.release(); stage_qorg.release(); stage_scores.release();
    stage_ids.release(); list_stage.release(); list_scores.release();
    filt_stage.release(); filt_mask.release(); filt_counts.release(); filt_rows.release(); filt_ids.release();
    if (ev_begin) cudaEventDestroy(ev_begin);
    if (ev_k0) cudaEventDestroy(ev_k0);
    if (ev_k1) cudaEventDestroy(ev_k1);
    if (ev_fin) cudaEventDestroy(ev_fin);
    if (ev_end) cudaEventDestroy(ev_end);
    if (own_stream) cudaStreamDestroy(own_stream);
  }
};

struct aur_index {
  std::shared_mutex rw;          // shared: searches and appends; exclusive: compaction, export, close
  std::mutex mu;                 // host metadata: id2row, live, options, the context pool
  std::mutex mu_write;           // one writer at a time (append / remove)
  int device = 0, dim = 0, dtype = 0;
  int64_t capacity = 0, live = 0;
  int64_t cap_pad = 0;                // capacity rounded up to a whole tile (TMA boxes never straddle an allocation):
                                      // the length of every per-row array
  std::atomic<int64_t> rows_pub{0};   // rows visible to searches (published after the data landed)
  size_t elt = 2;
  void* d_rows = nullptr;
  float* d_inv_norm = nullptr;
  int64_t* d_ids = nullptr;
  int32_t* d_user = nullptr;
  int32_t* d_org = nullptr;
  int32_t* d_attr[kFiltAttrCols] = {};   // attribute columns (program columns 2..), allocated on first aur_set_attrs; guarded by mu
  DevBuf<int32_t> attr_stage;            // aur_set_attrs: (row, code) pairs (writers hold mu_write)
  std::unordered_map<int64_t, int64_t> id2row;
  cudaStream_t stream = nullptr;         // the index's own stream: device-pointer calls with stream == NULL
  cudaStream_t ingest_stream = nullptr;  // host appends / tombstones, lowest priority so queries overtake them
  CUtensorMap tmap[2][2];  // [64-row, 128-row tiles][cta_group 1, 2]: box rows tile / cta_group
  bool tmap_ok = false;
  int sm_count = 0;
  size_t smem_optin = 0;
  int opt_kernel = AUR_KERNEL_AUTO;
  int opt_dbg_flags = 0;
  int opt_tc_tile = 0;           // corpus rows per tile: 0 = auto, 64, 128
  std::atomic<uint32_t> opt_dbg_epoch{0};   // bring-up: start value of the contexts' launch counters (0 = 1)
  std::vector<std::unique_ptr<SearchCtx>> ctxs;
  std::vector<SearchCtx*> free_ctxs;   // idle pool contexts
  SearchCtx* last_ctx = nullptr;       // context of the most recently enqueued search (aur_get_stats)
};

namespace {

int build_tmaps(aur_index* ix) {
  ix->tmap_ok = false;
  if (ix->dtype != AUR_BF16 || ix->dim % kTcKBlock != 0 || ix->dim > kTcMaxDim) return AUR_OK;  // SIMT only
  // rows past the capacity (a tile's tail, a whole half of the last tile of a pair) arrive as zeros
  for (int w = 0; w < 2; ++w)
    for (int g = 1; g <= 2; ++g) {
      const int tile_n = w ? kTcTileWide : kTcTileN;
      const int r = encode_tmap_2d_bf16(&ix->tmap[w][g - 1], ix->d_rows, static_cast<uint64_t>(ix->dim),
                                        static_cast<uint64_t>(ix->capacity), static_cast<uint64_t>(ix->dim) * 2, kTcKBlock,
                                        static_cast<uint32_t>(tile_n / g));
      if (r < 0) return fail(AUR_ERR_CUDA, "cuTensorMapEncodeTiled entry point not found");
      if (r != CUDA_SUCCESS) return fail(AUR_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d)", r);
    }
  ix->tmap_ok = true;
  return AUR_OK;
}

bool tc_shape_ok(const aur_index* ix, int k, bool filtered) {
  if (!ix->tmap_ok || filtered || k > kMaxK) return false;
  // candidate lists (k + slack per query) and the query block share the SM's shared memory with
  // the TMA ring: large k at large dim leaves no room for a pipeline
  return tc_pick_stages(k + kSlack, ix->dim, ix->smem_optin, kTcTileN, true) >= 2;
}

int ctx_init(SearchCtx* c) {
  int lo = 0, hi = 0;
  CU_TRY(cudaDeviceGetStreamPriorityRange(&lo, &hi));   // hi = numerically lowest = highest priority
  CU_TRY(cudaStreamCreateWithPriority(&c->own_stream, cudaStreamNonBlocking, hi));
  CU_TRY(cudaEventCreate(&c->ev_begin)); CU_TRY(cudaEventCreate(&c->ev_k0));
  CU_TRY(cudaEventCreate(&c->ev_k1));    CU_TRY(cudaEventCreate(&c->ev_end));
  CU_TRY(cudaEventCreate(&c->ev_fin));
  return AUR_OK;
}

// Context for a search on the caller's stream `s` (bound) or, with s == nullptr, an idle pool context.
int acquire_ctx(aur_index* ix, cudaStream_t s, SearchCtx** out) {
  std::lock_guard<std::mutex> lk(ix->mu);
  if (s) {
    for (auto& c : ix->ctxs)
      if (c->bound == s) { *out = c.get(); return AUR_OK; }
  } else if (!ix->free_ctxs.empty()) {
    *out = ix->free_ctxs.back(); ix->free_ctxs.pop_back();
    return AUR_OK;
  }
  std::unique_ptr<SearchCtx> c(new SearchCtx());
  int rc = ctx_init(c.get());
  if (rc != AUR_OK) { c->release(); return rc; }
  c->bound = s;
  *out = c.get();
  ix->ctxs.push_back(std::move(c));
  return AUR_OK;
}
void release_ctx(aur_index* ix, SearchCtx* c) {
  std::lock_guard<std::mutex> lk(ix->mu);
  if (!c->bound) ix->free_ctxs.push_back(c);
}

// Pinned caller buffers are mapped into the device's address space (UVA): the re-rank kernel then writes its nq x k
// results straight into them over PCIe and the two device-to-host copies (a launch + ~8 us of latency each) disappear.
// Returns whether *d_scores / *d_ids now point at the caller's buffers (else they keep the staging buffers).
bool direct_outputs(float* scores_out, int64_t* ids_out, float** d_scores, int64_t** d_ids) {
  cudaPointerAttributes as{}, ai{};
  if (cudaPointerGetAttributes(&as, scores_out) == cudaSuccess && cudaPointerGetAttributes(&ai, ids_out) == cudaSuccess &&
      as.type == cudaMemoryTypeHost && ai.type == cudaMemoryTypeHost && as.devicePointer && ai.devicePointer) {
    *d_scores = static_cast<float*>(as.devicePointer);
    *d_ids = static_cast<int64_t*>(ai.devicePointer);
    return true;
  }
  cudaGetLastError();
  return false;
}

// One call with host buffers: the index's shared lock, its device, an idle pool context locked for the call and given
// back when the call ends, the context's own stream, and the prefix published when the call began (open()).  A search
// call stages its queries and outputs with stage() and ends with finish().
struct HostCall {
  aur_index* ix;
  std::shared_lock<std::shared_mutex> rl;
  SearchCtx* c = nullptr;
  std::unique_lock<std::mutex> cl;
  cudaStream_t s = nullptr;
  int64_t n_rows = 0;
  float* d_scores = nullptr;   // where the search writes its results: the caller's pinned buffers or the staging buffers
  int64_t* d_ids = nullptr;
  bool direct = false;

  explicit HostCall(aur_index* index) : ix(index), rl(index->rw) {}
  HostCall(const HostCall&) = delete;
  HostCall& operator=(const HostCall&) = delete;
  ~HostCall() {
    if (!c) return;
    cl.unlock();
    release_ctx(ix, c);
  }
  int open() {
    CU_TRY(cudaSetDevice(ix->device));
    const int rc = acquire_ctx(ix, nullptr, &c);
    if (rc != AUR_OK) return rc;
    cl = std::unique_lock<std::mutex>(c->mu);
    s = c->own_stream;
    n_rows = ix->rows_pub.load(std::memory_order_acquire);
    return AUR_OK;
  }
  // Uploads the queries to c->stage_q and picks the outputs (direct_outputs).
  int stage(const void* queries_host, int32_t nq, int32_t k, float* scores_out, int64_t* ids_out) {
    const size_t qbytes = static_cast<size_t>(nq) * ix->dim * ix->elt;
    const size_t nout = static_cast<size_t>(nq) * k;
    CU_TRY(c->stage_q.reserve(qbytes));
    CU_TRY(c->stage_scores.reserve(nout));
    CU_TRY(c->stage_ids.reserve(nout));
    CU_TRY(cudaMemcpyAsync(c->stage_q.p, queries_host, qbytes, cudaMemcpyHostToDevice, s));
    d_scores = c->stage_scores.p;
    d_ids = c->stage_ids.p;
    direct = direct_outputs(scores_out, ids_out, &d_scores, &d_ids);
    return AUR_OK;
  }
  // Ends a search whose enqueue returned rc.  The caller's buffers are written only when every kernel of the search was
  // enqueued successfully; on any failure the stream drains and they are left untouched.
  int finish(int rc, int32_t nq, int32_t k, float* scores_out, int64_t* ids_out) {
    if (rc != AUR_OK) { cudaStreamSynchronize(s); return rc; }
    if (!direct) {   // into the caller's pageable buffers
      const size_t nout = static_cast<size_t>(nq) * k;
      CU_TRY(cudaMemcpyAsync(scores_out, c->stage_scores.p, nout * 4, cudaMemcpyDeviceToHost, s));
      CU_TRY(cudaMemcpyAsync(ids_out, c->stage_ids.p, nout * 8, cudaMemcpyDeviceToHost, s));
    }
    CU_TRY(cudaStreamSynchronize(s));
    return AUR_OK;
  }
};

// Calls f(i, row) for every ids[i] (i < n) that names a row of the prefix [0, n_rows); unknown and newer ids drop out.
template <typename F>
void resolve_ids(aur_index* ix, const int64_t* ids, int64_t n, int64_t n_rows, F&& f) {
  std::lock_guard<std::mutex> lk(ix->mu);
  for (int64_t i = 0; i < n; ++i) {
    auto it = ix->id2row.find(ids[i]);
    if (it != ix->id2row.end() && it->second < n_rows) f(i, static_cast<int32_t>(it->second));
  }
}

// Corpus rows per tile when the index leaves it to the launch.  A 128-row tile (wgmma m64n128) fetches each operand for
// twice the work of a 64-row one, but its layout leaves fewer, larger ring stages: it runs with at least
// kTcWideMinStages stages, so at dim 1024, at large k and for most tenant-scoped batches the 64-row kernel stays.  The
// bring-up score dump (dbg) keeps the 64-row tile it documents.
int tc_auto_tile(int ksel, int dim, size_t smem_optin, bool mask, bool dbg) {
  if (dbg) return kTcTileN;
  return tc_pick_stages(ksel, dim, smem_optin, kTcTileWide, mask) >= kTcWideMinStages ? kTcTileWide : kTcTileN;
}

// Query super-blocks of a two-CTA launch (CTA pairs of 128 queries each that walk the same tiles side by side, sharing
// them through L2): at most `want`, fewer while the threshold exchange would need more than ceil(ksel / tile sets) = 4
// rows vouched for per CTA.
int tc2_super_blocks(const aur_index* ix, int ksel, int want) {
  const int pairs = ix->sm_count / 2;
  int n_super = want;
  while (n_super > 1 && (ksel + pairs / n_super - 1) / (pairs / n_super) > 4) --n_super;
  return n_super;
}

// Runs one block of queries (<= 128 single CTAs, <= 512 pairs) through the tensor-core kernel over the first n_rows rows.  Leaves candidate keys
// in c->cand_a as [nqb_pad, n_lists, ksel]; returns n_lists.
int run_tc_block(aur_index* ix, SearchCtx* c, int cta_group, const void* q_dev, int nqb, int ksel, int64_t n_rows, float* dbg,
                 int* n_lists_out, cudaStream_t s, const float* inv_norm = nullptr, const uint32_t* row_mask = nullptr,
                 const int32_t* q_scope = nullptr) {
  int n_qblocks = (nqb > kTcQRows) ? 2 : 1;
  if (cta_group == 2 && nqb <= kTcQRows) cta_group = 1;   // a pair works on 128 query rows: a short tail runs as single CTAs
  const int pairs = ix->sm_count / 2;
  int n_super = 1;
  if (cta_group == 2) {
    n_super = tc2_super_blocks(ix, ksel, (nqb + 2 * kTcQRows - 1) / (2 * kTcQRows));
    if (nqb > n_super * 2 * kTcQRows) return fail(AUR_ERR_INVALID, "internal: query block larger than the launch geometry");
    n_qblocks = 2 * n_super;
  }
  int grid = (cta_group == 2) ? (pairs / n_super) * n_super * 2 : (ix->sm_count & ~1);
  const int n_lists = (cta_group == 2) ? pairs / n_super : grid / n_qblocks;   // tile sets = candidate lists per query
  const bool mask = row_mask != nullptr;
  int tile_n = ix->opt_tc_tile;
  if (tile_n == 0) tile_n = tc_auto_tile(ksel, ix->dim, ix->smem_optin, mask, dbg != nullptr);
  const int stages = tc_pick_stages(ksel, ix->dim, ix->smem_optin, tile_n, mask);
  if (stages < 2) return fail(AUR_ERR_UNSUPPORTED, "k too large for the tensor-core path's shared memory");
  const size_t smem = tc_smem_bytes(stages, ksel, ix->dim, tile_n, mask);
  const size_t ncand = static_cast<size_t>(n_qblocks) * kTcQRows * n_lists * ksel;
  CU_TRY(c->cand_a.reserve(ncand));
  const size_t npub = static_cast<size_t>(n_qblocks) * kTcQRows * (((n_lists + 1) & ~1) + 1);
  if (npub > c->pub.n) {
    CU_TRY(c->pub.reserve(npub));
    CU_TRY(cudaMemsetAsync(c->pub.p, 0, npub * 8, s));  // epoch 0 is never used by a launch
  }
  if (c->cand_count.n < 8 * kTcQRows) {
    CU_TRY(c->cand_count.reserve(8 * kTcQRows));
    CU_TRY(cudaMemsetAsync(c->cand_count.p, 0, 8 * kTcQRows * 4, s));
  }
  if (c->d_epoch.n == 0) {
    const uint32_t e0 = ix->opt_dbg_epoch.load() ? ix->opt_dbg_epoch.load() : 1u;
    CU_TRY(c->d_epoch.reserve(1));
    CU_TRY(cudaMemcpyAsync(c->d_epoch.p, &e0, 4, cudaMemcpyHostToDevice, s));   // pageable source: staged before return
  }
  ++c->epoch;
  TcParams p;
  p.q = static_cast<const __nv_bfloat16*>(q_dev);
  p.inv_norm = inv_norm ? inv_norm : ix->d_inv_norm;
  p.row_mask = row_mask; p.q_scope = q_scope;
  p.ids = ix->d_ids;
  p.cand = c->cand_a.p;
  p.cand_count = c->cand_count.p;
  p.dbg_scores = dbg;
  p.pub = c->pub.p;
  // searches: device-resident counter (1 .. kSearchEpochMax), advanced by the finalize kernel that follows; the bring-up
  // entry point (no finalize behind it) tags its entries from the disjoint upper half on the host
  p.epoch = (kSearchEpochMax + 1u) | c->epoch;
  p.epoch_ptr = dbg ? nullptr : c->d_epoch.p;
  p.n_rows = n_rows;
  p.nq = nqb; p.dim = ix->dim; p.ksel = ksel; p.n_lists = n_lists; p.n_qblocks = n_qblocks;
  p.num_stages = stages;
  p.dbg_flags = ix->opt_dbg_flags;
  p.n_tiles = static_cast<int>((n_rows + tile_n - 1) / tile_n);
  CU_TRY(tc_launch(cta_group, tile_n, grid, &ix->tmap[tile_n == kTcTileWide][cta_group - 1], p, smem, s));
  c->last_tile_n = tile_n;
  *n_lists_out = n_lists;
  return AUR_OK;
}

// Visibility of a search besides tombstones: per-query tenant codes (generic kernel), one tenant scope for the
// whole batch, or an explicit list of visible rows -- the last two fold into the row scale (NaN = invisible), so
// the tensor-core kernel serves them.
struct Scope {
  const int32_t* q_user = nullptr;       // device, per query (nullptr = no tenant filter)
  const int32_t* q_org = nullptr;
  const int32_t* uniform = nullptr;      // host {user, org}: every query of the batch carries this scope
  const int32_t* allow_rows = nullptr;   // device: rows that stay visible (subset search)
  int64_t n_allow = -1;                  // -1 = no subset
  const int32_t* scope_tab = nullptr;    // device [n_scopes][2]: the batch's distinct tenant scopes, when there are <= 32
  const int32_t* q_scope = nullptr;      // device [nq]: scope index of every query
  int n_scopes = 0;
  const uint32_t* match_mask = nullptr;  // device [n_rows]: rows with bit 0 set stay visible (a device-evaluated filter)
};

// Stats of one search call (aur_get_stats), kept on the context that runs it.  The call opens them with stats_begin
// (counters reset, ev_begin) and closes them with stats_end (ev_fin, ev_end; the context becomes the one aur_get_stats
// reads).  In between the search sets last_kernel, counts every launch in last_launches and brackets the main kernels
// of its first block of queries with ev_k0 / ev_k1.
int stats_begin(SearchCtx* c, cudaStream_t s, int nq, int64_t n_rows) {
  c->last_launches = 0;
  c->last_tile_n = 0;
  c->last_nq = nq;
  c->snapshot_rows = n_rows;
  CU_TRY(cudaEventRecord(c->ev_begin, s));
  return AUR_OK;
}
int stats_end(aur_index* ix, SearchCtx* c, cudaStream_t s) {
  CU_TRY(cudaEventRecord(c->ev_fin, s));
  CU_TRY(cudaEventRecord(c->ev_end, s));
  c->have_timing = true;
  std::lock_guard<std::mutex> lk(ix->mu);
  ix->last_ctx = c;
  return AUR_OK;
}

// The tail of one block of queries q0 .. q0 + nqb: its candidate lists [nqb, n_lists, ksel] in c->cand_a are folded
// until one sort of <= 4096 keys finishes them, then re-ranked exactly into the block's rows of the outputs.  compact:
// the tensor-core kernel already compacted its survivors per query (counted in c->cand_count), nothing to fold.
int candidate_tail(aur_index* ix, SearchCtx* c, cudaStream_t s, const void* qb, int q0, int nqb, int k, int n_lists, bool compact,
                   float* scores, int64_t* ids, double* scores64, const FinalizeArgs::ExchangeOut* ex) {
  const int ksel = k + kSlack;
  uint64_t* cur = c->cand_a.p;
  bool in_a = true;
  while (!compact && static_cast<int64_t>(n_lists) * ksel > 4096) {
    const int group = 4096 / ksel;
    const int n_groups = (n_lists + group - 1) / group;
    DevBuf<uint64_t>& dst = in_a ? c->cand_b : c->cand_a;
    // rows of cand are indexed by the query position inside the block (TC pads to 128/256)
    CU_TRY(dst.reserve(static_cast<size_t>(nqb) * n_groups * ksel));
    CU_TRY(launch_reduce_lists(cur, nqb, n_lists, ksel, group, ix->d_ids, dst.p, s));
    c->last_launches += 1;
    cur = dst.p; n_lists = n_groups; in_a = !in_a;
  }
  FinalizeArgs fa{};
  fa.cand = cur; fa.n_lists = n_lists; fa.ksel = ksel;
  fa.counts = compact ? c->cand_count.p : nullptr;
  fa.epoch_bump = compact ? c->d_epoch.p : nullptr;
  fa.cand_read = c->cand_read.p + q0;
  fa.q = qb; fa.rows = ix->d_rows; fa.dtype = ix->dtype; fa.dim = ix->dim; fa.nq = nqb; fa.k = k;
  fa.ids = ix->d_ids;
  fa.out_scores = scores ? scores + static_cast<size_t>(q0) * k : nullptr;
  fa.out_ids = ids ? ids + static_cast<size_t>(q0) * k : nullptr;
  fa.out_scores64 = scores64 ? scores64 + static_cast<size_t>(q0) * k : nullptr;
  if (ex) { fa.ex = *ex; fa.ex.q0 = q0; }
  CU_TRY(launch_finalize(fa, s));
  c->last_launches += 1;
  return AUR_OK;
}

// Enqueues one search over the published prefix `n_rows` on stream s using context c, inside the call's stats.
int search_enqueue(aur_index* ix, SearchCtx* c, const void* q_dev, int nq, int k, const Scope& sc, int64_t n_rows,
                   float* scores, int64_t* ids, double* scores64, cudaStream_t s,
                   const FinalizeArgs::ExchangeOut* ex = nullptr) {
  const bool subset = sc.n_allow >= 0;
  const bool scoped_tc = sc.n_scopes > 0 && !subset && sc.uniform == nullptr;        // per-query scopes through bit masks
  const bool filtered = sc.q_user != nullptr && sc.uniform == nullptr && !subset && !scoped_tc;   // else: generic kernel only
  const int ksel = k + kSlack;
  int kernel = ix->opt_kernel;
  if (kernel == AUR_KERNEL_AUTO) kernel = tc_shape_ok(ix, k, filtered) ? AUR_KERNEL_TC2 : AUR_KERNEL_SIMT;
  if (kernel != AUR_KERNEL_SIMT && !tc_shape_ok(ix, k, filtered))
    return fail(AUR_ERR_UNSUPPORTED, "tensor-core path needs bf16, dim %% 64 == 0, dim <= %d, no per-query tenant filter, and k small "
                "enough for its shared-memory lists at this dim", kTcMaxDim);
  c->last_kernel = kernel;
  CU_TRY(c->cand_read.reserve(static_cast<size_t>(nq)));
  bool k_timed = false;
  const float* inv = nullptr;   // masked inverse norms (nullptr = the shard's own)
  if (subset && n_rows > 0) {
    CU_TRY(c->masked_inv.reserve(static_cast<size_t>(ix->capacity) + 64));
    CU_TRY(launch_fill_f32(c->masked_inv.p, nanf(""), n_rows, s));
    CU_TRY(launch_scatter_inv_norm(ix->d_inv_norm, sc.allow_rows, sc.n_allow, n_rows, c->masked_inv.p, s));
    c->last_launches += 2;
    inv = c->masked_inv.p;
  } else if (sc.match_mask && n_rows > 0) {
    CU_TRY(c->masked_inv.reserve(static_cast<size_t>(ix->capacity) + 64));
    CU_TRY(launch_mask_match(ix->d_inv_norm, sc.match_mask, n_rows, c->masked_inv.p, s));
    ++c->last_launches;
    inv = c->masked_inv.p;
  } else if (kernel != AUR_KERNEL_SIMT && scoped_tc && n_rows > 0) {              // up to 32 scopes in the batch: row bit masks
    CU_TRY(c->row_mask.reserve(static_cast<size_t>(ix->capacity) + 64));
    CU_TRY(launch_row_scope_mask(ix->d_user, ix->d_org, sc.scope_tab, sc.n_scopes, n_rows, c->row_mask.p, s));
    ++c->last_launches;
  } else if (kernel != AUR_KERNEL_SIMT && sc.q_user != nullptr && sc.uniform != nullptr && n_rows > 0) {   // one scope for the whole batch
    CU_TRY(c->masked_inv.reserve(static_cast<size_t>(ix->capacity) + 64));
    CU_TRY(launch_mask_inv_norm(ix->d_inv_norm, ix->d_user, ix->d_org, sc.uniform[0], sc.uniform[1], n_rows, c->masked_inv.p, s));
    ++c->last_launches;
    inv = c->masked_inv.p;
  }

  // queries per launch: the generic kernel takes 1024; the tensor-core kernel 128 per CTA pair and up to four pairs side by
  // side on the same corpus tiles (fewer when k + slack is too large for the threshold exchange of that geometry)
  int qstep = 1024;
  if (kernel == AUR_KERNEL_TC1) qstep = 2 * kTcQRows;
  else if (kernel == AUR_KERNEL_TC2) qstep = tc2_super_blocks(ix, ksel, 4) * 2 * kTcQRows;
  for (int q0 = 0; q0 < nq; q0 += qstep) {
    const int nqb = (nq - q0 < qstep) ? nq - q0 : qstep;
    const uint8_t* qb = static_cast<const uint8_t*>(q_dev) + static_cast<size_t>(q0) * ix->dim * ix->elt;
    int n_lists = 0;
    if (kernel == AUR_KERNEL_SIMT) {
      if (n_rows == 0) {
        n_lists = 1;
        CU_TRY(c->cand_a.reserve(static_cast<size_t>(nqb) * ksel));
        CU_TRY(cudaMemsetAsync(c->cand_a.p, 0, static_cast<size_t>(nqb) * ksel * 8, s));
      } else {
        n_lists = static_cast<int>((n_rows + kSimtSeg - 1) / kSimtSeg);
        CU_TRY(c->cand_a.reserve(static_cast<size_t>(nqb) * n_lists * ksel));
        const int64_t chunk = 16 * kSimtSeg;  // 32768 rows of scores at a time
        CU_TRY(c->score_chunk.reserve(static_cast<size_t>(nqb) * chunk));
        FilterArgs f{ix->d_user, ix->d_org, nullptr, nullptr};
        if (!subset && sc.q_user && !inv) { f.q_user = sc.q_user + q0; f.q_org = sc.q_org ? sc.q_org + q0 : nullptr; }
        if (!k_timed) CU_TRY(cudaEventRecord(c->ev_k0, s));
        for (int64_t r0 = 0; r0 < n_rows; r0 += chunk) {
          const int64_t nr = (n_rows - r0 < chunk) ? n_rows - r0 : chunk;
          CU_TRY(launch_simt_scores(qb, ix->d_rows, ix->dtype, ix->dim, nqb, r0, nr, n_rows, inv ? inv : ix->d_inv_norm, f,
                                    c->score_chunk.p, s));
          CU_TRY(launch_simt_select(c->score_chunk.p, nqb, r0, nr, ksel, ix->d_ids, c->cand_a.p, n_lists,
                                    static_cast<int>(r0 / kSimtSeg), s));
          c->last_launches += 2;
        }
        if (!k_timed) { CU_TRY(cudaEventRecord(c->ev_k1, s)); k_timed = true; }
      }
    } else {
      if (!k_timed) CU_TRY(cudaEventRecord(c->ev_k0, s));
      const bool use_mask = scoped_tc && n_rows > 0;
      int rc = run_tc_block(ix, c, kernel == AUR_KERNEL_TC1 ? 1 : 2, qb, nqb, ksel, n_rows, nullptr, &n_lists, s, inv,
                            use_mask ? c->row_mask.p : nullptr, use_mask ? sc.q_scope + q0 : nullptr);
      if (rc != AUR_OK) return rc;
      if (!k_timed) { CU_TRY(cudaEventRecord(c->ev_k1, s)); k_timed = true; }
      c->last_launches += 1;
    }
    const int rc = candidate_tail(ix, c, s, qb, q0, nqb, k, n_lists, kernel != AUR_KERNEL_SIMT, scores, ids, scores64, ex);
    if (rc != AUR_OK) return rc;
  }
  if (!k_timed) { CU_TRY(cudaEventRecord(c->ev_k0, s)); CU_TRY(cudaEventRecord(c->ev_k1, s)); }
  return AUR_OK;
}

// Append n rows behind the published prefix and publish them once they have landed.  Caller holds mu_write.
int add_common(aur_index* ix, const void* rows, bool rows_on_device, const int64_t* ids, const int32_t* users,
               const int32_t* orgs, int64_t n, cudaStream_t s) {
  if (n < 0) return fail(AUR_ERR_INVALID, "n < 0");
  if (n == 0) return AUR_OK;
  if (!rows || !ids) return fail(AUR_ERR_INVALID, "rows and ids are required");
  const int64_t base = ix->rows_pub.load(std::memory_order_relaxed);   // writers are serialised: nobody else moves it
  if (base + n > ix->capacity)
    return fail(AUR_ERR_NOMEM, "shard full: %lld + %lld > capacity %lld (aur_compact reclaims tombstones)", (long long)base,
                (long long)n, (long long)ix->capacity);
  for (int64_t i = 0; i < n; ++i)
    if (ids[i] < 0) return fail(AUR_ERR_INVALID, "ids must be >= 0");
  uint8_t* dst = static_cast<uint8_t*>(ix->d_rows) + static_cast<size_t>(base) * ix->dim * ix->elt;
  CU_TRY(cudaMemcpyAsync(dst, rows, static_cast<size_t>(n) * ix->dim * ix->elt,
                         rows_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, s));
  CU_TRY(cudaMemcpyAsync(ix->d_ids + base, ids, static_cast<size_t>(n) * 8, cudaMemcpyHostToDevice, s));
  std::vector<int32_t> fill;
  if (!users) { fill.assign(static_cast<size_t>(n), 0); users = fill.data(); }
  CU_TRY(cudaMemcpyAsync(ix->d_user + base, users, static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, s));
  std::vector<int32_t> fill2;
  if (!orgs) { fill2.assign(static_cast<size_t>(n), -1); orgs = fill2.data(); }
  CU_TRY(cudaMemcpyAsync(ix->d_org + base, orgs, static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, s));
  CU_TRY(launch_row_inv_norms(dst, ix->dtype, ix->dim, n, ix->d_inv_norm + base, s));
  // upsert: an id that already exists loses its old row (weaviate_client.py:172 uuid5 semantics).  The old rows
  // are tombstoned before the new ones are published: a racing search may briefly miss the object, never see it twice.
  std::vector<int64_t> dead;
  {
    std::lock_guard<std::mutex> lk(ix->mu);
    for (int64_t i = 0; i < n; ++i) {
      auto it = ix->id2row.find(ids[i]);
      if (it != ix->id2row.end()) { dead.push_back(it->second); it->second = base + i; }
      else { ix->id2row.emplace(ids[i], base + i); ++ix->live; }
    }
  }
  const float nanv = nanf("");
  for (int64_t row : dead) CU_TRY(cudaMemcpyAsync(ix->d_inv_norm + row, &nanv, 4, cudaMemcpyHostToDevice, s));
  CU_TRY(cudaStreamSynchronize(s));  // the data has landed (and the host staging vectors may go out of scope)
  ix->rows_pub.store(base + n, std::memory_order_release);
  return AUR_OK;
}

int check_search_args(aur_index* ix, const void* q, int32_t nq, int32_t k, const void* s_out, const void* i_out) {
  if (!ix || !q || !s_out || !i_out) return fail(AUR_ERR_INVALID, "null argument");
  if (nq <= 0 || k <= 0) return fail(AUR_ERR_INVALID, "nq and k must be positive");
  return AUR_OK;
}

// Limits of one search batch: top-k lists of at most kMaxK, and no more queries than the kernels' grids index.
int check_batch(int32_t nq, int32_t k) {
  if (k > kMaxK) return fail(AUR_ERR_UNSUPPORTED, "k > %d", kMaxK);
  if (nq > 65535) return fail(AUR_ERR_UNSUPPORTED, "nq > 65535: split the batch");
  return AUR_OK;
}

// Per-query tenant codes (host) of a search into c's staging on stream s, and how the search applies them: the reference
// asks one tenant's question at a time (weaviate_client.py:244-249), so when every query of the batch carries the same
// (user, org) scope the filter folds into the row scale and the tensor-core kernel serves it (sc->uniform = scope, which
// must outlive the search's enqueue); a coalesced batch of several tenants' questions with at most 32 distinct scopes
// gives every corpus row a bit mask (one pre-pass) on the same kernel; more scopes -> the generic kernel.
int stage_tenant_scope(SearchCtx* c, cudaStream_t s, int32_t nq, const int32_t* q_user, const int32_t* q_org, int32_t* scope,
                       Scope* sc) {
  CU_TRY(c->stage_quser.reserve(nq));
  CU_TRY(cudaMemcpyAsync(c->stage_quser.p, q_user, static_cast<size_t>(nq) * 4, cudaMemcpyHostToDevice, s));
  sc->q_user = c->stage_quser.p;
  if (q_org) {
    CU_TRY(c->stage_qorg.reserve(nq));
    CU_TRY(cudaMemcpyAsync(c->stage_qorg.p, q_org, static_cast<size_t>(nq) * 4, cudaMemcpyHostToDevice, s));
    sc->q_org = c->stage_qorg.p;
  }
  bool uniform = true;
  scope[0] = q_user[0]; scope[1] = q_org ? q_org[0] : -1;
  for (int i = 1; i < nq && uniform; ++i) uniform = q_user[i] == scope[0] && (q_org ? q_org[i] : -1) == scope[1];
  if (uniform) { sc->uniform = scope; return AUR_OK; }
  std::vector<int32_t> tab; std::vector<int32_t> qs(static_cast<size_t>(nq));
  for (int i = 0; i < nq; ++i) {
    const int32_t u = q_user[i], o = q_org ? q_org[i] : -1;
    int found = -1;
    for (size_t t = 0; t < tab.size() / 2; ++t) if (tab[2 * t] == u && tab[2 * t + 1] == o) { found = static_cast<int>(t); break; }
    if (found < 0) {
      if (tab.size() / 2 == 32) return AUR_OK;
      found = static_cast<int>(tab.size() / 2); tab.push_back(u); tab.push_back(o);
    }
    qs[static_cast<size_t>(i)] = found;
  }
  CU_TRY(c->scope_tab.reserve(64)); CU_TRY(c->q_scope.reserve(static_cast<size_t>(nq)));
  CU_TRY(cudaMemcpyAsync(c->scope_tab.p, tab.data(), tab.size() * 4, cudaMemcpyHostToDevice, s));
  CU_TRY(cudaMemcpyAsync(c->q_scope.p, qs.data(), static_cast<size_t>(nq) * 4, cudaMemcpyHostToDevice, s));
  CU_TRY(cudaStreamSynchronize(s));          // tab / qs are host temporaries
  sc->scope_tab = c->scope_tab.p; sc->q_scope = c->q_scope.p; sc->n_scopes = static_cast<int>(tab.size() / 2);
  return AUR_OK;
}

// Host-buffer search: H2D of the queries, kernels, D2H of the results on a pool context's own stream.
int search_host(aur_index* ix, const void* queries_host, int32_t nq, int32_t k, const int32_t* q_user, const int32_t* q_org,
                const int64_t* allow_ids, int64_t n_allow, float* scores_out, int64_t* ids_out, int64_t* snapshot_out) {
  int rc = check_search_args(ix, queries_host, nq, k, scores_out, ids_out);
  if (rc != AUR_OK) return rc;
  const bool subset = allow_ids || n_allow > 0;
  if (subset && (n_allow < 0 || (n_allow > 0 && !allow_ids))) return fail(AUR_ERR_INVALID, "allow_ids / n_allow");
  if ((rc = check_batch(nq, k)) != AUR_OK) return rc;
  HostCall call(ix);
  if ((rc = call.open()) != AUR_OK) return rc;
  SearchCtx* c = call.c;
  cudaStream_t s = call.s;
  const int64_t n_rows = call.n_rows;
  if ((rc = call.stage(queries_host, nq, k, scores_out, ids_out)) != AUR_OK) return rc;
  Scope sc;
  int32_t scope[2] = {0, -1};
  std::vector<int32_t> rows_host;
  if (subset) {
    // resolved metadata pre-filter: ids -> rows of the published prefix (unknown / newer ids drop out)
    rows_host.reserve(static_cast<size_t>(n_allow));
    resolve_ids(ix, allow_ids, n_allow, n_rows, [&](int64_t, int32_t row) { rows_host.push_back(row); });
    CU_TRY(c->allow_rows.reserve(rows_host.size() + 1));
    if (!rows_host.empty())
      CU_TRY(cudaMemcpyAsync(c->allow_rows.p, rows_host.data(), rows_host.size() * 4, cudaMemcpyHostToDevice, s));
    sc.allow_rows = c->allow_rows.p;
    sc.n_allow = static_cast<int64_t>(rows_host.size());
  } else if (q_user && (rc = stage_tenant_scope(c, s, nq, q_user, q_org, scope, &sc)) != AUR_OK) {
    return rc;
  }
  rc = stats_begin(c, s, nq, n_rows);
  if (rc == AUR_OK) rc = search_enqueue(ix, c, c->stage_q.p, nq, k, sc, n_rows, call.d_scores, call.d_ids, nullptr, s);
  if (rc == AUR_OK) rc = stats_end(ix, c, s);
  if ((rc = call.finish(rc, nq, k, scores_out, ids_out)) != AUR_OK) return rc;
  if (snapshot_out) *snapshot_out = n_rows;
  return AUR_OK;
}

// Search with a pre-filter list per query (aur_search_lists).  The batch runs in blocks of kListQBlock queries (one
// dense candidate buffer each, as on the generic path); a block's work items are (list, <= kListQMax of its queries
// naming that list, kSimtSeg-row segment of the list), launched in batches whose score scratch stays within
// kListScoreSlots rows of kSimtSeg floats.
constexpr int kListQBlock = 1024;
constexpr int64_t kListScoreSlots = 16384;   // 128 MB of scores

int check_list_args(aur_index* ix, const void* q, int32_t nq, int32_t k, const void* s_out, const void* i_out) {
  int rc = check_search_args(ix, q, nq, k, s_out, i_out);
  if (rc != AUR_OK) return rc;
  if ((rc = check_batch(nq, k)) != AUR_OK) return rc;
  if (ix->dtype != AUR_BF16) return fail(AUR_ERR_UNSUPPORTED, "list search needs a bf16 index");
  return AUR_OK;
}

// The host side of a list search, built from the lists' lengths alone: blocks of queries, each with its work items cut
// into launches, and the int32 staging the device side uploads in one copy.
struct ListPlan {
  struct Launch { size_t items; int n_items, max_nq; };   // items: offset of the launch's first item in `stage`
  struct Block { int q0, nqb, n_segs; std::vector<Launch> launches; };
  std::vector<Block> blocks;
  std::vector<int32_t> stage;   // [the lists' rows, when the host resolved them][per block: its queries' positions, its items]
  size_t max_slots = 0, max_cand = 0;
};

// List l is rows lrow0[l] .. lrow0[l] + llen[l] of the lists' rows, ascending and without repeats.
int plan_list_search(int32_t nq, int32_t k, const int32_t* q_list, const std::vector<int64_t>& lrow0,
                     const std::vector<int64_t>& llen, ListPlan* pl) {
  const int ksel = k + kSlack;
  constexpr int kItemWords = sizeof(ListItem) / 4;
  std::vector<ListItem> items;
  for (int q0 = 0; q0 < nq; q0 += kListQBlock) {
    ListPlan::Block b{q0, std::min(kListQBlock, nq - q0), 1, {}};
    std::vector<int32_t> order(static_cast<size_t>(b.nqb));
    for (int i = 0; i < b.nqb; ++i) order[static_cast<size_t>(i)] = i;
    std::stable_sort(order.begin(), order.end(), [&](int32_t x, int32_t y) { return q_list[q0 + x] < q_list[q0 + y]; });
    const size_t qidx0 = pl->stage.size();
    pl->stage.insert(pl->stage.end(), order.begin(), order.end());
    items.clear();
    for (int i = 0; i < b.nqb;) {
      const int32_t l = q_list[q0 + order[static_cast<size_t>(i)]];
      int e = i;
      while (e < b.nqb && q_list[q0 + order[static_cast<size_t>(e)]] == l) ++e;
      const int64_t len = llen[static_cast<size_t>(l)];
      const int segs = static_cast<int>((len + kSimtSeg - 1) / kSimtSeg);
      b.n_segs = std::max(b.n_segs, segs);
      for (int g = i; g < e; g += kListQMax)
        for (int sg = 0; sg < segs; ++sg) {
          ListItem it;
          it.row0 = static_cast<int32_t>(lrow0[static_cast<size_t>(l)] + static_cast<int64_t>(sg) * kSimtSeg);
          it.n_rows = static_cast<int32_t>(std::min<int64_t>(kSimtSeg, len - static_cast<int64_t>(sg) * kSimtSeg));
          it.seg = sg;
          it.q0 = static_cast<int32_t>(qidx0 + g);
          it.nq = std::min(kListQMax, e - g);
          it.out = 0;
          items.push_back(it);
        }
      i = e;
    }
    // cut into launches; `out` = the item's first score row inside its launch
    int64_t slots = 0;
    for (size_t i = 0; i < items.size(); ++i) {
      if (b.launches.empty() || slots + items[i].nq > kListScoreSlots) {
        b.launches.push_back(ListPlan::Launch{pl->stage.size() + i * kItemWords, 0, 0});
        slots = 0;
      }
      ListPlan::Launch& ln = b.launches.back();
      items[i].out = static_cast<int32_t>(slots);
      slots += items[i].nq;
      ++ln.n_items;
      ln.max_nq = std::max(ln.max_nq, items[i].nq);
      pl->max_slots = std::max(pl->max_slots, static_cast<size_t>(slots));
    }
    const int32_t* w = reinterpret_cast<const int32_t*>(items.data());
    pl->stage.insert(pl->stage.end(), w, w + items.size() * kItemWords);
    pl->max_cand = std::max(pl->max_cand, static_cast<size_t>(b.nqb) * b.n_segs * ksel);
    pl->blocks.push_back(std::move(b));
  }
  if (pl->stage.size() > static_cast<size_t>(INT32_MAX))
    return fail(AUR_ERR_UNSUPPORTED, "the lists of this batch are too long for one call: split the batch");
  return AUR_OK;
}

// The device side of a planned list search over the queries in c->stage_q: the plan is uploaded, every block's work
// items launched, and its candidates folded and re-ranked exactly into d_scores / d_ids.  list_rows: the lists' rows on
// the device (nullptr: at the front of the plan's staging).
int run_list_search(aur_index* ix, SearchCtx* c, cudaStream_t s, const ListPlan& pl, int32_t nq, int32_t k,
                    const int32_t* list_rows, float* d_scores, int64_t* d_ids) {
  const int ksel = k + kSlack;
  CU_TRY(c->list_stage.reserve(pl.stage.size()));
  CU_TRY(c->list_scores.reserve(std::max<size_t>(pl.max_slots, 1) * kSimtSeg));
  CU_TRY(c->cand_a.reserve(pl.max_cand));
  CU_TRY(c->cand_read.reserve(static_cast<size_t>(nq)));
  c->last_kernel = AUR_KERNEL_LIST;
  CU_TRY(cudaMemcpyAsync(c->list_stage.p, pl.stage.data(), pl.stage.size() * 4, cudaMemcpyHostToDevice, s));
  for (size_t bi = 0; bi < pl.blocks.size(); ++bi) {
    const ListPlan::Block& b = pl.blocks[bi];
    const uint8_t* qb = c->stage_q.p + static_cast<size_t>(b.q0) * ix->dim * 2;
    CU_TRY(cudaMemsetAsync(c->cand_a.p, 0, static_cast<size_t>(b.nqb) * b.n_segs * ksel * 8, s));   // 0 = empty slot
    if (bi == 0) CU_TRY(cudaEventRecord(c->ev_k0, s));
    for (const ListPlan::Launch& ln : b.launches) {
      ListParams p{};
      p.q = reinterpret_cast<const __nv_bfloat16*>(qb);
      p.rows = static_cast<const __nv_bfloat16*>(ix->d_rows);
      p.inv_norm = ix->d_inv_norm;
      p.ids = ix->d_ids;
      p.items = reinterpret_cast<const ListItem*>(c->list_stage.p + ln.items);
      p.n_items = ln.n_items;
      p.list_rows = list_rows ? list_rows : c->list_stage.p;
      p.qidx = c->list_stage.p;
      p.scores = c->list_scores.p;
      p.cand = c->cand_a.p;
      p.dim = ix->dim; p.ksel = ksel; p.n_lists = b.n_segs;
      CU_TRY(launch_list_search(p, ln.max_nq, s));
      c->last_launches += 2;
    }
    if (bi == 0) CU_TRY(cudaEventRecord(c->ev_k1, s));
    const int rc = candidate_tail(ix, c, s, qb, b.q0, b.nqb, k, b.n_segs, false, d_scores, d_ids, nullptr, nullptr);
    if (rc != AUR_OK) return rc;
  }
  return AUR_OK;
}

// Filter programs (aur_search_filtered, aur_filter_ids): n_programs programs, program q = tokens
// prog[4 * prog_off[q] .. 4 * prog_off[q + 1]), each token {kind, column, bitmap offset, bitmap length}.
int check_programs(aur_index* ix, const int32_t* prog, const int32_t* prog_off, int32_t n_programs, const uint32_t* bitmap,
                   int64_t bitmap_words) {
  if (!prog || !prog_off) return fail(AUR_ERR_INVALID, "null program");
  if (n_programs < 1 || n_programs > kFiltCallPrograms) return fail(AUR_ERR_INVALID, "1 <= n_programs <= %d", kFiltCallPrograms);
  if (bitmap_words < 0 || (bitmap_words > 0 && !bitmap)) return fail(AUR_ERR_INVALID, "bitmap / bitmap_words");
  if (prog_off[0] != 0) return fail(AUR_ERR_INVALID, "program offsets must start at 0");
  std::lock_guard<std::mutex> lk(ix->mu);   // the attribute columns that exist
  for (int32_t q = 0; q < n_programs; ++q) {
    if (prog_off[q + 1] < prog_off[q]) return fail(AUR_ERR_INVALID, "program offsets decrease at program %d", q);
    int depth = 0, leaves = 0;
    for (int32_t t = prog_off[q]; t < prog_off[q + 1]; ++t) {
      const int32_t* tk = prog + 4 * static_cast<int64_t>(t);
      if (tk[0] == kFiltLeaf) {
        if (++leaves > kFiltMaxLeaves) return fail(AUR_ERR_INVALID, "program %d has more than %d leaves", q, kFiltMaxLeaves);
        if (tk[1] < 0 || tk[1] >= kFiltCols) return fail(AUR_ERR_INVALID, "program %d: column %d out of range", q, tk[1]);
        if (tk[1] >= 2 && !ix->d_attr[tk[1] - 2]) return fail(AUR_ERR_INVALID, "program %d: column %d was never set", q, tk[1]);
        if (tk[2] < 0 || tk[3] < 0 || static_cast<int64_t>(tk[2]) + tk[3] > bitmap_words * 32)
          return fail(AUR_ERR_INVALID, "program %d: bitmap slice [%d, +%d) outside the bitmap", q, tk[2], tk[3]);
        ++depth;
      } else if (tk[0] == kFiltAnd || tk[0] == kFiltOr) {
        if (depth < 2) return fail(AUR_ERR_INVALID, "program %d: operator without two operands", q);
        --depth;
      } else {
        return fail(AUR_ERR_INVALID, "program %d: unknown token kind %d", q, tk[0]);
      }
    }
    if (depth != 1) return fail(AUR_ERR_INVALID, "program %d leaves %d values, not one", q, depth);
  }
  return AUR_OK;
}

// Where pass `ps` of a filter evaluation (programs 32 ps .. 32 ps + 31) keeps its data: c->filt_mask holds one mask per
// pass, c->filt_counts every pass's 32 totals and then every pass's block counts.
struct FiltPass { uint32_t* mask; uint32_t* totals; uint32_t* counts; int n_programs; };
FiltPass filt_pass(SearchCtx* c, int ps, int n_programs, int64_t n_rows) {
  const int n_passes = (n_programs + kFiltMaxPrograms - 1) / kFiltMaxPrograms;
  const size_t rows = static_cast<size_t>(std::max<int64_t>(n_rows, 1)), nb = static_cast<size_t>(std::max(filter_blocks(n_rows), 1));
  return FiltPass{c->filt_mask.p + ps * rows, c->filt_counts.p + ps * kFiltMaxPrograms,
                  c->filt_counts.p + static_cast<size_t>(n_passes) * kFiltMaxPrograms + ps * kFiltMaxPrograms * nb,
                  std::min(kFiltMaxPrograms, n_programs - ps * kFiltMaxPrograms)};
}

// Uploads checked programs, evaluates them over the snapshot's rows [0, n_rows) in passes of up to 32 programs (masks
// and counts in c->filt_mask / c->filt_counts, filt_pass) and reads back each program's number of matching rows (one
// small copy and a sync for all passes).
int filter_count(aur_index* ix, SearchCtx* c, cudaStream_t s, const int32_t* prog, const int32_t* prog_off, int32_t n_programs,
                 const uint32_t* bitmap, int64_t bitmap_words, int64_t n_rows, std::vector<int64_t>* totals) {
  const size_t n_tok = static_cast<size_t>(prog_off[n_programs]);
  std::vector<int32_t> st(n_tok * 4 + static_cast<size_t>(n_programs) + 1 + static_cast<size_t>(bitmap_words));
  if (n_tok) memcpy(st.data(), prog, n_tok * 16);
  memcpy(st.data() + n_tok * 4, prog_off, (static_cast<size_t>(n_programs) + 1) * 4);
  if (bitmap_words) memcpy(st.data() + n_tok * 4 + n_programs + 1, bitmap, static_cast<size_t>(bitmap_words) * 4);
  const int n_passes = (n_programs + kFiltMaxPrograms - 1) / kFiltMaxPrograms;
  const size_t nb = static_cast<size_t>(std::max(filter_blocks(n_rows), 1));
  CU_TRY(c->filt_stage.reserve(st.size()));
  CU_TRY(c->filt_mask.reserve(static_cast<size_t>(n_passes) * static_cast<size_t>(std::max<int64_t>(n_rows, 1))));
  CU_TRY(c->filt_counts.reserve(static_cast<size_t>(n_passes) * kFiltMaxPrograms * (1 + nb)));
  CU_TRY(cudaMemcpyAsync(c->filt_stage.p, st.data(), st.size() * 4, cudaMemcpyHostToDevice, s));   // pageable: staged on return
  FiltParams p{};
  p.cols[0] = ix->d_user; p.cols[1] = ix->d_org;
  {
    std::lock_guard<std::mutex> lk(ix->mu);
    for (int i = 0; i < kFiltAttrCols; ++i) p.cols[2 + i] = ix->d_attr[i];
  }
  const int32_t* d_off = c->filt_stage.p + n_tok * 4;   // token indices stay absolute: a pass starts at its first offset
  p.tok = reinterpret_cast<const FiltToken*>(c->filt_stage.p);
  p.bitmap = reinterpret_cast<const uint32_t*>(d_off + n_programs + 1);
  p.inv_norm = ix->d_inv_norm;
  p.n_rows = n_rows;
  for (int ps = 0; ps < n_passes; ++ps) {
    const FiltPass fp = filt_pass(c, ps, n_programs, n_rows);
    p.prog_off = d_off + ps * kFiltMaxPrograms;
    p.n_programs = fp.n_programs;
    CU_TRY(launch_filter_count(p, fp.mask, fp.counts, fp.totals, s));
    ++c->last_launches;
  }
  std::vector<uint32_t> h(static_cast<size_t>(n_passes) * kFiltMaxPrograms);
  CU_TRY(cudaMemcpyAsync(h.data(), c->filt_counts.p, h.size() * 4, cudaMemcpyDeviceToHost, s));
  CU_TRY(cudaStreamSynchronize(s));
  totals->assign(h.begin(), h.begin() + n_programs);   // pass ps's totals are words 32 ps .. 32 ps + 31: program order
  return AUR_OK;
}

// After filter_count: every program's matching rows, ascending, program after program, into c->filt_rows (and with
// `with_ids` their ids into c->filt_ids).
int filter_write(aur_index* ix, SearchCtx* c, cudaStream_t s, int32_t n_programs, const std::vector<int64_t>& tot, int64_t n_rows,
                 bool with_ids) {
  int64_t total = 0;
  for (int64_t t : tot) total += t;
  if (total > INT32_MAX) return fail(AUR_ERR_UNSUPPORTED, "the programs of this call match too many rows for one call: split it");
  CU_TRY(c->filt_rows.reserve(static_cast<size_t>(std::max<int64_t>(total, 1))));
  if (with_ids) CU_TRY(c->filt_ids.reserve(static_cast<size_t>(std::max<int64_t>(total, 1))));
  int64_t base = 0;
  for (int ps = 0; ps * kFiltMaxPrograms < n_programs; ++ps) {
    const FiltPass fp = filt_pass(c, ps, n_programs, n_rows);
    CU_TRY(launch_filter_write(fp.mask, fp.counts, fp.totals, fp.n_programs, n_rows, with_ids ? ix->d_ids : nullptr,
                               c->filt_rows.p + base, with_ids ? c->filt_ids.p + base : nullptr, s));
    if (n_rows > 0) c->last_launches += 2;
    for (int q = 0; q < fp.n_programs; ++q) base += tot[static_cast<size_t>(ps * kFiltMaxPrograms + q)];
  }
  return AUR_OK;
}

}  // namespace

namespace aur {
int dense_leg(aur_index* ix, int device, cudaStream_t s, const void* queries_host, int32_t nq, int32_t k, const int32_t* q_user,
              const int32_t* q_org, float* scores, int64_t* ids, int64_t* snapshot_rows) {
  if (ix->dtype != AUR_BF16) return fail(AUR_ERR_UNSUPPORTED, "hybrid search needs a bf16 index");
  if (ix->device != device) return fail(AUR_ERR_INVALID, "the keyword store is on device %d, the index on device %d", device, ix->device);
  int rc = check_batch(nq, k);
  if (rc != AUR_OK) return rc;
  std::shared_lock<std::shared_mutex> rl(ix->rw);   // (compaction waits for the device before it moves a row)
  CU_TRY(cudaSetDevice(ix->device));
  SearchCtx* c = nullptr;
  if ((rc = acquire_ctx(ix, s, &c)) != AUR_OK) return rc;
  std::lock_guard<std::mutex> cl(c->mu);
  const int64_t n_rows = ix->rows_pub.load(std::memory_order_acquire);
  const size_t qbytes = static_cast<size_t>(nq) * ix->dim * ix->elt;
  CU_TRY(c->stage_q.reserve(qbytes));
  CU_TRY(cudaMemcpyAsync(c->stage_q.p, queries_host, qbytes, cudaMemcpyHostToDevice, s));
  Scope sc;
  int32_t scope[2] = {0, -1};
  if (q_user && (rc = stage_tenant_scope(c, s, nq, q_user, q_org, scope, &sc)) != AUR_OK) return rc;
  if ((rc = stats_begin(c, s, nq, n_rows)) != AUR_OK) return rc;
  if ((rc = search_enqueue(ix, c, c->stage_q.p, nq, k, sc, n_rows, scores, ids, nullptr, s)) != AUR_OK) return rc;
  if ((rc = stats_end(ix, c, s)) != AUR_OK) return rc;
  *snapshot_rows = n_rows;
  return AUR_OK;
}

int index_device(const aur_index* ix) { return ix->device; }
int index_is_bf16(const aur_index* ix) { return ix->dtype == AUR_BF16; }
}  // namespace aur

extern "C" {

int aur_abi_version(void) { return AUR_ABI_VERSION; }
const char* aur_last_error(void) { return g_err.c_str(); }

int aur_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

int aur_open(const aur_config* cfg, aur_index** out) {
  if (!cfg || !out) return fail(AUR_ERR_INVALID, "null argument");
  *out = nullptr;
  if (cfg->dim <= 0 || cfg->capacity <= 0) return fail(AUR_ERR_INVALID, "dim and capacity must be positive");
  if (cfg->dtype != AUR_BF16 && cfg->dtype != AUR_F32) return fail(AUR_ERR_INVALID, "dtype must be AUR_BF16 or AUR_F32");
  if (cfg->dtype == AUR_BF16 && cfg->dim % 8 != 0) return fail(AUR_ERR_INVALID, "bf16 rows need dim %% 8 == 0");
  if (cfg->capacity > 0x7FFFFFC0ll) return fail(AUR_ERR_INVALID, "capacity exceeds int32 row indexing");
  int ndev = aur_device_count();
  if (ndev == 0) return fail(AUR_ERR_NO_DEVICE, "no CUDA device: aurora_b200 has no CPU fallback");
  if (cfg->device < 0 || cfg->device >= ndev) return fail(AUR_ERR_INVALID, "device %d out of range", cfg->device);
  CU_TRY(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  CU_TRY(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9) return fail(AUR_ERR_UNSUPPORTED, "sm_%d%d device: this library is built for sm_90a only", prop.major, prop.minor);
  aur_index* ix = new aur_index();
  ix->device = cfg->device; ix->dim = cfg->dim; ix->dtype = cfg->dtype; ix->capacity = cfg->capacity;
  ix->elt = cfg->dtype == AUR_BF16 ? 2 : 4;
  ix->sm_count = prop.multiProcessorCount;
  ix->smem_optin = prop.sharedMemPerBlockOptin;
  auto bail = [&](int rc) { aur_close(ix); return rc; };
#define OPEN_TRY(expr)                                                                                  \
  do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) return bail(fail(e_ == cudaErrorMemoryAllocation ? AUR_ERR_NOMEM : AUR_ERR_CUDA, \
                                                                 "%s: %s", #expr, cudaGetErrorString(e_))); } while (0)
  int prio_lo = 0, prio_hi = 0;
  OPEN_TRY(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
  OPEN_TRY(cudaStreamCreateWithPriority(&ix->stream, cudaStreamNonBlocking, prio_hi));
  OPEN_TRY(cudaStreamCreateWithPriority(&ix->ingest_stream, cudaStreamNonBlocking, prio_lo));
  ix->cap_pad = (cfg->capacity + kTcTileN - 1) / kTcTileN * kTcTileN;
  const size_t cap_pad = static_cast<size_t>(ix->cap_pad);
  OPEN_TRY(cudaMalloc(&ix->d_rows, cap_pad * ix->dim * ix->elt));
  OPEN_TRY(cudaMalloc(&ix->d_inv_norm, cap_pad * 4));
  OPEN_TRY(cudaMalloc(&ix->d_ids, cap_pad * 8));
  OPEN_TRY(cudaMalloc(&ix->d_user, cap_pad * 4));
  OPEN_TRY(cudaMalloc(&ix->d_org, cap_pad * 4));
#undef OPEN_TRY
  int rc = build_tmaps(ix);
  if (rc != AUR_OK) return bail(rc);
  *out = ix;
  return AUR_OK;
}

int aur_close(aur_index* ix) {
  if (!ix) return AUR_OK;
  cudaSetDevice(ix->device);
  cudaDeviceSynchronize();   // searches bound to caller streams may still be in flight
  cudaFree(ix->d_rows); cudaFree(ix->d_inv_norm); cudaFree(ix->d_ids); cudaFree(ix->d_user); cudaFree(ix->d_org);
  for (int32_t* a : ix->d_attr) cudaFree(a);
  ix->attr_stage.release();
  for (auto& c : ix->ctxs) c->release();
  if (ix->stream) cudaStreamDestroy(ix->stream);
  if (ix->ingest_stream) cudaStreamDestroy(ix->ingest_stream);
  delete ix;
  return AUR_OK;
}

int aur_get_stats(aur_index* ix, aur_stats* out) {
  if (!ix || !out) return fail(AUR_ERR_INVALID, "null argument");
  memset(out, 0, sizeof *out);
  SearchCtx* c = nullptr;
  {
    std::lock_guard<std::mutex> lk(ix->mu);
    out->rows = ix->rows_pub.load(std::memory_order_acquire); out->live = ix->live; out->capacity = ix->capacity;
    out->dim = ix->dim; out->dtype = ix->dtype;
    c = ix->last_ctx;
  }
  if (c) {
    std::lock_guard<std::mutex> cl(c->mu);
    out->last_kernel = c->last_kernel; out->last_launches = c->last_launches; out->last_tile_n = c->last_tile_n;
    if (c->have_timing) {
      CU_TRY(cudaSetDevice(ix->device));
      CU_TRY(cudaEventSynchronize(c->ev_end));
      CU_TRY(cudaEventElapsedTime(&out->last_kernel_ms, c->ev_k0, c->ev_k1));
      CU_TRY(cudaEventElapsedTime(&out->last_total_ms, c->ev_begin, c->ev_end));
      CU_TRY(cudaEventElapsedTime(&out->last_finalize_ms, c->ev_k1, c->ev_fin));
      CU_TRY(cudaEventElapsedTime(&out->last_merge_ms, c->ev_fin, c->ev_end));
      std::vector<uint32_t> n(std::min(static_cast<size_t>(c->last_nq), c->cand_read.n));
      CU_TRY(cudaMemcpy(n.data(), c->cand_read.p, n.size() * 4, cudaMemcpyDeviceToHost));
      for (uint32_t v : n) {
        out->last_candidates += v;
        out->last_candidates_max = std::max(out->last_candidates_max, static_cast<int32_t>(v));
      }
    }
  }
  return AUR_OK;
}

int aur_export(aur_index* ix, void* rows_out, int64_t* ids_out, int32_t* user_out, int32_t* org_out, uint8_t* live_out,
               int64_t n) {
  if (!ix || !rows_out || !ids_out || !live_out) return fail(AUR_ERR_INVALID, "null argument");
  std::unique_lock<std::shared_mutex> wl(ix->rw);
  const int64_t rows = ix->rows_pub.load(std::memory_order_acquire);
  if (n != rows) return fail(AUR_ERR_INVALID, "n must equal aur_stats.rows (%lld)", (long long)rows);
  if (n == 0) return AUR_OK;
  CU_TRY(cudaSetDevice(ix->device));
  CU_TRY(cudaDeviceSynchronize());
  std::vector<float> inv(static_cast<size_t>(n));
  CU_TRY(cudaMemcpy(inv.data(), ix->d_inv_norm, sizeof(float) * n, cudaMemcpyDeviceToHost));
  CU_TRY(cudaMemcpy(rows_out, ix->d_rows, static_cast<size_t>(n) * ix->dim * ix->elt, cudaMemcpyDeviceToHost));
  CU_TRY(cudaMemcpy(ids_out, ix->d_ids, sizeof(int64_t) * n, cudaMemcpyDeviceToHost));
  if (user_out) CU_TRY(cudaMemcpy(user_out, ix->d_user, sizeof(int32_t) * n, cudaMemcpyDeviceToHost));
  if (org_out) CU_TRY(cudaMemcpy(org_out, ix->d_org, sizeof(int32_t) * n, cudaMemcpyDeviceToHost));
  for (int64_t i = 0; i < n; ++i) live_out[i] = inv[static_cast<size_t>(i)] == inv[static_cast<size_t>(i)];   // NaN = tombstone
  return AUR_OK;
}

int aur_read_rows(aur_index* ix, int64_t row0, int64_t n, void* rows_out, int64_t* ids_out) {
  if (!ix || (n > 0 && (!rows_out || !ids_out))) return fail(AUR_ERR_INVALID, "null argument");
  std::shared_lock<std::shared_mutex> rl(ix->rw);
  const int64_t rows = ix->rows_pub.load(std::memory_order_acquire);
  if (row0 < 0 || n < 0 || row0 + n > rows) return fail(AUR_ERR_INVALID, "rows [%lld, %lld) are not inside the published prefix of %lld",
                                                        (long long)row0, (long long)(row0 + n), (long long)rows);
  if (n == 0) return AUR_OK;
  CU_TRY(cudaSetDevice(ix->device));
  const size_t rb = static_cast<size_t>(ix->dim) * ix->elt;
  CU_TRY(cudaMemcpy(rows_out, static_cast<const uint8_t*>(ix->d_rows) + static_cast<size_t>(row0) * rb, static_cast<size_t>(n) * rb,
                    cudaMemcpyDeviceToHost));
  CU_TRY(cudaMemcpy(ids_out, ix->d_ids + row0, static_cast<size_t>(n) * 8, cudaMemcpyDeviceToHost));
  return AUR_OK;
}

int aur_compact(aur_index* ix, int64_t* reclaimed) {
  if (!ix) return fail(AUR_ERR_INVALID, "null index");
  if (reclaimed) *reclaimed = 0;
  std::unique_lock<std::shared_mutex> wl(ix->rw);   // no search or append is being enqueued ...
  std::lock_guard<std::mutex> wk(ix->mu_write);
  CU_TRY(cudaSetDevice(ix->device));
  CU_TRY(cudaDeviceSynchronize());                  // ... and none is still running
  const int64_t rows = ix->rows_pub.load(std::memory_order_acquire);
  std::vector<std::pair<int64_t, int64_t>> order;   // (old row, id) of the live rows, in row order
  {
    std::lock_guard<std::mutex> lk(ix->mu);
    order.reserve(ix->id2row.size());
    for (auto& kv : ix->id2row) order.emplace_back(kv.second, kv.first);
  }
  std::sort(order.begin(), order.end());
  const int64_t nlive = static_cast<int64_t>(order.size());
  if (nlive == rows) return AUR_OK;                 // nothing to reclaim
  // Stable compaction in place, a bounce buffer at a time: live row j moves down to row j.  Chunk [i0, i1) only
  // overwrites rows < i1 <= old(i1), i.e. rows whose content has already been gathered or moved.
  const int64_t chunk = 65536;
  DevBuf<int32_t> d_map; DevBuf<uint8_t> bounce; DevBuf<float> b_inv; DevBuf<int64_t> b_ids; DevBuf<int32_t> b_user, b_org, b_attr;
  std::vector<int32_t*> attrs;
  {
    std::lock_guard<std::mutex> lk(ix->mu);
    for (int32_t* a : ix->d_attr) if (a) attrs.push_back(a);
  }
  cudaError_t e = d_map.reserve(static_cast<size_t>(chunk));
  if (e == cudaSuccess) e = bounce.reserve(static_cast<size_t>(chunk) * ix->dim * ix->elt);
  if (e == cudaSuccess) e = b_inv.reserve(chunk);
  if (e == cudaSuccess) e = b_ids.reserve(chunk);
  if (e == cudaSuccess) e = b_user.reserve(chunk);
  if (e == cudaSuccess) e = b_org.reserve(chunk);
  if (e == cudaSuccess && !attrs.empty()) e = b_attr.reserve(chunk);
  auto drop = [&]() { d_map.release(); bounce.release(); b_inv.release(); b_ids.release(); b_user.release(); b_org.release(); b_attr.release(); };
  if (e != cudaSuccess) { drop(); return fail(AUR_ERR_NOMEM, "aur_compact: %s", cudaGetErrorString(e)); }
  cudaStream_t s = ix->ingest_stream;
  std::vector<int32_t> map_host(static_cast<size_t>(chunk));
  int64_t first_moved = 0;
  while (first_moved < nlive && order[static_cast<size_t>(first_moved)].first == first_moved) ++first_moved;   // untouched prefix
  for (int64_t i0 = first_moved; i0 < nlive && e == cudaSuccess; i0 += chunk) {
    const int64_t m = (nlive - i0 < chunk) ? nlive - i0 : chunk;
    for (int64_t j = 0; j < m; ++j) map_host[static_cast<size_t>(j)] = static_cast<int32_t>(order[static_cast<size_t>(i0 + j)].first);
    e = cudaMemcpyAsync(d_map.p, map_host.data(), static_cast<size_t>(m) * 4, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = launch_gather_rows(ix->d_rows, ix->d_inv_norm, ix->d_ids, ix->d_user, ix->d_org, d_map.p, m,
                                                 static_cast<int>(ix->dim * ix->elt), bounce.p, b_inv.p, b_ids.p, b_user.p, b_org.p, s);
    const size_t rb = static_cast<size_t>(ix->dim) * ix->elt;
    if (e == cudaSuccess) e = cudaMemcpyAsync(static_cast<uint8_t*>(ix->d_rows) + static_cast<size_t>(i0) * rb, bounce.p, static_cast<size_t>(m) * rb, cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(ix->d_inv_norm + i0, b_inv.p, static_cast<size_t>(m) * 4, cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(ix->d_ids + i0, b_ids.p, static_cast<size_t>(m) * 8, cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(ix->d_user + i0, b_user.p, static_cast<size_t>(m) * 4, cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(ix->d_org + i0, b_org.p, static_cast<size_t>(m) * 4, cudaMemcpyDeviceToDevice, s);
    for (int32_t* a : attrs) {
      if (e == cudaSuccess) e = launch_gather_i32(a, d_map.p, m, b_attr.p, s);
      if (e == cudaSuccess) e = cudaMemcpyAsync(a + i0, b_attr.p, static_cast<size_t>(m) * 4, cudaMemcpyDeviceToDevice, s);
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);   // map_host is reused by the next chunk
  }
  // the freed rows are appended to again: their attributes start absent, as in a fresh column
  for (int32_t* a : attrs)
    if (e == cudaSuccess) e = cudaMemsetAsync(a + nlive, 0xFF, static_cast<size_t>(rows - nlive) * 4, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  drop();
  if (e != cudaSuccess) return fail(AUR_ERR_CUDA, "aur_compact: %s (the shard may be inconsistent: restore the last snapshot)", cudaGetErrorString(e));
  {
    std::lock_guard<std::mutex> lk(ix->mu);
    for (int64_t j = 0; j < nlive; ++j) ix->id2row[order[static_cast<size_t>(j)].second] = j;
    ix->live = nlive;
  }
  ix->rows_pub.store(nlive, std::memory_order_release);
  if (reclaimed) *reclaimed = rows - nlive;
  return AUR_OK;
}

int aur_set_option(aur_index* ix, const char* key, int64_t value) {
  if (!ix || !key) return fail(AUR_ERR_INVALID, "null argument");
  if (strcmp(key, "dbg_epoch") == 0) {   // bring-up: move every context's launch counter, e.g. to just before it wraps
    if (value < 1 || value > kSearchEpochMax) return fail(AUR_ERR_INVALID, "dbg_epoch must be in 1 .. %u", kSearchEpochMax);
    std::vector<SearchCtx*> cs;
    {
      std::lock_guard<std::mutex> lk(ix->mu);
      ix->opt_dbg_epoch.store(static_cast<uint32_t>(value));   // contexts that start their counter later
      for (auto& c : ix->ctxs) cs.push_back(c.get());
    }
    CU_TRY(cudaSetDevice(ix->device));
    const uint32_t e = static_cast<uint32_t>(value);
    for (SearchCtx* c : cs) {
      std::lock_guard<std::mutex> cl(c->mu);
      if (c->d_epoch.n == 0) continue;
      CU_TRY(cudaDeviceSynchronize());   // searches already enqueued on the context finish with their own counter
      CU_TRY(cudaMemcpy(c->d_epoch.p, &e, 4, cudaMemcpyHostToDevice));
    }
    return AUR_OK;
  }
  std::lock_guard<std::mutex> lk(ix->mu);
  if (strcmp(key, "kernel") == 0) {
    if (value < AUR_KERNEL_AUTO || value > AUR_KERNEL_TC2) return fail(AUR_ERR_INVALID, "unknown kernel %lld", (long long)value);
    ix->opt_kernel = static_cast<int>(value);
    return AUR_OK;
  }
  if (strcmp(key, "tc_tile") == 0) {
    if (value != 0 && value != kTcTileN && value != kTcTileWide) return fail(AUR_ERR_INVALID, "tc_tile must be 0 (auto), 64 or 128");
    ix->opt_tc_tile = static_cast<int>(value);
    return AUR_OK;
  }
  if (strcmp(key, "dbg_flags") == 0) { ix->opt_dbg_flags = static_cast<int>(value); return AUR_OK; }
  return fail(AUR_ERR_INVALID, "unknown option '%s'", key);
}

int aur_sync(aur_index* ix) {
  if (!ix) return fail(AUR_ERR_INVALID, "null argument");
  CU_TRY(cudaSetDevice(ix->device));
  CU_TRY(cudaStreamSynchronize(ix->stream));
  return AUR_OK;
}

int aur_add(aur_index* ix, const void* rows_host, const int64_t* ids, const int32_t* user_codes,
            const int32_t* org_codes, int64_t n) {
  if (!ix) return fail(AUR_ERR_INVALID, "null index");
  std::shared_lock<std::shared_mutex> rl(ix->rw);
  std::lock_guard<std::mutex> wk(ix->mu_write);
  CU_TRY(cudaSetDevice(ix->device));
  return add_common(ix, rows_host, false, ids, user_codes, org_codes, n, ix->ingest_stream);
}

int aur_add_dev(aur_index* ix, const void* rows_dev, const int64_t* ids_host, const int32_t* user_codes_host,
                const int32_t* org_codes_host, int64_t n, void* stream) {
  if (!ix) return fail(AUR_ERR_INVALID, "null index");
  std::shared_lock<std::shared_mutex> rl(ix->rw);
  std::lock_guard<std::mutex> wk(ix->mu_write);
  CU_TRY(cudaSetDevice(ix->device));
  return add_common(ix, rows_dev, true, ids_host, user_codes_host, org_codes_host, n,
                    stream ? static_cast<cudaStream_t>(stream) : ix->ingest_stream);
}

int aur_remove(aur_index* ix, const int64_t* ids, int64_t n, int64_t* removed) {
  if (!ix || (n > 0 && !ids)) return fail(AUR_ERR_INVALID, "null argument");
  std::shared_lock<std::shared_mutex> rl(ix->rw);
  std::lock_guard<std::mutex> wk(ix->mu_write);
  CU_TRY(cudaSetDevice(ix->device));
  const float nanv = nanf("");
  std::vector<int64_t> dead;
  {
    std::lock_guard<std::mutex> lk(ix->mu);
    for (int64_t i = 0; i < n; ++i) {
      auto it = ix->id2row.find(ids[i]);
      if (it == ix->id2row.end()) continue;
      dead.push_back(it->second);
      ix->id2row.erase(it);
      --ix->live;
    }
  }
  for (int64_t row : dead) CU_TRY(cudaMemcpyAsync(ix->d_inv_norm + row, &nanv, 4, cudaMemcpyHostToDevice, ix->ingest_stream));
  CU_TRY(cudaStreamSynchronize(ix->ingest_stream));
  if (removed) *removed = static_cast<int64_t>(dead.size());
  return AUR_OK;
}

int aur_search_dev(aur_index* ix, const void* queries_dev, int32_t nq, int32_t k, const int32_t* q_user_dev,
                   const int32_t* q_org_dev, float* scores_dev, int64_t* ids_dev, double* scores64_dev, void* stream) {
  int rc = check_search_args(ix, queries_dev, nq, k, scores_dev, ids_dev);
  if (rc != AUR_OK) return rc;
  if ((rc = check_batch(nq, k)) != AUR_OK) return rc;
  std::shared_lock<std::shared_mutex> rl(ix->rw);
  CU_TRY(cudaSetDevice(ix->device));
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : ix->stream;
  SearchCtx* c = nullptr;
  if ((rc = acquire_ctx(ix, s, &c)) != AUR_OK) return rc;
  std::lock_guard<std::mutex> cl(c->mu);
  const int64_t n_rows = ix->rows_pub.load(std::memory_order_acquire);
  Scope sc;
  sc.q_user = q_user_dev; sc.q_org = q_org_dev;
  if ((rc = stats_begin(c, s, nq, n_rows)) != AUR_OK) return rc;
  if ((rc = search_enqueue(ix, c, queries_dev, nq, k, sc, n_rows, scores_dev, ids_dev, scores64_dev, s)) != AUR_OK) return rc;
  return stats_end(ix, c, s);
}

int aur_search(aur_index* ix, const void* queries_host, int32_t nq, int32_t k, const int32_t* q_user,
               const int32_t* q_org, float* scores_out, int64_t* ids_out) {
  return search_host(ix, queries_host, nq, k, q_user, q_org, nullptr, -1, scores_out, ids_out, nullptr);
}

int aur_search_ex(aur_index* ix, const void* queries_host, int32_t nq, int32_t k, const int32_t* q_user,
                  const int32_t* q_org, float* scores_out, int64_t* ids_out, int64_t* snapshot_rows_out) {
  return search_host(ix, queries_host, nq, k, q_user, q_org, nullptr, -1, scores_out, ids_out, snapshot_rows_out);
}

int aur_search_subset(aur_index* ix, const void* queries_host, int32_t nq, int32_t k, const int64_t* allow_ids,
                      int64_t n_allow, float* scores_out, int64_t* ids_out) {
  if (n_allow < 0) return fail(AUR_ERR_INVALID, "n_allow < 0");
  static const int64_t none = 0;
  return search_host(ix, queries_host, nq, k, nullptr, nullptr, allow_ids ? allow_ids : &none, n_allow, scores_out, ids_out, nullptr);
}

int aur_search_lists(aur_index* ix, const void* queries_host, int32_t nq, int32_t k, const int64_t* list_ids,
                     const int64_t* list_offsets, int32_t n_lists, const int32_t* q_list, float* scores_out,
                     int64_t* ids_out, int64_t* snapshot_rows_out) {
  int rc = check_list_args(ix, queries_host, nq, k, scores_out, ids_out);
  if (rc != AUR_OK) return rc;
  if (!list_offsets || !q_list || n_lists < 1) return fail(AUR_ERR_INVALID, "list_offsets, q_list and n_lists >= 1 are required");
  if (list_offsets[0] != 0) return fail(AUR_ERR_INVALID, "list_offsets[0] must be 0");
  for (int32_t l = 0; l < n_lists; ++l)
    if (list_offsets[l + 1] < list_offsets[l]) return fail(AUR_ERR_INVALID, "list_offsets decrease at list %d", l);
  if (list_offsets[n_lists] > 0 && !list_ids) return fail(AUR_ERR_INVALID, "list_ids is required");
  for (int32_t q = 0; q < nq; ++q)
    if (q_list[q] < 0 || q_list[q] >= n_lists) return fail(AUR_ERR_INVALID, "q_list[%d] = %d is not a list", q, q_list[q]);

  HostCall call(ix);
  if ((rc = call.open()) != AUR_OK) return rc;
  SearchCtx* c = call.c;
  cudaStream_t s = call.s;
  // staging (int32): [every named list's rows of the published prefix, sorted, once each][the plan's blocks]
  std::vector<char> named(static_cast<size_t>(n_lists), 0);
  for (int32_t q = 0; q < nq; ++q) named[static_cast<size_t>(q_list[q])] = 1;
  ListPlan pl;
  std::vector<int64_t> lrow0(static_cast<size_t>(n_lists), 0), llen(static_cast<size_t>(n_lists), 0);
  for (int32_t l = 0; l < n_lists; ++l) {
    const size_t r0 = pl.stage.size();
    lrow0[static_cast<size_t>(l)] = static_cast<int64_t>(r0);
    if (!named[static_cast<size_t>(l)]) continue;
    resolve_ids(ix, list_ids + list_offsets[l], list_offsets[l + 1] - list_offsets[l], call.n_rows,
                [&](int64_t, int32_t row) { pl.stage.push_back(row); });
    std::sort(pl.stage.begin() + r0, pl.stage.end());
    pl.stage.erase(std::unique(pl.stage.begin() + r0, pl.stage.end()), pl.stage.end());
    llen[static_cast<size_t>(l)] = static_cast<int64_t>(pl.stage.size() - r0);
  }
  if ((rc = plan_list_search(nq, k, q_list, lrow0, llen, &pl)) != AUR_OK) return rc;
  rc = stats_begin(c, s, nq, call.n_rows);
  if (rc == AUR_OK) rc = call.stage(queries_host, nq, k, scores_out, ids_out);
  if (rc == AUR_OK) rc = run_list_search(ix, c, s, pl, nq, k, nullptr, call.d_scores, call.d_ids);
  if (rc == AUR_OK) rc = stats_end(ix, c, s);
  if ((rc = call.finish(rc, nq, k, scores_out, ids_out)) != AUR_OK) return rc;
  if (snapshot_rows_out) *snapshot_rows_out = call.n_rows;
  return AUR_OK;
}

int aur_set_attrs(aur_index* ix, int32_t col, const int64_t* ids, const int32_t* codes, int64_t n) {
  if (!ix || n < 0 || (n > 0 && (!ids || !codes))) return fail(AUR_ERR_INVALID, "null argument");
  if (col < 2 || col >= kFiltCols) return fail(AUR_ERR_INVALID, "attribute columns are 2 .. %d", kFiltCols - 1);
  std::shared_lock<std::shared_mutex> rl(ix->rw);
  std::lock_guard<std::mutex> wk(ix->mu_write);
  CU_TRY(cudaSetDevice(ix->device));
  cudaStream_t s = ix->ingest_stream;
  int32_t* a = nullptr;
  {
    std::lock_guard<std::mutex> lk(ix->mu);
    a = ix->d_attr[col - 2];
  }
  if (!a) {   // first use: every row absent (-1), at the padded capacity like the tenant codes
    cudaError_t e = cudaMalloc(&a, static_cast<size_t>(ix->cap_pad) * 4);
    if (e != cudaSuccess) return fail(AUR_ERR_NOMEM, "attribute column: %s", cudaGetErrorString(e));
    e = cudaMemsetAsync(a, 0xFF, static_cast<size_t>(ix->cap_pad) * 4, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) { cudaFree(a); return fail(AUR_ERR_CUDA, "attribute column: %s", cudaGetErrorString(e)); }
    std::lock_guard<std::mutex> lk(ix->mu);
    ix->d_attr[col - 2] = a;
  }
  std::vector<int32_t> pairs;
  pairs.reserve(2 * static_cast<size_t>(n));
  resolve_ids(ix, ids, n, INT64_MAX, [&](int64_t i, int32_t row) { pairs.push_back(row); pairs.push_back(codes[i]); });
  if (pairs.empty()) return AUR_OK;
  CU_TRY(ix->attr_stage.reserve(pairs.size()));
  CU_TRY(cudaMemcpyAsync(ix->attr_stage.p, pairs.data(), pairs.size() * 4, cudaMemcpyHostToDevice, s));
  CU_TRY(launch_scatter_codes(ix->attr_stage.p, static_cast<int64_t>(pairs.size() / 2), a, s));
  CU_TRY(cudaStreamSynchronize(s));
  return AUR_OK;
}

int aur_search_filtered(aur_index* ix, const void* queries_host, int32_t nq, int32_t k, const int32_t* prog,
                        const int32_t* prog_offsets, int32_t n_programs, const uint32_t* bitmap, int64_t bitmap_words,
                        const int32_t* q_program, int64_t max_list_rows, float* scores_out, int64_t* ids_out,
                        int64_t* matched_out, int64_t* snapshot_rows_out) {
  int rc = check_list_args(ix, queries_host, nq, k, scores_out, ids_out);
  if (rc != AUR_OK) return rc;
  if ((rc = check_programs(ix, prog, prog_offsets, n_programs, bitmap, bitmap_words)) != AUR_OK) return rc;
  if (!q_program) return fail(AUR_ERR_INVALID, "q_program is required");
  for (int32_t q = 0; q < nq; ++q)
    if (q_program[q] < 0 || q_program[q] >= n_programs) return fail(AUR_ERR_INVALID, "q_program[%d] = %d is not a program", q, q_program[q]);
  if (max_list_rows < 0) return fail(AUR_ERR_INVALID, "max_list_rows < 0");

  HostCall call(ix);
  if ((rc = call.open()) != AUR_OK) return rc;
  SearchCtx* c = call.c;
  cudaStream_t s = call.s;
  const int64_t n_rows = call.n_rows;
  if ((rc = stats_begin(c, s, nq, n_rows)) != AUR_OK) return rc;
  std::vector<int64_t> tot;
  if ((rc = filter_count(ix, c, s, prog, prog_offsets, n_programs, bitmap, bitmap_words, n_rows, &tot)) != AUR_OK) return rc;
  if (n_programs == 1 && tot[0] > max_list_rows) {
    // dense: the matching rows as a row mask, and the masked scan aur_search_subset runs
    Scope sc;
    sc.match_mask = c->filt_mask.p;
    rc = call.stage(queries_host, nq, k, scores_out, ids_out);
    if (rc == AUR_OK) rc = search_enqueue(ix, c, c->stage_q.p, nq, k, sc, n_rows, call.d_scores, call.d_ids, nullptr, s);
  } else {
    // lists: every program's rows written on the device, in the order the host path stages them; items from the lengths
    std::vector<int64_t> lrow0(static_cast<size_t>(n_programs), 0);
    for (int32_t q = 1; q < n_programs; ++q)
      lrow0[static_cast<size_t>(q)] = lrow0[static_cast<size_t>(q - 1)] + tot[static_cast<size_t>(q - 1)];
    if ((rc = filter_write(ix, c, s, n_programs, tot, n_rows, false)) != AUR_OK) return rc;
    ListPlan pl;
    rc = plan_list_search(nq, k, q_program, lrow0, tot, &pl);
    if (rc == AUR_OK) rc = call.stage(queries_host, nq, k, scores_out, ids_out);
    if (rc == AUR_OK) rc = run_list_search(ix, c, s, pl, nq, k, c->filt_rows.p, call.d_scores, call.d_ids);
  }
  if (rc == AUR_OK) rc = stats_end(ix, c, s);
  if ((rc = call.finish(rc, nq, k, scores_out, ids_out)) != AUR_OK) return rc;
  if (matched_out) for (int32_t q = 0; q < n_programs; ++q) matched_out[q] = tot[static_cast<size_t>(q)];
  if (snapshot_rows_out) *snapshot_rows_out = n_rows;
  return AUR_OK;
}

int aur_filter_ids(aur_index* ix, const int32_t* prog, int32_t n_tokens, const uint32_t* bitmap, int64_t bitmap_words,
                   int64_t* ids_out, int64_t cap, int64_t* n_out) {
  if (!ix || !n_out || cap < 0 || (cap > 0 && !ids_out)) return fail(AUR_ERR_INVALID, "null argument");
  if (n_tokens < 0) return fail(AUR_ERR_INVALID, "n_tokens < 0");
  const int32_t off[2] = {0, n_tokens};
  int rc = check_programs(ix, prog, off, 1, bitmap, bitmap_words);
  if (rc != AUR_OK) return rc;
  HostCall call(ix);
  if ((rc = call.open()) != AUR_OK) return rc;
  SearchCtx* c = call.c;
  cudaStream_t s = call.s;
  std::vector<int64_t> tot;
  if ((rc = filter_count(ix, c, s, prog, off, 1, bitmap, bitmap_words, call.n_rows, &tot)) != AUR_OK) return rc;
  const int64_t n = tot[0], m = std::min(n, cap);
  if ((rc = filter_write(ix, c, s, 1, tot, call.n_rows, true)) != AUR_OK) return rc;
  std::vector<int64_t> got(static_cast<size_t>(m));
  if (m) CU_TRY(cudaMemcpyAsync(got.data(), c->filt_ids.p, static_cast<size_t>(m) * 8, cudaMemcpyDeviceToHost, s));
  CU_TRY(cudaStreamSynchronize(s));
  if (m) memcpy(ids_out, got.data(), static_cast<size_t>(m) * 8);
  *n_out = n;
  return AUR_OK;
}


// ---------------------------------------------------------------------------------------------------------------
// Fused cross-shard exchange (row-sharded corpus, one process per GPU).  Each rank owns one buffer in its HBM that
// every other rank maps through CUDA IPC; a shard's exact top-k rows are stored into all buffers by the finalize
// kernel itself and a flag per (parity, source rank) says when a slot is complete.  No NCCL call, no host
// round trip: local search -> peer stores -> merge is three kernels on one stream.
struct aur_exchange {
  int device = 0, rank = 0, world = 1, nq_max = 0, k_max = 0;
  size_t entries = 0, slot_stride = 0, parity_stride = 0, bytes = 0;   // slot_stride / parity_stride in 8-byte words
  uint64_t* local = nullptr;           // this rank's buffer (cudaMalloc, exported through cudaIpc)
  uint64_t* peer[8] = {};              // every rank's buffer as mapped here (peer[rank] == local)
  uint64_t* d_seq = nullptr;           // exchanges completed
  uint32_t* d_done = nullptr;          // merge kernel's block counter, then the status word
  bool connected = false;
};

int aur_merge_topk_dev(int32_t device, const double* in_scores64, const int64_t* in_ids, int32_t n_shards, int32_t nq,
                       int32_t k, float* out_scores, int64_t* out_ids, double* out_scores64, void* stream) {
  if (!in_scores64 || !in_ids || !out_scores || !out_ids) return fail(AUR_ERR_INVALID, "null argument");
  if (n_shards <= 0 || nq <= 0 || k <= 0 || k > kMaxK || n_shards * k > 2048) return fail(AUR_ERR_INVALID, "bad merge shape");
  if (aur_device_count() == 0) return fail(AUR_ERR_NO_DEVICE, "no CUDA device");
  CU_TRY(cudaSetDevice(device));
  CU_TRY(launch_merge_topk(in_scores64, in_ids, static_cast<size_t>(nq) * k, n_shards, nq, k, out_scores, out_ids,
                           out_scores64, static_cast<cudaStream_t>(stream)));
  return AUR_OK;
}

int aur_merge_topk_packed_dev(int32_t device, const void* packed, int32_t n_shards, int32_t nq, int32_t k,
                              float* out_scores, int64_t* out_ids, double* out_scores64, void* stream) {
  if (!packed || !out_scores || !out_ids) return fail(AUR_ERR_INVALID, "null argument");
  if (n_shards <= 0 || nq <= 0 || k <= 0 || k > kMaxK || n_shards * k > 2048) return fail(AUR_ERR_INVALID, "bad merge shape");
  if (aur_device_count() == 0) return fail(AUR_ERR_NO_DEVICE, "no CUDA device");
  CU_TRY(cudaSetDevice(device));
  const size_t plane = static_cast<size_t>(nq) * k;
  const double* s64 = static_cast<const double*>(packed);
  const int64_t* ids = static_cast<const int64_t*>(packed) + plane;
  CU_TRY(launch_merge_topk(s64, ids, 2 * plane, n_shards, nq, k, out_scores, out_ids, out_scores64,
                           static_cast<cudaStream_t>(stream)));
  return AUR_OK;
}

int aur_exchange_create(int32_t device, int32_t rank, int32_t world, int32_t nq_max, int32_t k_max, aur_exchange** out,
                        uint8_t* handle_out /* [64] */) {
  if (!out || !handle_out) return fail(AUR_ERR_INVALID, "null argument");
  *out = nullptr;
  if (world < 1 || world > 8 || rank < 0 || rank >= world) return fail(AUR_ERR_INVALID, "1 <= world <= 8, 0 <= rank < world");
  if (nq_max <= 0 || k_max <= 0 || k_max > kMaxK || world * k_max > 2048) return fail(AUR_ERR_INVALID, "bad nq_max / k_max");
  if (aur_device_count() == 0) return fail(AUR_ERR_NO_DEVICE, "no CUDA device");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
  CU_TRY(cudaSetDevice(device));
  aur_exchange* ex = new aur_exchange();
  ex->device = device; ex->rank = rank; ex->world = world; ex->nq_max = nq_max; ex->k_max = k_max;
  ex->entries = static_cast<size_t>(nq_max) * k_max;
  ex->slot_stride = 4 * ex->entries;                       // an entry = 4 tagged words (score lo / hi, id lo / hi)
  ex->parity_stride = static_cast<size_t>(world) * ex->slot_stride;
  ex->bytes = 2 * ex->parity_stride * 8 + 256;
  cudaError_t e = cudaMalloc(&ex->local, ex->bytes);
  if (e == cudaSuccess) e = cudaMemset(ex->local, 0, ex->bytes);
  if (e == cudaSuccess) e = cudaMalloc(&ex->d_seq, 8);
  if (e == cudaSuccess) e = cudaMemset(ex->d_seq, 0, 8);
  if (e == cudaSuccess) e = cudaMalloc(&ex->d_done, 16);      // [0] merge block counter, [1] status, [2] finalize block counter
  if (e == cudaSuccess) e = cudaMemset(ex->d_done, 0, 16);
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  cudaIpcMemHandle_t h;
  if (e == cudaSuccess && world > 1) e = cudaIpcGetMemHandle(&h, ex->local);
  if (e != cudaSuccess) {
    cudaFree(ex->local); cudaFree(ex->d_seq); cudaFree(ex->d_done); delete ex;
    return fail(AUR_ERR_CUDA, "aur_exchange_create: %s", cudaGetErrorString(e));
  }
  if (world > 1) memcpy(handle_out, &h, 64); else memset(handle_out, 0, 64);
  ex->peer[rank] = ex->local;
  ex->connected = world == 1;
  *out = ex;
  return AUR_OK;
}

int aur_exchange_connect(aur_exchange* ex, const uint8_t* all_handles /* [world][64], rank order */) {
  if (!ex || !all_handles) return fail(AUR_ERR_INVALID, "null argument");
  CU_TRY(cudaSetDevice(ex->device));
  for (int r = 0; r < ex->world; ++r) {
    if (r == ex->rank || ex->peer[r]) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, all_handles + static_cast<size_t>(r) * 64, 64);
    void* p = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) return fail(AUR_ERR_CUDA, "cudaIpcOpenMemHandle(rank %d): %s", r, cudaGetErrorString(e));
    ex->peer[r] = static_cast<uint64_t*>(p);
  }
  ex->connected = true;
  return AUR_OK;
}

int aur_exchange_close(aur_exchange* ex) {
  if (!ex) return AUR_OK;
  cudaSetDevice(ex->device);
  cudaDeviceSynchronize();
  for (int r = 0; r < ex->world; ++r)
    if (r != ex->rank && ex->peer[r]) cudaIpcCloseMemHandle(ex->peer[r]);
  cudaFree(ex->local); cudaFree(ex->d_seq); cudaFree(ex->d_done);
  delete ex;
  return AUR_OK;
}

int aur_exchange_status(aur_exchange* ex, int64_t* exchanges_done, int32_t* status) {
  if (!ex) return fail(AUR_ERR_INVALID, "null argument");
  CU_TRY(cudaSetDevice(ex->device));
  uint64_t seq = 0; uint32_t st[2] = {0, 0};
  CU_TRY(cudaMemcpy(&seq, ex->d_seq, 8, cudaMemcpyDeviceToHost));
  CU_TRY(cudaMemcpy(st, ex->d_done, 8, cudaMemcpyDeviceToHost));
  if (exchanges_done) *exchanges_done = static_cast<int64_t>(seq);
  if (status) *status = static_cast<int32_t>(st[1]);
  return AUR_OK;
}

int aur_search_exchange_dev(aur_index* ix, aur_exchange* ex, const void* queries_dev, int32_t nq, int32_t k,
                            float* scores_dev, int64_t* ids_dev, void* stream) {
  int rc = check_search_args(ix, queries_dev, nq, k, scores_dev, ids_dev);
  if (rc != AUR_OK) return rc;
  if (!ex || !ex->connected) return fail(AUR_ERR_INVALID, "exchange not connected");
  if (ex->device != ix->device) return fail(AUR_ERR_INVALID, "exchange and index live on different devices");
  if (nq > ex->nq_max || k > ex->k_max || static_cast<size_t>(nq) * k > ex->entries)
    return fail(AUR_ERR_INVALID, "batch %d x top-%d exceeds the exchange's %d x %d", nq, k, ex->nq_max, ex->k_max);
  if ((rc = check_batch(nq, k)) != AUR_OK) return rc;
  std::shared_lock<std::shared_mutex> rl(ix->rw);
  CU_TRY(cudaSetDevice(ix->device));
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : ix->stream;
  SearchCtx* c = nullptr;
  if ((rc = acquire_ctx(ix, s, &c)) != AUR_OK) return rc;
  std::lock_guard<std::mutex> cl(c->mu);
  FinalizeArgs::ExchangeOut eo{};
  eo.n_peers = ex->world;
  for (int r = 0; r < ex->world; ++r) eo.slot[r] = ex->peer[r] + static_cast<size_t>(ex->rank) * ex->slot_stride;
  eo.seq = ex->d_seq;
  eo.parity_stride = ex->parity_stride;
  const int64_t n_rows = ix->rows_pub.load(std::memory_order_acquire);
  Scope sc;
  if ((rc = stats_begin(c, s, nq, n_rows)) != AUR_OK) return rc;
  if ((rc = search_enqueue(ix, c, queries_dev, nq, k, sc, n_rows, nullptr, nullptr, nullptr, s, &eo)) != AUR_OK) return rc;
  if ((rc = stats_end(ix, c, s)) != AUR_OK) return rc;
  ExchangeParams p{};
  p.slots = ex->local;
  p.seq = ex->d_seq; p.done = ex->d_done; p.status = ex->d_done + 1;
  p.world = ex->world; p.rank = ex->rank; p.nq = nq; p.k = k;
  p.parity_stride = ex->parity_stride; p.slot_stride = ex->slot_stride;
  p.out_scores = scores_dev; p.out_ids = ids_dev;
  CU_TRY(launch_exchange_merge(p, s));
  c->last_launches += 1;
  CU_TRY(cudaEventRecord(c->ev_end, s));
  return AUR_OK;
}

int aur_cosine_pairs(int32_t device, const float* a_host, const float* b_host, int64_t n, int32_t dim, int32_t clamp,
                     double* out_host) {
  if (n < 0 || dim < 0) return fail(AUR_ERR_INVALID, "negative size");
  if (n == 0) return AUR_OK;
  if (!a_host || !b_host || !out_host) return fail(AUR_ERR_INVALID, "null argument");
  if (aur_device_count() == 0) return fail(AUR_ERR_NO_DEVICE, "no CUDA device: aurora_b200 has no CPU fallback");
  CU_TRY(cudaSetDevice(device));
  if (dim == 0) { for (int64_t i = 0; i < n; ++i) out_host[i] = 0.0; return AUR_OK; }
  float *da = nullptr, *db = nullptr; double* dout = nullptr;
  const size_t bytes = static_cast<size_t>(n) * dim * 4;
  cudaError_t e = cudaMalloc(&da, bytes);
  if (e == cudaSuccess) e = cudaMalloc(&db, bytes);
  if (e == cudaSuccess) e = cudaMalloc(&dout, static_cast<size_t>(n) * 8);
  if (e == cudaSuccess) e = cudaMemcpy(da, a_host, bytes, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(db, b_host, bytes, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = launch_cosine_pairs(da, db, n, dim, clamp, dout, nullptr);
  std::vector<double> tmp(static_cast<size_t>(n));
  if (e == cudaSuccess) e = cudaMemcpy(tmp.data(), dout, static_cast<size_t>(n) * 8, cudaMemcpyDeviceToHost);
  cudaFree(da); cudaFree(db); cudaFree(dout);
  if (e != cudaSuccess) return fail(AUR_ERR_CUDA, "cosine_pairs: %s", cudaGetErrorString(e));
  memcpy(out_host, tmp.data(), static_cast<size_t>(n) * 8);
  return AUR_OK;
}

int aur_dev_malloc(int32_t device, uint64_t bytes, void** out) {
  if (!out) return fail(AUR_ERR_INVALID, "null argument");
  *out = nullptr;
  if (aur_device_count() == 0) return fail(AUR_ERR_NO_DEVICE, "no CUDA device");
  CU_TRY(cudaSetDevice(device));
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, bytes ? bytes : 1);
  if (e != cudaSuccess) return fail(AUR_ERR_NOMEM, "cudaMalloc(%llu): %s", (unsigned long long)bytes, cudaGetErrorString(e));
  *out = p;
  return AUR_OK;
}
int aur_dev_free(int32_t device, void* p) {
  if (!p) return AUR_OK;
  CU_TRY(cudaSetDevice(device));
  CU_TRY(cudaFree(p));
  return AUR_OK;
}
int aur_memcpy_h2d(int32_t device, void* dst_dev, const void* src_host, uint64_t bytes) {
  if (bytes == 0) return AUR_OK;
  if (!dst_dev || !src_host) return fail(AUR_ERR_INVALID, "null argument");
  CU_TRY(cudaSetDevice(device));
  CU_TRY(cudaMemcpy(dst_dev, src_host, bytes, cudaMemcpyHostToDevice));
  return AUR_OK;
}
int aur_memcpy_d2h(int32_t device, void* dst_host, const void* src_dev, uint64_t bytes) {
  if (bytes == 0) return AUR_OK;
  if (!dst_host || !src_dev) return fail(AUR_ERR_INVALID, "null argument");
  CU_TRY(cudaSetDevice(device));
  CU_TRY(cudaDeviceSynchronize());
  CU_TRY(cudaMemcpy(dst_host, src_dev, bytes, cudaMemcpyDeviceToHost));
  return AUR_OK;
}

int aur_debug_tc_scores(aur_index* ix, const void* queries_dev, int32_t nq, int32_t cta_group, float* out_dev,
                        int32_t* n_ctas_out, void* stream) {
  if (!ix || !queries_dev || !out_dev) return fail(AUR_ERR_INVALID, "null argument");
  std::shared_lock<std::shared_mutex> rl(ix->rw);
  CU_TRY(cudaSetDevice(ix->device));
  if (!ix->tmap_ok) return fail(AUR_ERR_UNSUPPORTED, "index shape has no tensor-core path");
  if (nq <= 0 || nq > 2 * kTcQRows) return fail(AUR_ERR_INVALID, "1..%d queries", 2 * kTcQRows);
  int n_lists = 0;
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : ix->stream;
  SearchCtx* c = nullptr;
  int rc = acquire_ctx(ix, s, &c);
  if (rc != AUR_OK) return rc;
  std::lock_guard<std::mutex> cl(c->mu);
  rc = run_tc_block(ix, c, cta_group, queries_dev, nq, 32 + kSlack, ix->rows_pub.load(std::memory_order_acquire), out_dev,
                    &n_lists, s);
  if (rc != AUR_OK) return rc;
  CU_TRY(cudaMemsetAsync(c->cand_count.p, 0, 8 * kTcQRows * 4, s));  // no finalize ran to reset them
  if (n_ctas_out) *n_ctas_out = ix->sm_count & ~1;
  return AUR_OK;
}

}  // extern "C"
