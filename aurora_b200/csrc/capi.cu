// Host runtime + C ABI (include/aurora_b200.h).  Owns one corpus shard in HBM:
//   rows      [capacity, dim]  bf16, f32 or int8 (AUR_I8: quantized from bf16 on ingest), row-major (K-major for the
//                              MMA, 128-bit coalesced for everything else)
//   inv_norm  [capacity] f32   1/|row|; 0 for zero rows; NaN marks a tombstone
//   ids       [capacity] i64   caller ids;  user / org [capacity] i32 tenant codes
//   attr      up to 16 x [capacity] i32 attribute codes for device-evaluated filters (allocated on first aur_set_attrs)
// each on a growable virtual-memory mapping (VmmBuf): aur_reserve maps more rows at its end and nothing moves;
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
#include <map>
#include <memory>
#include <mutex>
#include <shared_mutex>
#include <string>
#include <type_traits>
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

// The driver's virtual memory management entry points (VmmRange), obtained as cuTensorMapEncodeTiled is.
struct VmmFns {
  decltype(&cuMemAddressReserve) reserve = nullptr;
  decltype(&cuMemAddressFree) free = nullptr;
  decltype(&cuMemCreate) create = nullptr;
  decltype(&cuMemRelease) release = nullptr;
  decltype(&cuMemMap) map = nullptr;
  decltype(&cuMemUnmap) unmap = nullptr;
  decltype(&cuMemSetAccess) set_access = nullptr;
  decltype(&cuMemGetAllocationGranularity) granularity = nullptr;
  bool ok = false;
};
const VmmFns& vmm_fns() {
  static VmmFns f;
  static std::once_flag once;
  std::call_once(once, [] {
    auto get = [](const char* name, auto* fn) {
      void* p = nullptr;
      cudaDriverEntryPointQueryResult qres;
      if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &qres) != cudaSuccess || qres != cudaDriverEntryPointSuccess) {
        cudaGetLastError();
        return false;
      }
      *fn = reinterpret_cast<std::remove_pointer_t<decltype(fn)>>(p);
      return true;
    };
    f.ok = get("cuMemAddressReserve", &f.reserve) && get("cuMemAddressFree", &f.free) && get("cuMemCreate", &f.create) &&
           get("cuMemRelease", &f.release) && get("cuMemMap", &f.map) && get("cuMemUnmap", &f.unmap) &&
           get("cuMemSetAccess", &f.set_access) && get("cuMemGetAllocationGranularity", &f.granularity);
  });
  return f;
}
cudaError_t vmm_err(CUresult r) {
  if (r == CUDA_SUCCESS) return cudaSuccess;
  return r == CUDA_ERROR_OUT_OF_MEMORY ? cudaErrorMemoryAllocation : cudaErrorUnknown;
}
CUmemAllocationProp vmm_prop(int device) {
  CUmemAllocationProp prop{};
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = device;
  return prop;
}

}  // namespace

namespace aur {
cudaError_t vmm_max_rows(size_t row_bytes, size_t* out) {
  size_t free_b = 0, total_b = 0;
  AUR_CU_RET(cudaMemGetInfo(&free_b, &total_b));
  *out = std::min(static_cast<size_t>(kMaxRows), total_b / std::max<size_t>(row_bytes, 1));
  return cudaSuccess;
}

cudaError_t VmmRange::open(int device, size_t max_bytes, size_t bytes) {
  release();
  const VmmFns& f = vmm_fns();
  if (!f.ok) return cudaErrorNotSupported;
  const CUmemAllocationProp prop = vmm_prop(device);
  size_t g = 0;
  AUR_CU_RET(vmm_err(f.granularity(&g, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED)));
  const size_t want = std::max(max_bytes, bytes);
  const size_t reserved = (want + g - 1) / g * g;
  CUdeviceptr b = 0;
  AUR_CU_RET(vmm_err(f.reserve(&b, reserved, g, 0, 0)));
  base_ = b; reserved_ = reserved; mapped_ = 0; gran_ = g; device_ = device;
  const cudaError_t e = grow(bytes);
  if (e != cudaSuccess) release();
  return e;
}

cudaError_t VmmRange::grow(size_t bytes) {
  bytes = (bytes + gran_ - 1) / gran_ * gran_;
  if (bytes <= mapped_) return cudaSuccess;
  if (bytes > reserved_) return cudaErrorMemoryAllocation;   // more than the device could ever hold
  const VmmFns& f = vmm_fns();
  const CUmemAllocationProp prop = vmm_prop(device_);
  const size_t add = bytes - mapped_;
  const CUdeviceptr at = base_ + mapped_;
  CUmemGenericAllocationHandle h = 0;
  AUR_CU_RET(vmm_err(f.create(&h, add, &prop, 0)));
  CUresult r = f.map(at, add, 0, h, 0);
  if (r == CUDA_SUCCESS) {
    CUmemAccessDesc acc{};
    acc.location = prop.location;
    acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    r = f.set_access(at, add, &acc, 1);
    if (r != CUDA_SUCCESS) f.unmap(at, add);
  }
  if (r != CUDA_SUCCESS) { f.release(h); return vmm_err(r); }
  chunks_.push_back(Chunk{h, mapped_, add});
  mapped_ = bytes;
  return cudaSuccess;
}

void VmmRange::shrink_to(size_t bytes) {
  const VmmFns& f = vmm_fns();
  while (!chunks_.empty() && chunks_.back().offset >= bytes) {
    const Chunk c = chunks_.back();
    f.unmap(base_ + c.offset, c.bytes);
    f.release(c.handle);
    chunks_.pop_back();
    mapped_ = c.offset;
  }
}

void VmmRange::release() {
  if (!base_) return;
  shrink_to(0);
  vmm_fns().free(base_, reserved_);
  base_ = 0; reserved_ = mapped_ = 0;
}

cudaError_t raise_smem_limit(const void* kern, size_t smem) {
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, size_t> raised;   // (kernel, device) -> limit set so far
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> g(mu);
  size_t& cur = raised[{kern, dev}];
  if (cur >= smem) return cudaSuccess;
  e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  if (e == cudaSuccess) cur = smem;
  return e;
}

int report_error(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
  g_err = buf;
  return code;
}
namespace {
int encode_tmap_2d(CUtensorMapDataType type, void* tmap, const void* base, uint64_t cols, uint64_t rows, uint64_t row_stride_bytes,
                   uint32_t box_cols, uint32_t box_rows) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return -1;
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {row_stride_bytes};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  return static_cast<int>(enc(static_cast<CUtensorMap*>(tmap), type, 2,
                              const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                              CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE));
}
}  // namespace
int encode_tmap_2d_bf16(void* tmap, const void* base, uint64_t cols, uint64_t rows, uint64_t row_stride_bytes,
                        uint32_t box_cols, uint32_t box_rows) {
  return encode_tmap_2d(CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, tmap, base, cols, rows, row_stride_bytes, box_cols, box_rows);
}
int encode_tmap_2d_u8(void* tmap, const void* base, uint64_t cols, uint64_t rows, uint64_t row_stride_bytes,
                      uint32_t box_cols, uint32_t box_rows) {
  return encode_tmap_2d(CU_TENSOR_MAP_DATA_TYPE_UINT8, tmap, base, cols, rows, row_stride_bytes, box_cols, box_rows);
}
}  // namespace aur

namespace {
int (&fail)(int, const char*, ...) = report_error;
}  // namespace

// Scratch and bookkeeping of ONE in-flight search.  Device-pointer searches are bound to the caller's stream
// (same stream -> same context -> stream order protects the scratch); host-buffer searches lease a context from the
// index's pool and run on its own stream, so N threads can search at once.
struct SearchCtx {
  std::mutex mu;                  // one enqueue at a time
  Stream stream;
  Event ev_begin, ev_k0, ev_k1, ev_fin, ev_end;
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
  DevBuf<int8_t> q_img;          // int8 shards: the tensor-core kernel's query image (launch_query_image_i8)
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
  HostBuf<uint32_t> h_totals;    // page-locked landing area of the count pass's totals (kFiltCallPrograms words)

  int init(int /* device: current */) {
    int lo = 0, hi = 0;
    AUR_TRY(cudaDeviceGetStreamPriorityRange(&lo, &hi));   // hi = numerically lowest = highest priority
    AUR_TRY(stream.create(cudaStreamNonBlocking, hi));
    AUR_TRY(ev_begin.create()); AUR_TRY(ev_k0.create());
    AUR_TRY(ev_k1.create());    AUR_TRY(ev_end.create());
    AUR_TRY(ev_fin.create());
    return AUR_OK;
  }
};

struct aur_index {
  std::shared_mutex rw;          // shared: searches and appends; exclusive: compaction, export, close
  std::mutex mu;                 // host metadata: id2row, live, options, the bound contexts
  std::mutex mu_write;           // one writer at a time (append / remove)
  int device = 0, dim = 0, dtype = 0;
  int64_t live = 0;
  // capacity, cap_pad and tmap change only in aur_reserve, published together under tmap_mu; a search copies its
  // tensor map under it (tc_tmap) when it launches.  A lock of its own: an append holds mu over its id bookkeeping,
  // and a launch does not wait for that.
  std::mutex tmap_mu;
  std::atomic<int64_t> capacity{0};
  std::atomic<int64_t> cap_pad{0};    // capacity rounded up to a whole tile (TMA boxes never straddle an allocation):
                                      // the rows mapped in every per-row array
  std::atomic<int64_t> rows_pub{0};   // rows visible to searches (published after the data landed)
  size_t elt = 2;                        // bytes per stored row element (int8 rows: 1)
  size_t qelt = 2;                       // bytes per query / input row element (bf16 for bf16 and int8 rows, f32 for f32)
  DevBuf<uint8_t> i8_stage;              // int8 shards: host bf16 rows on their way to the quantizer (writers hold mu_write)
  DevBuf<int32_t> tomb_rows;             // aur_remove: the rows it tombstones, one upload (writers hold mu_write)
  // per-row arrays on growable mappings (aur_reserve): their addresses never change
  VmmBuf<uint8_t> d_rows;
  VmmBuf<float> d_inv_norm;
  VmmBuf<int64_t> d_ids;
  VmmBuf<int32_t> d_user, d_org;
  AttrColumns attrs;                     // program columns 2.., cap_pad rows each (aur_set_attrs, writers hold mu_write)
  int64_t compactions = 0;               // aur_compact calls over the shard's life (bumped under the exclusive lock)
  DevBuf<uint32_t> live_bits;            // aur_live_bits: live and nonfinite words (writers hold mu_write)
  HostBuf<uint32_t> live_bits_host;      // (their page-locked landing area)
  std::mutex mu_export;                  // aur_export_rows' staging: one copy-out at a time
  HostBuf<uint8_t> export_stage;         // two halves, each filled by the ingest stream while the host drains the other
  Event export_ev[2];
  std::unordered_map<int64_t, int64_t> id2row;
  Stream stream;                         // the index's own stream: device-pointer calls with stream == NULL
  Stream ingest_stream;                  // host appends / tombstones, lowest priority so queries overtake them
  CUtensorMap tmap[2][2];  // [64-row, 128-row tiles][cta_group 1, 2]: box rows tile / cta_group
  bool tmap_ok = false;
  int sm_count = 0;
  size_t smem_optin = 0;
  int opt_kernel = AUR_KERNEL_AUTO;
  int opt_dbg_flags = 0;
  int opt_tc_tile = 0;           // corpus rows per tile: 0 = auto, 64, 128
  int opt_tc_stages = 0;         // cap on the TMA ring's depth: 0 = the deepest that fits
  int opt_tc_qregs = -1;         // query k-blocks in the MMA warpgroup's registers: -1 = auto, 0 = none, kTcQRegs
  std::atomic<uint32_t> opt_dbg_epoch{0};   // bring-up: start value of the contexts' launch counters (0 = 1)
  CtxPool<SearchCtx> ctxs;             // host-buffer calls (HostCall)
  std::unordered_map<cudaStream_t, std::unique_ptr<SearchCtx>> bound;   // device-pointer calls, by caller stream
  SearchCtx* last_ctx = nullptr;       // context of the most recently enqueued search (aur_get_stats)
};

namespace {

bool tc_layout(const aur_index* ix) {
  // int8 rows: 128 of them per 128-byte k-block, so the path needs dim % 128 == 0
  return ix->dtype != AUR_F32 && ix->dim % (ix->dtype == AUR_I8 ? kTcKBlockI8 : kTcKBlock) == 0 && ix->dim <= kTcMaxDim;
}

// The tensor maps of the rows over `capacity` rows into out (nothing for a shape without the tensor-core path).
int encode_tmaps(const aur_index* ix, int64_t capacity, CUtensorMap (&out)[2][2]) {
  if (!tc_layout(ix)) return AUR_OK;   // SIMT only
  const bool i8 = ix->dtype == AUR_I8;
  // rows past the capacity (a tile's tail, a whole half of the last tile of a pair) arrive as zeros
  for (int w = 0; w < 2; ++w)
    for (int g = 1; g <= 2; ++g) {
      const int tile_n = w ? kTcTileWide : kTcTileN;
      const uint64_t cols = static_cast<uint64_t>(ix->dim), rows = static_cast<uint64_t>(capacity);
      const uint32_t box_rows = static_cast<uint32_t>(tile_n / g);
      const int r = i8 ? encode_tmap_2d_u8(&out[w][g - 1], ix->d_rows.p, cols, rows, cols, kTcKBlockI8, box_rows)
                       : encode_tmap_2d_bf16(&out[w][g - 1], ix->d_rows.p, cols, rows, cols * 2, kTcKBlock, box_rows);
      if (r < 0) return fail(AUR_ERR_CUDA, "cuTensorMapEncodeTiled entry point not found");
      if (r != CUDA_SUCCESS) return fail(AUR_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d)", r);
    }
  return AUR_OK;
}

// A copy of one tensor map as last published: a launch passes it by value (__grid_constant__), so a launch enqueued
// before a growth keeps the map of the capacity it was enqueued under.
CUtensorMap tc_tmap(aur_index* ix, int wide, int cta_group) {
  std::lock_guard<std::mutex> lk(ix->tmap_mu);
  return ix->tmap[wide][cta_group - 1];
}

bool tc_shape_ok(const aur_index* ix, int k, bool filtered) {
  if (!ix->tmap_ok || filtered || k > kMaxK) return false;
  // candidate lists (k + slack per query) and the query block share the SM's shared memory with
  // the TMA ring: large k at large dim leaves no room for a pipeline
  return tc_pick_stages(k + kSlack, ix->dim, ix->smem_optin, kTcTileN, true) >= 2;
}

// The context of the device-pointer searches on the caller's stream s, made on first use.  It is never pooled and never
// drained: those calls are asynchronous, and stream order protects its scratch.
int bound_ctx(aur_index* ix, cudaStream_t s, SearchCtx** out) {
  std::lock_guard<std::mutex> lk(ix->mu);
  auto it = ix->bound.find(s);
  if (it == ix->bound.end()) {
    std::unique_ptr<SearchCtx> c(new SearchCtx());
    const int rc = c->init(ix->device);
    if (rc != AUR_OK) return rc;
    it = ix->bound.emplace(s, std::move(c)).first;
  }
  *out = it->second.get();
  return AUR_OK;
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

// One call with host buffers: the index's shared lock, its device, a context leased from the index's pool and locked
// for the call, the context's own stream, and the prefix published when the call began (open()).  The lease comes after
// the shared lock, so the stream is idle before the lock is released.  A search call stages its queries and outputs
// with stage().
struct HostCall {
  aur_index* ix;
  std::shared_lock<std::shared_mutex> rl;
  CtxLease<SearchCtx> c;
  std::unique_lock<std::mutex> cl;
  cudaStream_t s = nullptr;
  int64_t n_rows = 0;
  float* d_scores = nullptr;   // where the search writes its results: the caller's pinned buffers or the staging buffers
  int64_t* d_ids = nullptr;
  bool direct = false;

  explicit HostCall(aur_index* index) : ix(index), rl(index->rw) {}
  HostCall(const HostCall&) = delete;
  HostCall& operator=(const HostCall&) = delete;
  int open() {
    AUR_TRY(cudaSetDevice(ix->device));
    const int rc = ix->ctxs.lease(&c);
    if (rc != AUR_OK) return rc;
    cl = std::unique_lock<std::mutex>(c->mu);
    s = c->stream;
    n_rows = ix->rows_pub.load(std::memory_order_acquire);
    return AUR_OK;
  }
  // Uploads the queries to c->stage_q and picks the outputs: the caller's host buffers when both are given, page-locked
  // and mapped (direct_outputs), else the staging buffers.
  int stage(const void* queries_host, int32_t nq, int32_t k, float* scores_out, int64_t* ids_out) {
    const size_t qbytes = static_cast<size_t>(nq) * ix->dim * ix->qelt;
    const size_t nout = static_cast<size_t>(nq) * k;
    AUR_TRY(c->stage_q.reserve(qbytes));
    AUR_TRY(c->stage_scores.reserve(nout));
    AUR_TRY(c->stage_ids.reserve(nout));
    AUR_TRY(cudaMemcpyAsync(c->stage_q.p, queries_host, qbytes, cudaMemcpyHostToDevice, s));
    d_scores = c->stage_scores.p;
    d_ids = c->stage_ids.p;
    direct = scores_out && ids_out && direct_outputs(scores_out, ids_out, &d_scores, &d_ids);
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
// score dump (dbg) keeps 64-row tiles unless the index's tc_tile option asks for 128.
int tc_auto_tile(int ksel, int dim, size_t smem_optin, bool mask, bool dbg) {
  if (dbg) return kTcTileN;
  return tc_pick_stages(ksel, dim, smem_optin, kTcTileWide, mask) >= kTcWideMinStages ? kTcTileWide : kTcTileN;
}
// The tile width a launch runs: the index's tc_tile option, else tc_auto_tile.
int tc_tile(const aur_index* ix, int ksel, bool mask, bool dbg) {
  return ix->opt_tc_tile ? ix->opt_tc_tile : tc_auto_tile(ksel, ix->dim, ix->smem_optin, mask, dbg);
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
  const int tile_n = tc_tile(ix, ksel, mask, dbg != nullptr);
  // The width is settled (from the all-in-shared-memory layout); a 128-row launch then moves its first query k-blocks
  // into registers and spends the shared memory they leave on ring stages.
  // The bring-up switch that issues no MMAs (dbg_flags & 2) keeps the whole block in shared memory: without MMAs
  // nothing holds the warpgroup's four warps in step, and the one such run with register k-blocks stopped making progress.
  const bool i8 = ix->dtype == AUR_I8;   // (its launches keep the whole query image in shared memory: no tc_qregs)
  const int qregs = (!i8 && tile_n == kTcTileWide && ix->opt_tc_qregs != 0 && !(ix->opt_dbg_flags & 2) && ix->dim / kTcKBlock >= kTcQRegs) ? kTcQRegs : 0;
  // (what fits is decided without the registers too: they deepen a ring, they do not admit a larger k)
  if (tc_pick_stages(ksel, ix->dim, ix->smem_optin, tile_n, mask) < 2) return fail(AUR_ERR_UNSUPPORTED, "k too large for the tensor-core path's shared memory");
  int stages = tc_pick_stages(ksel, ix->dim, ix->smem_optin, tile_n, mask, qregs);
  if (ix->opt_tc_stages >= 2 && ix->opt_tc_stages < stages) stages = ix->opt_tc_stages;
  const size_t smem = tc_smem_bytes(stages, ksel, ix->dim, tile_n, mask, qregs);
  const size_t ncand = static_cast<size_t>(n_qblocks) * kTcQRows * n_lists * ksel;
  AUR_TRY(c->cand_a.reserve(ncand));
  const size_t npub = static_cast<size_t>(n_qblocks) * kTcQRows * (((n_lists + 1) & ~1) + 1);
  if (npub > c->pub.n) {
    AUR_TRY(c->pub.reserve(npub));
    AUR_TRY(cudaMemsetAsync(c->pub.p, 0, npub * 8, s));  // epoch 0 is never used by a launch
  }
  if (c->cand_count.n < 8 * kTcQRows) {
    AUR_TRY(c->cand_count.reserve(8 * kTcQRows));
    AUR_TRY(cudaMemsetAsync(c->cand_count.p, 0, 8 * kTcQRows * 4, s));
  }
  if (c->d_epoch.n == 0) {
    const uint32_t e0 = ix->opt_dbg_epoch.load() ? ix->opt_dbg_epoch.load() : 1u;
    AUR_TRY(c->d_epoch.reserve(1));
    AUR_TRY(cudaMemcpyAsync(c->d_epoch.p, &e0, 4, cudaMemcpyHostToDevice, s));   // pageable source: staged before return
  }
  if (i8) {
    AUR_TRY(c->q_img.reserve(static_cast<size_t>(nqb) * ix->dim * 2));
    AUR_TRY(launch_query_image_i8(static_cast<const __nv_bfloat16*>(q_dev), ix->dim, nqb, c->q_img.p, s));
    c->last_launches += 1;
  }
  ++c->epoch;
  TcParams p;
  p.q = i8 ? reinterpret_cast<const __nv_bfloat16*>(c->q_img.p) : static_cast<const __nv_bfloat16*>(q_dev);
  p.inv_norm = inv_norm ? inv_norm : ix->d_inv_norm.p;
  p.row_mask = row_mask; p.q_scope = q_scope;
  p.ids = ix->d_ids.p;
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
  const CUtensorMap tm = tc_tmap(ix, tile_n == kTcTileWide, cta_group);
  AUR_TRY(tc_launch(cta_group, tile_n, qregs, i8, grid, &tm, p, smem, s));
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
  AUR_TRY(cudaEventRecord(c->ev_begin, s));
  return AUR_OK;
}
int stats_end(aur_index* ix, SearchCtx* c, cudaStream_t s) {
  AUR_TRY(cudaEventRecord(c->ev_fin, s));
  AUR_TRY(cudaEventRecord(c->ev_end, s));
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
    AUR_TRY(dst.reserve(static_cast<size_t>(nqb) * n_groups * ksel));
    AUR_TRY(launch_reduce_lists(cur, nqb, n_lists, ksel, group, ix->d_ids.p, dst.p, s));
    c->last_launches += 1;
    cur = dst.p; n_lists = n_groups; in_a = !in_a;
  }
  FinalizeArgs fa{};
  fa.cand = cur; fa.n_lists = n_lists; fa.ksel = ksel;
  fa.counts = compact ? c->cand_count.p : nullptr;
  fa.epoch_bump = compact ? c->d_epoch.p : nullptr;
  fa.cand_read = c->cand_read.p + q0;
  fa.q = qb; fa.rows = ix->d_rows.p; fa.dtype = ix->dtype; fa.dim = ix->dim; fa.nq = nqb; fa.k = k;
  fa.ids = ix->d_ids.p;
  fa.out_scores = scores ? scores + static_cast<size_t>(q0) * k : nullptr;
  fa.out_ids = ids ? ids + static_cast<size_t>(q0) * k : nullptr;
  fa.out_scores64 = scores64 ? scores64 + static_cast<size_t>(q0) * k : nullptr;
  if (ex) { fa.ex = *ex; fa.ex.q0 = q0; }
  AUR_TRY(launch_finalize(fa, s));
  c->last_launches += 1;
  return AUR_OK;
}

constexpr int64_t kSimtChunk = 16 * kSimtSeg;   // rows the generic kernel scores per launch (32768)
constexpr int kSimtQBlock = 1024;               // queries per generic-kernel launch

// The generic kernel's tenant filter for the queries from q0 on: their own codes, unless the scope is a row subset or
// already folded into the inverse norms (inv).
FilterArgs simt_filter(const aur_index* ix, const Scope& sc, const float* inv, int q0) {
  FilterArgs f{ix->d_user.p, ix->d_org.p, nullptr, nullptr};
  if (sc.n_allow < 0 && sc.q_user && !inv) { f.q_user = sc.q_user + q0; f.q_org = sc.q_org ? sc.q_org + q0 : nullptr; }
  return f;
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
    return fail(AUR_ERR_UNSUPPORTED, "tensor-core path needs bf16 rows with dim %% 64 == 0 or int8 rows with dim %% 128 == 0, dim <= %d, "
                "no per-query tenant filter, and k small enough for its shared-memory lists at this dim", kTcMaxDim);
  c->last_kernel = kernel;
  AUR_TRY(c->cand_read.reserve(static_cast<size_t>(nq)));
  bool k_timed = false;
  const float* inv = nullptr;   // masked inverse norms (nullptr = the shard's own)
  if (subset && n_rows > 0) {
    AUR_TRY(c->masked_inv.reserve(static_cast<size_t>(ix->capacity) + 64));
    AUR_TRY(launch_fill_f32(c->masked_inv.p, nanf(""), n_rows, s));
    AUR_TRY(launch_scatter_inv_norm(ix->d_inv_norm.p, sc.allow_rows, sc.n_allow, n_rows, c->masked_inv.p, s));
    c->last_launches += 2;
    inv = c->masked_inv.p;
  } else if (sc.match_mask && n_rows > 0) {
    AUR_TRY(c->masked_inv.reserve(static_cast<size_t>(ix->capacity) + 64));
    AUR_TRY(launch_mask_match(ix->d_inv_norm.p, sc.match_mask, n_rows, c->masked_inv.p, s));
    ++c->last_launches;
    inv = c->masked_inv.p;
  } else if (kernel != AUR_KERNEL_SIMT && scoped_tc && n_rows > 0) {              // up to 32 scopes in the batch: row bit masks
    AUR_TRY(c->row_mask.reserve(static_cast<size_t>(ix->capacity) + 64));
    AUR_TRY(launch_row_scope_mask(ix->d_user.p, ix->d_org.p, sc.scope_tab, sc.n_scopes, n_rows, c->row_mask.p, s));
    ++c->last_launches;
  } else if (kernel != AUR_KERNEL_SIMT && sc.q_user != nullptr && sc.uniform != nullptr && n_rows > 0) {   // one scope for the whole batch
    AUR_TRY(c->masked_inv.reserve(static_cast<size_t>(ix->capacity) + 64));
    AUR_TRY(launch_mask_inv_norm(ix->d_inv_norm.p, ix->d_user.p, ix->d_org.p, sc.uniform[0], sc.uniform[1], n_rows, c->masked_inv.p, s));
    ++c->last_launches;
    inv = c->masked_inv.p;
  }

  // queries per launch: the generic kernel takes 1024; the tensor-core kernel 128 per CTA pair and up to four pairs side by
  // side on the same corpus tiles (fewer when k + slack is too large for the threshold exchange of that geometry)
  int qstep = kSimtQBlock;
  if (kernel == AUR_KERNEL_TC1) qstep = 2 * kTcQRows;
  else if (kernel == AUR_KERNEL_TC2) qstep = tc2_super_blocks(ix, ksel, 4) * 2 * kTcQRows;
  for (int q0 = 0; q0 < nq; q0 += qstep) {
    const int nqb = (nq - q0 < qstep) ? nq - q0 : qstep;
    const uint8_t* qb = static_cast<const uint8_t*>(q_dev) + static_cast<size_t>(q0) * ix->dim * ix->qelt;
    int n_lists = 0;
    if (kernel == AUR_KERNEL_SIMT) {
      if (n_rows == 0) {
        n_lists = 1;
        AUR_TRY(c->cand_a.reserve(static_cast<size_t>(nqb) * ksel));
        AUR_TRY(cudaMemsetAsync(c->cand_a.p, 0, static_cast<size_t>(nqb) * ksel * 8, s));
      } else {
        n_lists = static_cast<int>((n_rows + kSimtSeg - 1) / kSimtSeg);
        AUR_TRY(c->cand_a.reserve(static_cast<size_t>(nqb) * n_lists * ksel));
        AUR_TRY(c->score_chunk.reserve(static_cast<size_t>(nqb) * kSimtChunk));
        const FilterArgs f = simt_filter(ix, sc, inv, q0);
        if (!k_timed) AUR_TRY(cudaEventRecord(c->ev_k0, s));
        for (int64_t r0 = 0; r0 < n_rows; r0 += kSimtChunk) {
          const int64_t nr = std::min(n_rows - r0, kSimtChunk);
          AUR_TRY(launch_simt_scores(qb, ix->d_rows.p, ix->dtype, ix->dim, nqb, r0, nr, n_rows, inv ? inv : ix->d_inv_norm.p, f,
                                     c->score_chunk.p, s));
          AUR_TRY(launch_simt_select(c->score_chunk.p, nqb, r0, nr, ksel, ix->d_ids.p, c->cand_a.p, n_lists,
                                     static_cast<int>(r0 / kSimtSeg), s));
          c->last_launches += 2;
        }
        if (!k_timed) { AUR_TRY(cudaEventRecord(c->ev_k1, s)); k_timed = true; }
      }
    } else {
      if (!k_timed) AUR_TRY(cudaEventRecord(c->ev_k0, s));
      const bool use_mask = scoped_tc && n_rows > 0;
      int rc = run_tc_block(ix, c, kernel == AUR_KERNEL_TC1 ? 1 : 2, qb, nqb, ksel, n_rows, nullptr, &n_lists, s, inv,
                            use_mask ? c->row_mask.p : nullptr, use_mask ? sc.q_scope + q0 : nullptr);
      if (rc != AUR_OK) return rc;
      if (!k_timed) { AUR_TRY(cudaEventRecord(c->ev_k1, s)); k_timed = true; }
      c->last_launches += 1;
    }
    const int rc = candidate_tail(ix, c, s, qb, q0, nqb, k, n_lists, kernel != AUR_KERNEL_SIMT, scores, ids, scores64, ex);
    if (rc != AUR_OK) return rc;
  }
  if (!k_timed) { AUR_TRY(cudaEventRecord(c->ev_k0, s)); AUR_TRY(cudaEventRecord(c->ev_k1, s)); }
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
  uint8_t* dst = static_cast<uint8_t*>(ix->d_rows.p) + static_cast<size_t>(base) * ix->dim * ix->elt;
  if (ix->dtype == AUR_I8) {
    // bf16 rows in, quantized on s before the publish below: a search never sees an unquantized row.  Host rows pass
    // through a bounded device staging buffer, a slice at a time (stream order keeps the slices apart).
    const int64_t slice = rows_on_device ? n : std::min<int64_t>(n, 65536);
    const size_t in_row = static_cast<size_t>(ix->dim) * 2;
    if (!rows_on_device) AUR_TRY(ix->i8_stage.reserve(static_cast<size_t>(slice) * in_row));
    for (int64_t r0 = 0; r0 < n; r0 += slice) {
      const int64_t m = std::min(slice, n - r0);
      const uint8_t* src = static_cast<const uint8_t*>(rows) + static_cast<size_t>(r0) * in_row;
      if (!rows_on_device) {
        AUR_TRY(cudaMemcpyAsync(ix->i8_stage.p, src, static_cast<size_t>(m) * in_row, cudaMemcpyHostToDevice, s));
        src = ix->i8_stage.p;
      }
      AUR_TRY(launch_quantize_rows_i8(reinterpret_cast<const __nv_bfloat16*>(src), ix->dim, m,
                                      reinterpret_cast<int8_t*>(dst) + static_cast<size_t>(r0) * ix->dim, ix->d_inv_norm.p + base + r0, s));
    }
  } else {
    AUR_TRY(cudaMemcpyAsync(dst, rows, static_cast<size_t>(n) * ix->dim * ix->elt,
                            rows_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, s));
  }
  AUR_TRY(cudaMemcpyAsync(ix->d_ids.p + base, ids, static_cast<size_t>(n) * 8, cudaMemcpyHostToDevice, s));
  std::vector<int32_t> fill;
  if (!users) { fill.assign(static_cast<size_t>(n), 0); users = fill.data(); }
  AUR_TRY(cudaMemcpyAsync(ix->d_user.p + base, users, static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, s));
  std::vector<int32_t> fill2;
  if (!orgs) { fill2.assign(static_cast<size_t>(n), -1); orgs = fill2.data(); }
  AUR_TRY(cudaMemcpyAsync(ix->d_org.p + base, orgs, static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, s));
  if (ix->dtype != AUR_I8) AUR_TRY(launch_row_inv_norms(dst, ix->dtype, ix->dim, n, ix->d_inv_norm.p + base, s));
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
  for (int64_t row : dead) AUR_TRY(cudaMemcpyAsync(ix->d_inv_norm.p + row, &nanv, 4, cudaMemcpyHostToDevice, s));
  AUR_TRY(cudaStreamSynchronize(s));  // the data has landed (and the host staging vectors may go out of scope)
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
  AUR_TRY(c->stage_quser.reserve(nq));
  AUR_TRY(cudaMemcpyAsync(c->stage_quser.p, q_user, static_cast<size_t>(nq) * 4, cudaMemcpyHostToDevice, s));
  sc->q_user = c->stage_quser.p;
  if (q_org) {
    AUR_TRY(c->stage_qorg.reserve(nq));
    AUR_TRY(cudaMemcpyAsync(c->stage_qorg.p, q_org, static_cast<size_t>(nq) * 4, cudaMemcpyHostToDevice, s));
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
  AUR_TRY(c->scope_tab.reserve(64)); AUR_TRY(c->q_scope.reserve(static_cast<size_t>(nq)));
  AUR_TRY(cudaMemcpyAsync(c->scope_tab.p, tab.data(), tab.size() * 4, cudaMemcpyHostToDevice, s));
  AUR_TRY(cudaMemcpyAsync(c->q_scope.p, qs.data(), static_cast<size_t>(nq) * 4, cudaMemcpyHostToDevice, s));
  AUR_TRY(cudaStreamSynchronize(s));          // tab / qs are host temporaries
  sc->scope_tab = c->scope_tab.p; sc->q_scope = c->q_scope.p; sc->n_scopes = static_cast<int>(tab.size() / 2);
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
  if (ix->dtype == AUR_F32) return fail(AUR_ERR_UNSUPPORTED, "list search needs a bf16 or int8 index");
  return AUR_OK;
}
int check_lists(int32_t nq, const int64_t* list_ids, const int64_t* list_offsets, int32_t n_lists, const int32_t* q_list) {
  if (!list_offsets || !q_list || n_lists < 1) return fail(AUR_ERR_INVALID, "list_offsets, q_list and n_lists >= 1 are required");
  if (list_offsets[0] != 0) return fail(AUR_ERR_INVALID, "list_offsets[0] must be 0");
  for (int32_t l = 0; l < n_lists; ++l)
    if (list_offsets[l + 1] < list_offsets[l]) return fail(AUR_ERR_INVALID, "list_offsets decrease at list %d", l);
  if (list_offsets[n_lists] > 0 && !list_ids) return fail(AUR_ERR_INVALID, "list_ids is required");
  for (int32_t q = 0; q < nq; ++q)
    if (q_list[q] < 0 || q_list[q] >= n_lists) return fail(AUR_ERR_INVALID, "q_list[%d] = %d is not a list", q, q_list[q]);
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

// The list kernels' arguments for launch ln of block b, once the plan is in c->list_stage and the queries in c->stage_q.
ListParams list_params(const aur_index* ix, const SearchCtx* c, const ListPlan::Block& b, const ListPlan::Launch& ln,
                       const int32_t* list_rows, int ksel) {
  ListParams p{};
  p.q = reinterpret_cast<const __nv_bfloat16*>(c->stage_q.p + static_cast<size_t>(b.q0) * ix->dim * 2);
  p.rows = ix->d_rows.p;
  p.rows_i8 = ix->dtype == AUR_I8;
  p.inv_norm = ix->d_inv_norm.p;
  p.ids = ix->d_ids.p;
  p.items = reinterpret_cast<const ListItem*>(c->list_stage.p + ln.items);
  p.n_items = ln.n_items;
  p.list_rows = list_rows ? list_rows : c->list_stage.p;
  p.qidx = c->list_stage.p;
  p.scores = c->list_scores.p;
  p.cand = c->cand_a.p;
  p.dim = ix->dim; p.ksel = ksel; p.n_lists = b.n_segs;
  return p;
}

// The device side of a planned list search over the queries in c->stage_q: the plan is uploaded, every block's work
// items launched, and its candidates folded and re-ranked exactly into d_scores / d_ids.  list_rows: the lists' rows on
// the device (nullptr: at the front of the plan's staging).
int run_list_search(aur_index* ix, SearchCtx* c, cudaStream_t s, const ListPlan& pl, int32_t nq, int32_t k,
                    const int32_t* list_rows, float* d_scores, int64_t* d_ids) {
  const int ksel = k + kSlack;
  AUR_TRY(c->list_stage.reserve(pl.stage.size()));
  AUR_TRY(c->list_scores.reserve(std::max<size_t>(pl.max_slots, 1) * kSimtSeg));
  AUR_TRY(c->cand_a.reserve(pl.max_cand));
  AUR_TRY(c->cand_read.reserve(static_cast<size_t>(nq)));
  c->last_kernel = AUR_KERNEL_LIST;
  AUR_TRY(cudaMemcpyAsync(c->list_stage.p, pl.stage.data(), pl.stage.size() * 4, cudaMemcpyHostToDevice, s));
  for (size_t bi = 0; bi < pl.blocks.size(); ++bi) {
    const ListPlan::Block& b = pl.blocks[bi];
    const uint8_t* qb = c->stage_q.p + static_cast<size_t>(b.q0) * ix->dim * 2;
    AUR_TRY(cudaMemsetAsync(c->cand_a.p, 0, static_cast<size_t>(b.nqb) * b.n_segs * ksel * 8, s));   // 0 = empty slot
    if (bi == 0) AUR_TRY(cudaEventRecord(c->ev_k0, s));
    for (const ListPlan::Launch& ln : b.launches) {
      AUR_TRY(launch_list_search(list_params(ix, c, b, ln, list_rows, ksel), ln.max_nq, s));
      c->last_launches += 2;
    }
    if (bi == 0) AUR_TRY(cudaEventRecord(c->ev_k1, s));
    const int rc = candidate_tail(ix, c, s, qb, b.q0, b.nqb, k, b.n_segs, false, d_scores, d_ids, nullptr, nullptr);
    if (rc != AUR_OK) return rc;
  }
  return AUR_OK;
}

// Where pass `ps` of a filter evaluation (programs 32 ps .. 32 ps + 31) keeps its data: c->filt_mask holds one mask per
// pass, c->filt_counts every pass's 32 totals and then every pass's block counts.
struct FiltPass { uint32_t* mask; uint32_t* totals; uint32_t* counts; int n_programs; };
FiltPass filt_pass(SearchCtx* c, int ps, int n_programs, int64_t n_rows) {
  const size_t rows = static_cast<size_t>(std::max<int64_t>(n_rows, 1)), nb = static_cast<size_t>(std::max(filter_blocks(n_rows), 1));
  return FiltPass{c->filt_mask.p + ps * rows, c->filt_counts.p + ps * kFiltMaxPrograms,
                  c->filt_counts.p + static_cast<size_t>(filter_passes(n_programs)) * kFiltMaxPrograms + ps * kFiltMaxPrograms * nb,
                  filter_pass_programs(n_programs, ps)};
}

// Uploads checked programs, evaluates them over the snapshot's rows [0, n_rows) in passes of up to 32 programs (masks
// and counts in c->filt_mask / c->filt_counts, filt_pass) and enqueues the read-back of each program's number of
// matching rows into c->h_totals (one small copy for all passes).  Nothing waits: filter_totals reads them once the
// stream is idle.
int filter_count(aur_index* ix, SearchCtx* c, cudaStream_t s, const FiltProgs& fp, int64_t n_rows) {
  const int n_passes = filter_passes(fp.n_programs);
  const size_t nb = static_cast<size_t>(std::max(filter_blocks(n_rows), 1));
  AUR_TRY(c->h_totals.reserve(kFiltCallPrograms, cudaHostAllocPortable));
  AUR_TRY(c->filt_mask.reserve(static_cast<size_t>(n_passes) * static_cast<size_t>(std::max<int64_t>(n_rows, 1))));
  AUR_TRY(c->filt_counts.reserve(static_cast<size_t>(n_passes) * kFiltMaxPrograms * (1 + nb)));
  FiltParams p;
  AUR_TRY(filter_upload(fp, ix->d_user.p, ix->d_org.p, ix->attrs, c->filt_stage, s, &p));
  p.inv_norm = ix->d_inv_norm.p; p.n_rows = n_rows;
  for (int ps = 0; ps < n_passes; ++ps) {
    const FiltPass pass = filt_pass(c, ps, fp.n_programs, n_rows);
    AUR_TRY(launch_filter_count(filter_pass(p, ps), pass.mask, pass.counts, pass.totals, s));
    ++c->last_launches;
  }
  AUR_TRY(cudaMemcpyAsync(c->h_totals.p, c->filt_counts.p, static_cast<size_t>(n_passes) * kFiltMaxPrograms * 4,
                          cudaMemcpyDeviceToHost, s));
  return AUR_OK;
}

// After filter_count, with the stream idle: every program's number of matching rows (pass ps's totals are words
// 32 ps .. 32 ps + 31: program order).
void filter_totals(const SearchCtx* c, int32_t n_programs, std::vector<int64_t>* totals) {
  totals->assign(c->h_totals.p, c->h_totals.p + n_programs);
}

// After filter_count: every program's matching rows, ascending, program after program, into c->filt_rows (and with
// `with_ids` their ids into c->filt_ids).
int filter_write(aur_index* ix, SearchCtx* c, cudaStream_t s, int32_t n_programs, const std::vector<int64_t>& tot, int64_t n_rows,
                 bool with_ids) {
  int64_t total = 0;
  for (int64_t t : tot) total += t;
  if (total > INT32_MAX) return fail(AUR_ERR_UNSUPPORTED, "the programs of this call match too many rows for one call: split it");
  AUR_TRY(c->filt_rows.reserve(static_cast<size_t>(std::max<int64_t>(total, 1))));
  if (with_ids) AUR_TRY(c->filt_ids.reserve(static_cast<size_t>(std::max<int64_t>(total, 1))));
  int64_t base = 0;
  for (int ps = 0; ps < filter_passes(n_programs); ++ps) {
    const FiltPass fp = filt_pass(c, ps, n_programs, n_rows);
    AUR_TRY(launch_filter_write(fp.mask, fp.counts, fp.totals, fp.n_programs, n_rows, with_ids ? ix->d_ids.p : nullptr,
                                c->filt_rows.p + base, with_ids ? c->filt_ids.p + base : nullptr, s));
    if (n_rows > 0) c->last_launches += 2;
    for (int q = 0; q < fp.n_programs; ++q) base += tot[static_cast<size_t>(ps * kFiltMaxPrograms + q)];
  }
  return AUR_OK;
}

// After filter_count and its totals: the search of the queries in c->stage_q under the programs, into scores / ids.  One
// program matching more than max_list_rows rows runs the masked scan of aur_search_subset, anything else the list kernels.
int filtered_search(aur_index* ix, SearchCtx* c, cudaStream_t s, int32_t nq, int32_t k, const FiltProgs& fp,
                    const std::vector<int64_t>& tot, int64_t max_list_rows, int64_t n_rows, float* scores, int64_t* ids) {
  if (fp.n_programs == 1 && tot[0] > max_list_rows) {
    // dense: the matching rows as a row mask, and the masked scan aur_search_subset runs
    Scope sc;
    sc.match_mask = c->filt_mask.p;
    return search_enqueue(ix, c, c->stage_q.p, nq, k, sc, n_rows, scores, ids, nullptr, s);
  }
  // lists: every program's rows written on the device, in the order the host path stages them; items from the lengths
  std::vector<int64_t> lrow0(static_cast<size_t>(fp.n_programs), 0);
  for (int32_t q = 1; q < fp.n_programs; ++q)
    lrow0[static_cast<size_t>(q)] = lrow0[static_cast<size_t>(q - 1)] + tot[static_cast<size_t>(q - 1)];
  int rc = filter_write(ix, c, s, fp.n_programs, tot, n_rows, false);
  if (rc != AUR_OK) return rc;
  ListPlan pl;
  if ((rc = plan_list_search(nq, k, fp.q_program, lrow0, tot, &pl)) != AUR_OK) return rc;
  return run_list_search(ix, c, s, pl, nq, k, c->filt_rows.p, scores, ids);
}

// One shard's part of dense_legs: its call, its scope as the search reads it, and with programs every program's number
// of matching rows.
struct DensePart {
  std::unique_ptr<HostCall> call;
  Scope sc;
  int32_t scope[2] = {0, -1};     // the batch's one tenant scope (sc.uniform)
  std::vector<int32_t> allow;     // the allow-ids' rows
  ListPlan pl;                    // the lists' rows and work items
  std::vector<int64_t> tot;
};

// The host side of a staged call's scope: the tenant codes staged, the allow-ids resolved to rows of the published
// prefix, or the lists resolved and planned.  Programs need nothing before their count pass.
int prepare_scope(const DenseQuery& q, DensePart* pt) {
  HostCall& call = *pt->call;
  SearchCtx* c = call.c;
  if (q.n_allow >= 0) {
    // resolved metadata pre-filter: ids -> rows of the published prefix (unknown / newer ids drop out)
    pt->allow.reserve(static_cast<size_t>(q.n_allow));
    resolve_ids(call.ix, q.allow_ids, q.n_allow, call.n_rows, [&](int64_t, int32_t row) { pt->allow.push_back(row); });
    AUR_TRY(c->allow_rows.reserve(pt->allow.size() + 1));
    if (!pt->allow.empty())
      AUR_TRY(cudaMemcpyAsync(c->allow_rows.p, pt->allow.data(), pt->allow.size() * 4, cudaMemcpyHostToDevice, call.s));
    pt->sc.allow_rows = c->allow_rows.p;
    pt->sc.n_allow = static_cast<int64_t>(pt->allow.size());
    return AUR_OK;
  }
  if (q.q_list) {
    // staging (int32): [every named list's rows of the published prefix, sorted, once each][the plan's blocks]
    ListPlan& pl = pt->pl;
    std::vector<char> named(static_cast<size_t>(q.n_lists), 0);
    for (int32_t i = 0; i < q.nq; ++i) named[static_cast<size_t>(q.q_list[i])] = 1;
    std::vector<int64_t> lrow0(static_cast<size_t>(q.n_lists), 0), llen(static_cast<size_t>(q.n_lists), 0);
    for (int32_t l = 0; l < q.n_lists; ++l) {
      const size_t r0 = pl.stage.size();
      lrow0[static_cast<size_t>(l)] = static_cast<int64_t>(r0);
      if (!named[static_cast<size_t>(l)]) continue;
      resolve_ids(call.ix, q.list_ids + q.list_offsets[l], q.list_offsets[l + 1] - q.list_offsets[l], call.n_rows,
                  [&](int64_t, int32_t row) { pl.stage.push_back(row); });
      std::sort(pl.stage.begin() + r0, pl.stage.end());
      pl.stage.erase(std::unique(pl.stage.begin() + r0, pl.stage.end()), pl.stage.end());
      llen[static_cast<size_t>(l)] = static_cast<int64_t>(pl.stage.size() - r0);
    }
    return plan_list_search(q.nq, q.k, q.q_list, lrow0, llen, &pl);
  }
  if (q.q_user) return stage_tenant_scope(c, call.s, q.nq, q.q_user, q.q_org, pt->scope, &pt->sc);
  return AUR_OK;
}

}  // namespace

namespace aur {
int index_device(const aur_index* ix) { return ix->device; }
int index_bf16_queries(const aur_index* ix) { return ix->dtype == AUR_BF16 || ix->dtype == AUR_I8; }

AttrColumns& index_attrs(aur_index* ix) { return ix->attrs; }

int dense_legs(aur_index* const* shards, int n, const DenseQuery& q, const DenseLegsThen& then, float* scores_host,
               int64_t* ids_host) {
  std::vector<DensePart> parts(static_cast<size_t>(n));
  // shared locks in one order (by address), as the keyword legs take theirs
  std::vector<int> order(static_cast<size_t>(n));
  for (int s = 0; s < n; ++s) order[static_cast<size_t>(s)] = s;
  std::sort(order.begin(), order.end(), [&](int a, int b) { return std::less<aur_index*>()(shards[a], shards[b]); });
  for (int s : order) parts[static_cast<size_t>(s)].call.reset(new HostCall(shards[s]));
  int rc = AUR_OK;
  // every shard's queries, scope and (programs) count pass, then one wait for all the counts
  for (DensePart& pt : parts) {
    HostCall& call = *pt.call;
    if ((rc = call.open()) != AUR_OK) return rc;
    if ((rc = call.stage(q.queries, q.nq, q.k, n == 1 ? scores_host : nullptr, n == 1 ? ids_host : nullptr)) != AUR_OK) return rc;
    if ((rc = prepare_scope(q, &pt)) != AUR_OK) return rc;
    if ((rc = stats_begin(call.c, call.s, q.nq, call.n_rows)) != AUR_OK) return rc;
    if (q.fp && (rc = filter_count(call.ix, call.c, call.s, *q.fp, call.n_rows)) != AUR_OK) return rc;
  }
  if (q.fp)
    for (DensePart& pt : parts) {
      AUR_TRY(cudaSetDevice(pt.call->ix->device));
      AUR_TRY(cudaStreamSynchronize(pt.call->s));
      filter_totals(pt.call->c, q.fp->n_programs, &pt.tot);
    }
  std::vector<DenseLeg> legs;
  for (DensePart& pt : parts) {
    HostCall& call = *pt.call;
    AUR_TRY(cudaSetDevice(call.ix->device));
    if (q.fp)
      rc = filtered_search(call.ix, call.c, call.s, q.nq, q.k, *q.fp, pt.tot, q.max_list_rows, call.n_rows, call.d_scores, call.d_ids);
    else if (q.q_list)
      rc = run_list_search(call.ix, call.c, call.s, pt.pl, q.nq, q.k, nullptr, call.d_scores, call.d_ids);
    else
      rc = search_enqueue(call.ix, call.c, call.c->stage_q.p, q.nq, q.k, pt.sc, call.n_rows, call.d_scores, call.d_ids, nullptr, call.s);
    if (rc == AUR_OK) rc = stats_end(call.ix, call.c, call.s);
    if (rc != AUR_OK) return rc;
    legs.push_back(DenseLeg{call.ix->device, call.s, call.d_scores, call.d_ids, call.n_rows, &pt.tot, call.direct});
  }
  return then(legs);
}
}  // namespace aur

namespace {
// dense_legs over one shard, its lists copied into the caller's host buffers (directly written when they are
// page-locked).  They are written only when every kernel of the search was enqueued; on any failure they stay untouched.
int search_into_host(aur_index* ix, const DenseQuery& q, float* scores_out, int64_t* ids_out, int64_t* snapshot_rows_out,
                     int64_t* matched_out = nullptr) {
  return dense_legs(&ix, 1, q, [&](const std::vector<DenseLeg>& legs) -> int {
    const DenseLeg& l = legs[0];
    if (!l.direct) {   // into the caller's pageable buffers
      const size_t nout = static_cast<size_t>(q.nq) * q.k;
      AUR_TRY(cudaMemcpyAsync(scores_out, l.scores, nout * 4, cudaMemcpyDeviceToHost, l.stream));
      AUR_TRY(cudaMemcpyAsync(ids_out, l.ids, nout * 8, cudaMemcpyDeviceToHost, l.stream));
    }
    AUR_TRY(cudaStreamSynchronize(l.stream));
    if (matched_out) std::copy(l.matched->begin(), l.matched->end(), matched_out);
    if (snapshot_rows_out) *snapshot_rows_out = l.snapshot_rows;
    return AUR_OK;
  }, scores_out, ids_out);
}
}  // namespace

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
  if (cfg->dtype != AUR_BF16 && cfg->dtype != AUR_F32 && cfg->dtype != AUR_I8)
    return fail(AUR_ERR_INVALID, "dtype must be AUR_BF16, AUR_F32 or AUR_I8");
  if (cfg->dtype == AUR_BF16 && cfg->dim % 8 != 0) return fail(AUR_ERR_INVALID, "bf16 rows need dim %% 8 == 0");
  if (cfg->dtype == AUR_I8 && cfg->dim % 16 != 0) return fail(AUR_ERR_INVALID, "int8 rows need dim %% 16 == 0");
  if (cfg->capacity > 0x7FFFFFC0ll) return fail(AUR_ERR_INVALID, "capacity exceeds int32 row indexing");
  int ndev = aur_device_count();
  if (ndev == 0) return fail(AUR_ERR_NO_DEVICE, "no CUDA device: aurora_b200 has no CPU fallback");
  if (cfg->device < 0 || cfg->device >= ndev) return fail(AUR_ERR_INVALID, "device %d out of range", cfg->device);
  AUR_TRY(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  AUR_TRY(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9) return fail(AUR_ERR_UNSUPPORTED, "sm_%d%d device: this library is built for sm_90a only", prop.major, prop.minor);
  std::unique_ptr<aur_index> ix(new aur_index());
  ix->device = cfg->device; ix->dim = cfg->dim; ix->dtype = cfg->dtype; ix->capacity = cfg->capacity;
  ix->elt = cfg->dtype == AUR_BF16 ? 2 : (cfg->dtype == AUR_I8 ? 1 : 4);
  ix->qelt = cfg->dtype == AUR_F32 ? 4 : 2;
  ix->sm_count = prop.multiProcessorCount;
  ix->smem_optin = prop.sharedMemPerBlockOptin;
  ix->ctxs.device = cfg->device;
  int prio_lo = 0, prio_hi = 0;
  AUR_TRY(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
  AUR_TRY(ix->stream.create(cudaStreamNonBlocking, prio_hi));
  AUR_TRY(ix->ingest_stream.create(cudaStreamNonBlocking, prio_lo));
  ix->cap_pad = (cfg->capacity + kTcTileN - 1) / kTcTileN * kTcTileN;
  const size_t cap_pad = static_cast<size_t>(ix->cap_pad);
  AUR_TRY(ix->d_rows.open(ix->device, static_cast<size_t>(ix->dim) * ix->elt, cap_pad));
  AUR_TRY(ix->d_inv_norm.open(ix->device, 1, cap_pad));
  AUR_TRY(ix->d_ids.open(ix->device, 1, cap_pad));
  AUR_TRY(ix->d_user.open(ix->device, 1, cap_pad));
  AUR_TRY(ix->d_org.open(ix->device, 1, cap_pad));
  int rc = encode_tmaps(ix.get(), cfg->capacity, ix->tmap);
  if (rc != AUR_OK) return rc;
  ix->tmap_ok = tc_layout(ix.get());
  *out = ix.release();
  return AUR_OK;
}

int aur_reserve(aur_index* ix, int64_t capacity) {
  if (!ix) return fail(AUR_ERR_INVALID, "null index");
  if (capacity > kMaxRows) return fail(AUR_ERR_INVALID, "capacity exceeds int32 row indexing");
  std::shared_lock<std::shared_mutex> rl(ix->rw);   // a writer: searches and their enqueue go on
  std::lock_guard<std::mutex> wk(ix->mu_write);
  const int64_t old_cap = ix->capacity.load(), old_pad = ix->cap_pad.load();
  if (capacity <= old_cap) return AUR_OK;
  AUR_TRY(cudaSetDevice(ix->device));
  const int64_t pad = (capacity + kTcTileN - 1) / kTcTileN * kTcTileN;
  const size_t rows = static_cast<size_t>(pad);
  // the maps need only the rows' address, which never changes: encoded before anything grows
  CUtensorMap tm[2][2];
  int rc = encode_tmaps(ix, capacity, tm);
  if (rc != AUR_OK) return rc;
  // every array maps its new rows at its end, or none keeps them: the shard stays as it was on a failure
  const size_t b_rows = ix->d_rows.r.mapped(), b_inv = ix->d_inv_norm.r.mapped(), b_ids = ix->d_ids.r.mapped(),
               b_user = ix->d_user.r.mapped(), b_org = ix->d_org.r.mapped();
  cudaStream_t s = ix->ingest_stream;
  cudaError_t e = [&]() -> cudaError_t {
    AUR_CU_RET(ix->d_rows.grow(rows * ix->dim * ix->elt));
    AUR_CU_RET(ix->d_inv_norm.grow(rows));
    AUR_CU_RET(ix->d_ids.grow(rows));
    AUR_CU_RET(ix->d_user.grow(rows));
    AUR_CU_RET(ix->d_org.grow(rows));
    // the new rows start absent in the tenant columns, as in the attribute columns
    AUR_CU_RET(cudaMemsetAsync(ix->d_user.p + old_pad, 0xFF, static_cast<size_t>(pad - old_pad) * 4, s));
    AUR_CU_RET(cudaMemsetAsync(ix->d_org.p + old_pad, 0xFF, static_cast<size_t>(pad - old_pad) * 4, s));
    AUR_CU_RET(cudaStreamSynchronize(s));
    return ix->attrs.grow(old_pad, pad, s);   // (rolls its own columns back on a failure)
  }();
  if (e != cudaSuccess) {
    cudaStreamSynchronize(s);   // a tail memset may still be pending: nothing is unmapped under it
    cudaGetLastError();
    ix->d_rows.shrink_to_bytes(b_rows); ix->d_inv_norm.shrink_to_bytes(b_inv); ix->d_ids.shrink_to_bytes(b_ids);
    ix->d_user.shrink_to_bytes(b_user); ix->d_org.shrink_to_bytes(b_org);
    return fail(e == cudaErrorMemoryAllocation ? AUR_ERR_NOMEM : AUR_ERR_CUDA, "aur_reserve(%lld): %s (the shard keeps %lld rows)",
                (long long)capacity, cudaGetErrorString(e), (long long)old_cap);
  }
  std::lock_guard<std::mutex> lk(ix->tmap_mu);
  if (ix->tmap_ok) memcpy(ix->tmap, tm, sizeof tm);
  ix->cap_pad.store(pad);
  ix->capacity.store(capacity);
  return AUR_OK;
}

int aur_close(aur_index* ix) {
  if (!ix) return AUR_OK;
  cudaSetDevice(ix->device);
  cudaDeviceSynchronize();   // searches bound to caller streams may still be in flight
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
      AUR_TRY(cudaSetDevice(ix->device));
      AUR_TRY(cudaEventSynchronize(c->ev_end));
      AUR_TRY(cudaEventElapsedTime(&out->last_kernel_ms, c->ev_k0, c->ev_k1));
      AUR_TRY(cudaEventElapsedTime(&out->last_total_ms, c->ev_begin, c->ev_end));
      AUR_TRY(cudaEventElapsedTime(&out->last_finalize_ms, c->ev_k1, c->ev_fin));
      AUR_TRY(cudaEventElapsedTime(&out->last_merge_ms, c->ev_fin, c->ev_end));
      std::vector<uint32_t> n(std::min(static_cast<size_t>(c->last_nq), c->cand_read.n));
      AUR_TRY(cudaMemcpy(n.data(), c->cand_read.p, n.size() * 4, cudaMemcpyDeviceToHost));
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
  AUR_TRY(cudaSetDevice(ix->device));
  AUR_TRY(cudaDeviceSynchronize());
  std::vector<float> inv(static_cast<size_t>(n));
  AUR_TRY(cudaMemcpy(inv.data(), ix->d_inv_norm.p, sizeof(float) * n, cudaMemcpyDeviceToHost));
  AUR_TRY(cudaMemcpy(rows_out, ix->d_rows.p, static_cast<size_t>(n) * ix->dim * ix->elt, cudaMemcpyDeviceToHost));
  AUR_TRY(cudaMemcpy(ids_out, ix->d_ids.p, sizeof(int64_t) * n, cudaMemcpyDeviceToHost));
  if (user_out) AUR_TRY(cudaMemcpy(user_out, ix->d_user.p, sizeof(int32_t) * n, cudaMemcpyDeviceToHost));
  if (org_out) AUR_TRY(cudaMemcpy(org_out, ix->d_org.p, sizeof(int32_t) * n, cudaMemcpyDeviceToHost));
  // NaN = tombstone; an int8 row stored from a row with a NaN / inf (scale +inf, never returned) is live, reported as 2
  for (int64_t i = 0; i < n; ++i) {
    const float v = inv[static_cast<size_t>(i)];
    live_out[i] = v != v ? 0 : (ix->dtype == AUR_I8 && isinf(v) ? 2 : 1);
  }
  return AUR_OK;
}

int aur_read_rows(aur_index* ix, int64_t row0, int64_t n, void* rows_out, int64_t* ids_out) {
  if (!ix || (n > 0 && (!rows_out || !ids_out))) return fail(AUR_ERR_INVALID, "null argument");
  std::shared_lock<std::shared_mutex> rl(ix->rw);
  const int64_t rows = ix->rows_pub.load(std::memory_order_acquire);
  if (row0 < 0 || n < 0 || row0 + n > rows) return fail(AUR_ERR_INVALID, "rows [%lld, %lld) are not inside the published prefix of %lld",
                                                        (long long)row0, (long long)(row0 + n), (long long)rows);
  if (n == 0) return AUR_OK;
  AUR_TRY(cudaSetDevice(ix->device));
  const size_t rb = static_cast<size_t>(ix->dim) * ix->elt;
  AUR_TRY(cudaMemcpy(rows_out, static_cast<const uint8_t*>(ix->d_rows.p) + static_cast<size_t>(row0) * rb, static_cast<size_t>(n) * rb,
                     cudaMemcpyDeviceToHost));
  AUR_TRY(cudaMemcpy(ids_out, ix->d_ids.p + row0, static_cast<size_t>(n) * 8, cudaMemcpyDeviceToHost));
  return AUR_OK;
}

int aur_live_bits(aur_index* ix, uint32_t* live_out, uint32_t* nonfinite_out, int64_t words, int64_t* rows_out,
                  int64_t* compactions_out) {
  if (!ix || !live_out || !rows_out) return fail(AUR_ERR_INVALID, "null argument");
  if (ix->dtype == AUR_I8 && !nonfinite_out) return fail(AUR_ERR_INVALID, "an int8 shard needs nonfinite_out");
  // the writers' lock orders this after every append and remove that has returned; searches go on
  std::shared_lock<std::shared_mutex> rl(ix->rw);
  std::lock_guard<std::mutex> wk(ix->mu_write);
  const int64_t rows = ix->rows_pub.load(std::memory_order_acquire);
  const int64_t need = (rows + 31) / 32;
  if (words < need) return fail(AUR_ERR_INVALID, "%lld rows need %lld words, got %lld", (long long)rows, (long long)need, (long long)words);
  *rows_out = rows;
  if (compactions_out) *compactions_out = ix->compactions;
  if (rows == 0) return AUR_OK;
  AUR_TRY(cudaSetDevice(ix->device));
  const size_t w = static_cast<size_t>(need);
  AUR_TRY(ix->live_bits.reserve(2 * w));
  AUR_TRY(ix->live_bits_host.reserve(2 * w, cudaHostAllocDefault));
  cudaStream_t s = ix->ingest_stream;
  AUR_TRY(launch_live_bits(ix->d_inv_norm.p, rows, ix->dtype == AUR_I8, ix->live_bits.p, ix->live_bits.p + w, s));
  AUR_TRY(cudaMemcpyAsync(ix->live_bits_host.p, ix->live_bits.p, 2 * w * 4, cudaMemcpyDeviceToHost, s));
  AUR_TRY(cudaStreamSynchronize(s));
  memcpy(live_out, ix->live_bits_host.p, w * 4);
  if (nonfinite_out) memcpy(nonfinite_out, ix->live_bits_host.p + w, w * 4);
  return AUR_OK;
}

int aur_export_rows(aur_index* ix, int64_t row0, int64_t n, void* rows_out, int64_t* ids_out, int32_t* user_out,
                    int32_t* org_out) {
  if (!ix || (n > 0 && (!rows_out || !ids_out))) return fail(AUR_ERR_INVALID, "null argument");
  std::shared_lock<std::shared_mutex> rl(ix->rw);   // published rows never change under it: appends and searches go on
  const int64_t rows = ix->rows_pub.load(std::memory_order_acquire);
  if (row0 < 0 || n < 0 || row0 + n > rows) return fail(AUR_ERR_INVALID, "rows [%lld, %lld) are not inside the published prefix of %lld",
                                                        (long long)row0, (long long)(row0 + n), (long long)rows);
  if (n == 0) return AUR_OK;
  AUR_TRY(cudaSetDevice(ix->device));
  std::lock_guard<std::mutex> ek(ix->mu_export);
  const size_t rb = static_cast<size_t>(ix->dim) * ix->elt, per = rb + 16;   // a row, its id and its two tenant codes
  const int64_t chunk = std::max<int64_t>(1, static_cast<int64_t>((size_t(4) << 20) / per));   // rows per half: ~4 MB
  AUR_TRY(ix->export_stage.reserve(2 * static_cast<size_t>(chunk) * per, cudaHostAllocDefault));
  for (Event& ev : ix->export_ev)
    if (!ev.ev) AUR_TRY(ev.create(cudaEventDisableTiming));
  cudaStream_t s = ix->ingest_stream;
  const uint8_t* d_rows = static_cast<const uint8_t*>(ix->d_rows.p);
  auto half = [&](int64_t c) { return ix->export_stage.p + static_cast<size_t>(c & 1) * static_cast<size_t>(chunk) * per; };
  auto enqueue = [&](int64_t c) -> cudaError_t {   // chunk c's rows, ids, user and org codes into its half
    const int64_t r = row0 + c * chunk, m = std::min(chunk, row0 + n - r);
    uint8_t* h = half(c);
    AUR_CU_RET(cudaMemcpyAsync(h, d_rows + static_cast<size_t>(r) * rb, static_cast<size_t>(m) * rb, cudaMemcpyDeviceToHost, s));
    h += static_cast<size_t>(m) * rb;
    AUR_CU_RET(cudaMemcpyAsync(h, ix->d_ids.p + r, static_cast<size_t>(m) * 8, cudaMemcpyDeviceToHost, s));
    AUR_CU_RET(cudaMemcpyAsync(h + m * 8, ix->d_user.p + r, static_cast<size_t>(m) * 4, cudaMemcpyDeviceToHost, s));
    AUR_CU_RET(cudaMemcpyAsync(h + m * 12, ix->d_org.p + r, static_cast<size_t>(m) * 4, cudaMemcpyDeviceToHost, s));
    return cudaEventRecord(ix->export_ev[c & 1], s);
  };
  const int64_t n_chunks = (n + chunk - 1) / chunk;
  cudaError_t e = enqueue(0);
  for (int64_t c = 0; e == cudaSuccess && c < n_chunks; ++c) {
    if (c + 1 < n_chunks) e = enqueue(c + 1);   // the other half: its last contents were drained in the previous pass
    if (e == cudaSuccess) e = cudaEventSynchronize(ix->export_ev[c & 1]);
    if (e != cudaSuccess) break;
    const int64_t m = std::min(chunk, n - c * chunk), o = c * chunk;
    const uint8_t* h = half(c);
    memcpy(static_cast<uint8_t*>(rows_out) + static_cast<size_t>(o) * rb, h, static_cast<size_t>(m) * rb);
    h += static_cast<size_t>(m) * rb;
    memcpy(ids_out + o, h, static_cast<size_t>(m) * 8);
    if (user_out) memcpy(user_out + o, h + m * 8, static_cast<size_t>(m) * 4);
    if (org_out) memcpy(org_out + o, h + m * 12, static_cast<size_t>(m) * 4);
  }
  if (e != cudaSuccess) {
    cudaStreamSynchronize(s);   // no copy may still land in the staging after the lock is released
    return fail(AUR_ERR_CUDA, "aur_export_rows: %s", cudaGetErrorString(e));
  }
  return AUR_OK;
}

int aur_compact(aur_index* ix, int64_t* reclaimed) {
  if (!ix) return fail(AUR_ERR_INVALID, "null index");
  if (reclaimed) *reclaimed = 0;
  std::unique_lock<std::shared_mutex> wl(ix->rw);   // no search or append is being enqueued ...
  std::lock_guard<std::mutex> wk(ix->mu_write);
  ++ix->compactions;                                 // counted before anything can fail: a failed one may have moved rows
  AUR_TRY(cudaSetDevice(ix->device));
  AUR_TRY(cudaDeviceSynchronize());                  // ... and none is still running
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
  cudaError_t e = [&]() -> cudaError_t {
    AUR_CU_RET(d_map.reserve(static_cast<size_t>(chunk)));
    AUR_CU_RET(bounce.reserve(static_cast<size_t>(chunk) * ix->dim * ix->elt));
    AUR_CU_RET(b_inv.reserve(chunk));
    AUR_CU_RET(b_ids.reserve(chunk));
    AUR_CU_RET(b_user.reserve(chunk));
    AUR_CU_RET(b_org.reserve(chunk));
    return ix->attrs.any() ? b_attr.reserve(chunk) : cudaSuccess;
  }();
  if (e != cudaSuccess) return fail(AUR_ERR_NOMEM, "aur_compact: %s", cudaGetErrorString(e));
  cudaStream_t s = ix->ingest_stream;
  std::vector<int32_t> map_host(static_cast<size_t>(chunk));
  int64_t first_moved = 0;
  while (first_moved < nlive && order[static_cast<size_t>(first_moved)].first == first_moved) ++first_moved;   // untouched prefix
  e = [&]() -> cudaError_t {
    const size_t rb = static_cast<size_t>(ix->dim) * ix->elt;
    for (int64_t i0 = first_moved; i0 < nlive; i0 += chunk) {
      const int64_t m = (nlive - i0 < chunk) ? nlive - i0 : chunk;
      for (int64_t j = 0; j < m; ++j) map_host[static_cast<size_t>(j)] = static_cast<int32_t>(order[static_cast<size_t>(i0 + j)].first);
      AUR_CU_RET(cudaMemcpyAsync(d_map.p, map_host.data(), static_cast<size_t>(m) * 4, cudaMemcpyHostToDevice, s));
      AUR_CU_RET(launch_gather_rows(ix->d_rows.p, ix->d_inv_norm.p, ix->d_ids.p, ix->d_user.p, ix->d_org.p, d_map.p, m,
                                    static_cast<int>(ix->dim * ix->elt), bounce.p, b_inv.p, b_ids.p, b_user.p, b_org.p, s));
      AUR_CU_RET(cudaMemcpyAsync(ix->d_rows.p + static_cast<size_t>(i0) * rb, bounce.p, static_cast<size_t>(m) * rb, cudaMemcpyDeviceToDevice, s));
      AUR_CU_RET(cudaMemcpyAsync(ix->d_inv_norm.p + i0, b_inv.p, static_cast<size_t>(m) * 4, cudaMemcpyDeviceToDevice, s));
      AUR_CU_RET(cudaMemcpyAsync(ix->d_ids.p + i0, b_ids.p, static_cast<size_t>(m) * 8, cudaMemcpyDeviceToDevice, s));
      AUR_CU_RET(cudaMemcpyAsync(ix->d_user.p + i0, b_user.p, static_cast<size_t>(m) * 4, cudaMemcpyDeviceToDevice, s));
      AUR_CU_RET(cudaMemcpyAsync(ix->d_org.p + i0, b_org.p, static_cast<size_t>(m) * 4, cudaMemcpyDeviceToDevice, s));
      AUR_CU_RET(ix->attrs.gather(d_map.p, m, i0, b_attr.p, s));
      AUR_CU_RET(cudaStreamSynchronize(s));   // map_host is reused by the next chunk
    }
    // the freed rows are appended to again: their attributes start absent, as in a fresh column
    AUR_CU_RET(ix->attrs.clear(nlive, rows, s));
    return cudaStreamSynchronize(s);
  }();
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
      cs = ix->ctxs.contexts();
      for (auto& b : ix->bound) cs.push_back(b.second.get());
    }
    AUR_TRY(cudaSetDevice(ix->device));
    const uint32_t e = static_cast<uint32_t>(value);
    for (SearchCtx* c : cs) {
      std::lock_guard<std::mutex> cl(c->mu);
      if (c->d_epoch.n == 0) continue;
      AUR_TRY(cudaDeviceSynchronize());   // searches already enqueued on the context finish with their own counter
      AUR_TRY(cudaMemcpy(c->d_epoch.p, &e, 4, cudaMemcpyHostToDevice));
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
  if (strcmp(key, "tc_stages") == 0) {
    if (value != 0 && (value < 2 || value > kTcMaxStages)) return fail(AUR_ERR_INVALID, "tc_stages must be 0 (deepest) or 2 .. %d", kTcMaxStages);
    ix->opt_tc_stages = static_cast<int>(value);
    return AUR_OK;
  }
  if (strcmp(key, "tc_qregs") == 0) {
    if (value != -1 && value != 0 && (value != kTcQRegs || ix->dim / kTcKBlock < kTcQRegs))
      return fail(AUR_ERR_INVALID, "tc_qregs must be -1 (auto), 0, or %d at dim >= %d", kTcQRegs, kTcQRegs * kTcKBlock);
    ix->opt_tc_qregs = static_cast<int>(value);
    return AUR_OK;
  }
  if (strcmp(key, "dbg_flags") == 0) { ix->opt_dbg_flags = static_cast<int>(value); return AUR_OK; }
  return fail(AUR_ERR_INVALID, "unknown option '%s'", key);
}

int aur_sync(aur_index* ix) {
  if (!ix) return fail(AUR_ERR_INVALID, "null argument");
  AUR_TRY(cudaSetDevice(ix->device));
  AUR_TRY(cudaStreamSynchronize(ix->stream));
  return AUR_OK;
}

int aur_add(aur_index* ix, const void* rows_host, const int64_t* ids, const int32_t* user_codes,
            const int32_t* org_codes, int64_t n) {
  if (!ix) return fail(AUR_ERR_INVALID, "null index");
  std::shared_lock<std::shared_mutex> rl(ix->rw);
  std::lock_guard<std::mutex> wk(ix->mu_write);
  AUR_TRY(cudaSetDevice(ix->device));
  return add_common(ix, rows_host, false, ids, user_codes, org_codes, n, ix->ingest_stream);
}

int aur_add_dev(aur_index* ix, const void* rows_dev, const int64_t* ids_host, const int32_t* user_codes_host,
                const int32_t* org_codes_host, int64_t n, void* stream) {
  if (!ix) return fail(AUR_ERR_INVALID, "null index");
  std::shared_lock<std::shared_mutex> rl(ix->rw);
  std::lock_guard<std::mutex> wk(ix->mu_write);
  AUR_TRY(cudaSetDevice(ix->device));
  return add_common(ix, rows_dev, true, ids_host, user_codes_host, org_codes_host, n,
                    stream ? static_cast<cudaStream_t>(stream) : ix->ingest_stream);
}

int aur_remove(aur_index* ix, const int64_t* ids, int64_t n, int64_t* removed) {
  if (!ix || (n > 0 && !ids)) return fail(AUR_ERR_INVALID, "null argument");
  std::shared_lock<std::shared_mutex> rl(ix->rw);
  std::lock_guard<std::mutex> wk(ix->mu_write);
  AUR_TRY(cudaSetDevice(ix->device));
  if (removed) *removed = 0;
  if (n <= 0) return AUR_OK;
  AUR_TRY(ix->tomb_rows.reserve(static_cast<size_t>(n)));   // before id2row changes: a failure here removes nothing
  std::vector<int32_t> dead;
  {
    std::lock_guard<std::mutex> lk(ix->mu);
    for (int64_t i = 0; i < n; ++i) {
      auto it = ix->id2row.find(ids[i]);
      if (it == ix->id2row.end()) continue;
      dead.push_back(static_cast<int32_t>(it->second));
      ix->id2row.erase(it);
      --ix->live;
    }
  }
  const int64_t m = static_cast<int64_t>(dead.size());
  cudaStream_t s = ix->ingest_stream;
  if (m) {
    AUR_TRY(cudaMemcpyAsync(ix->tomb_rows.p, dead.data(), static_cast<size_t>(m) * 4, cudaMemcpyHostToDevice, s));
    AUR_TRY(launch_tombstone_rows(ix->tomb_rows.p, m, ix->d_inv_norm.p, s));
    AUR_TRY(cudaStreamSynchronize(s));   // dead is pageable host memory and goes out of scope
  }
  if (removed) *removed = m;
  return AUR_OK;
}

int aur_search_dev(aur_index* ix, const void* queries_dev, int32_t nq, int32_t k, const int32_t* q_user_dev,
                   const int32_t* q_org_dev, float* scores_dev, int64_t* ids_dev, double* scores64_dev, void* stream) {
  int rc = check_search_args(ix, queries_dev, nq, k, scores_dev, ids_dev);
  if (rc != AUR_OK) return rc;
  if ((rc = check_batch(nq, k)) != AUR_OK) return rc;
  std::shared_lock<std::shared_mutex> rl(ix->rw);
  AUR_TRY(cudaSetDevice(ix->device));
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : ix->stream;
  SearchCtx* c = nullptr;
  if ((rc = bound_ctx(ix, s, &c)) != AUR_OK) return rc;
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
  return aur_search_ex(ix, queries_host, nq, k, q_user, q_org, scores_out, ids_out, nullptr);
}

int aur_search_ex(aur_index* ix, const void* queries_host, int32_t nq, int32_t k, const int32_t* q_user,
                  const int32_t* q_org, float* scores_out, int64_t* ids_out, int64_t* snapshot_rows_out) {
  int rc = check_search_args(ix, queries_host, nq, k, scores_out, ids_out);
  if (rc != AUR_OK) return rc;
  if ((rc = check_batch(nq, k)) != AUR_OK) return rc;
  DenseQuery q{queries_host, nq, k};
  q.q_user = q_user; q.q_org = q_org;
  return search_into_host(ix, q, scores_out, ids_out, snapshot_rows_out);
}

int aur_search_subset(aur_index* ix, const void* queries_host, int32_t nq, int32_t k, const int64_t* allow_ids,
                      int64_t n_allow, float* scores_out, int64_t* ids_out) {
  if (n_allow < 0) return fail(AUR_ERR_INVALID, "n_allow < 0");
  int rc = check_search_args(ix, queries_host, nq, k, scores_out, ids_out);
  if (rc != AUR_OK) return rc;
  if (n_allow > 0 && !allow_ids) return fail(AUR_ERR_INVALID, "allow_ids / n_allow");
  if ((rc = check_batch(nq, k)) != AUR_OK) return rc;
  DenseQuery q{queries_host, nq, k};
  q.allow_ids = allow_ids; q.n_allow = n_allow;
  return search_into_host(ix, q, scores_out, ids_out, nullptr);
}

int aur_search_lists(aur_index* ix, const void* queries_host, int32_t nq, int32_t k, const int64_t* list_ids,
                     const int64_t* list_offsets, int32_t n_lists, const int32_t* q_list, float* scores_out,
                     int64_t* ids_out, int64_t* snapshot_rows_out) {
  int rc = check_list_args(ix, queries_host, nq, k, scores_out, ids_out);
  if (rc != AUR_OK) return rc;
  if ((rc = check_lists(nq, list_ids, list_offsets, n_lists, q_list)) != AUR_OK) return rc;
  DenseQuery q{queries_host, nq, k};
  q.list_ids = list_ids; q.list_offsets = list_offsets; q.n_lists = n_lists; q.q_list = q_list;
  return search_into_host(ix, q, scores_out, ids_out, snapshot_rows_out);
}

int aur_set_attrs(aur_index* ix, int32_t col, const int64_t* ids, const int32_t* codes, int64_t n) {
  if (!ix || n < 0 || (n > 0 && (!ids || !codes))) return fail(AUR_ERR_INVALID, "null argument");
  std::shared_lock<std::shared_mutex> rl(ix->rw);
  std::lock_guard<std::mutex> wk(ix->mu_write);
  AUR_TRY(cudaSetDevice(ix->device));
  std::vector<int32_t> pairs;
  pairs.reserve(2 * static_cast<size_t>(n));
  resolve_ids(ix, ids, n, INT64_MAX, [&](int64_t i, int32_t row) { pairs.push_back(row); pairs.push_back(codes[i]); });
  return ix->attrs.write(col, pairs, ix->cap_pad.load(), ix->ingest_stream);   // padded, like the tenant codes
}

int aur_search_filtered(aur_index* ix, const void* queries_host, int32_t nq, int32_t k, const int32_t* prog,
                        const int32_t* prog_offsets, int32_t n_programs, const uint32_t* bitmap, int64_t bitmap_words,
                        const int32_t* q_program, int64_t max_list_rows, float* scores_out, int64_t* ids_out,
                        int64_t* matched_out, int64_t* snapshot_rows_out) {
  int rc = check_list_args(ix, queries_host, nq, k, scores_out, ids_out);
  if (rc != AUR_OK) return rc;
  const FiltProgs fp{prog, prog_offsets, n_programs, bitmap, bitmap_words, q_program};
  if ((rc = filter_check_programs(fp)) != AUR_OK || (rc = ix->attrs.check(fp, "shard")) != AUR_OK ||
      (rc = filter_check_queries(fp, nq, max_list_rows)) != AUR_OK)
    return rc;
  DenseQuery q{queries_host, nq, k};
  q.fp = &fp; q.max_list_rows = max_list_rows;
  return search_into_host(ix, q, scores_out, ids_out, snapshot_rows_out, matched_out);
}

int aur_filter_ids(aur_index* ix, const int32_t* prog, int32_t n_tokens, const uint32_t* bitmap, int64_t bitmap_words,
                   int64_t* ids_out, int64_t cap, int64_t* n_out) {
  if (!ix || !n_out || cap < 0 || (cap > 0 && !ids_out)) return fail(AUR_ERR_INVALID, "null argument");
  if (n_tokens < 0) return fail(AUR_ERR_INVALID, "n_tokens < 0");
  const int32_t off[2] = {0, n_tokens};
  const FiltProgs fp{prog, off, 1, bitmap, bitmap_words, nullptr};
  int rc = filter_check_programs(fp);
  if (rc != AUR_OK || (rc = ix->attrs.check(fp, "shard")) != AUR_OK) return rc;
  HostCall call(ix);
  if ((rc = call.open()) != AUR_OK) return rc;
  SearchCtx* c = call.c;
  cudaStream_t s = call.s;
  std::vector<int64_t> tot;
  if ((rc = filter_count(ix, c, s, fp, call.n_rows)) != AUR_OK) return rc;
  AUR_TRY(cudaStreamSynchronize(s));
  filter_totals(c, 1, &tot);
  const int64_t n = tot[0], m = std::min(n, cap);
  if ((rc = filter_write(ix, c, s, 1, tot, call.n_rows, true)) != AUR_OK) return rc;
  std::vector<int64_t> got(static_cast<size_t>(m));
  if (m) AUR_TRY(cudaMemcpyAsync(got.data(), c->filt_ids.p, static_cast<size_t>(m) * 8, cudaMemcpyDeviceToHost, s));
  AUR_TRY(cudaStreamSynchronize(s));
  if (m) memcpy(ids_out, got.data(), static_cast<size_t>(m) * 8);
  *n_out = n;
  return AUR_OK;
}

int aur_filter_count(aur_index* ix, const int32_t* prog, int32_t n_tokens, const uint32_t* bitmap, int64_t bitmap_words,
                     int64_t* n_out) {
  if (!ix || !n_out) return fail(AUR_ERR_INVALID, "null argument");
  if (n_tokens < 0) return fail(AUR_ERR_INVALID, "n_tokens < 0");
  const int32_t off[2] = {0, n_tokens};
  const FiltProgs fp{prog, off, 1, bitmap, bitmap_words, nullptr};
  int rc = filter_check_programs(fp);
  if (rc != AUR_OK || (rc = ix->attrs.check(fp, "shard")) != AUR_OK) return rc;
  HostCall call(ix);
  if ((rc = call.open()) != AUR_OK) return rc;
  if ((rc = filter_count(ix, call.c, call.s, fp, call.n_rows)) != AUR_OK) return rc;
  AUR_TRY(cudaStreamSynchronize(call.s));
  std::vector<int64_t> tot;
  filter_totals(call.c, 1, &tot);
  *n_out = tot[0];
  return AUR_OK;
}

int aur_remove_filtered(aur_index* ix, const int32_t* prog, int32_t n_tokens, const uint32_t* bitmap, int64_t bitmap_words,
                        int64_t* ids_out, int64_t cap, int64_t* n_out) {
  if (!ix || !n_out || cap < 0 || (cap > 0 && !ids_out)) return fail(AUR_ERR_INVALID, "null argument");
  if (n_tokens < 0) return fail(AUR_ERR_INVALID, "n_tokens < 0");
  const int32_t off[2] = {0, n_tokens};
  const FiltProgs fp{prog, off, 1, bitmap, bitmap_words, nullptr};
  int rc = filter_check_programs(fp);
  if (rc != AUR_OK || (rc = ix->attrs.check(fp, "shard")) != AUR_OK) return rc;
  HostCall call(ix);
  // the writer lock, as aur_remove takes it: no append publishes rows and no other delete runs until the matching rows
  // are tombstones and their ids have left id2row, so the rows counted are the rows removed
  std::lock_guard<std::mutex> wk(ix->mu_write);
  if ((rc = call.open()) != AUR_OK) return rc;
  SearchCtx* c = call.c;
  cudaStream_t s = call.s;
  if ((rc = filter_count(ix, c, s, fp, call.n_rows)) != AUR_OK) return rc;
  AUR_TRY(cudaStreamSynchronize(s));
  std::vector<int64_t> tot;
  filter_totals(c, 1, &tot);
  const int64_t n = tot[0];
  if (n == 0 || n > cap) {   // nothing to remove, or no room for the ids: nothing removed, the caller retries
    *n_out = n;
    return AUR_OK;
  }
  if ((rc = filter_write(ix, c, s, 1, tot, call.n_rows, true)) != AUR_OK) return rc;
  AUR_TRY(launch_tombstone_rows(c->filt_rows.p, n, ix->d_inv_norm.p, s));
  std::vector<int64_t> got(static_cast<size_t>(n));
  AUR_TRY(cudaMemcpyAsync(got.data(), c->filt_ids.p, static_cast<size_t>(n) * 8, cudaMemcpyDeviceToHost, s));
  AUR_TRY(cudaStreamSynchronize(s));
  {
    std::lock_guard<std::mutex> lk(ix->mu);
    for (int64_t id : got) ix->live -= static_cast<int64_t>(ix->id2row.erase(id));
  }
  memcpy(ids_out, got.data(), static_cast<size_t>(n) * 8);
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
  DevBuf<uint64_t> local;              // this rank's buffer (exported through cudaIpc)
  uint64_t* peer[8] = {};              // every rank's buffer as mapped here (peer[rank] == local)
  DevBuf<uint64_t> d_seq;              // exchanges completed
  DevBuf<uint32_t> d_done;             // merge kernel's block counter, then the status word
  bool connected = false;
};

int aur_merge_topk_dev(int32_t device, const double* in_scores64, const int64_t* in_ids, int32_t n_shards, int32_t nq,
                       int32_t k, float* out_scores, int64_t* out_ids, double* out_scores64, void* stream) {
  if (!in_scores64 || !in_ids || !out_scores || !out_ids) return fail(AUR_ERR_INVALID, "null argument");
  if (n_shards <= 0 || nq <= 0 || k <= 0 || k > kMaxK || n_shards * k > 2048) return fail(AUR_ERR_INVALID, "bad merge shape");
  if (aur_device_count() == 0) return fail(AUR_ERR_NO_DEVICE, "no CUDA device");
  AUR_TRY(cudaSetDevice(device));
  AUR_TRY(launch_merge_topk(in_scores64, in_ids, static_cast<size_t>(nq) * k, n_shards, nq, k, out_scores, out_ids,
                            out_scores64, static_cast<cudaStream_t>(stream)));
  return AUR_OK;
}

int aur_merge_topk_packed_dev(int32_t device, const void* packed, int32_t n_shards, int32_t nq, int32_t k,
                              float* out_scores, int64_t* out_ids, double* out_scores64, void* stream) {
  if (!packed || !out_scores || !out_ids) return fail(AUR_ERR_INVALID, "null argument");
  if (n_shards <= 0 || nq <= 0 || k <= 0 || k > kMaxK || n_shards * k > 2048) return fail(AUR_ERR_INVALID, "bad merge shape");
  if (aur_device_count() == 0) return fail(AUR_ERR_NO_DEVICE, "no CUDA device");
  AUR_TRY(cudaSetDevice(device));
  const size_t plane = static_cast<size_t>(nq) * k;
  const double* s64 = static_cast<const double*>(packed);
  const int64_t* ids = static_cast<const int64_t*>(packed) + plane;
  AUR_TRY(launch_merge_topk(s64, ids, 2 * plane, n_shards, nq, k, out_scores, out_ids, out_scores64,
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
  AUR_TRY(cudaSetDevice(device));
  std::unique_ptr<aur_exchange> ex(new aur_exchange());
  ex->device = device; ex->rank = rank; ex->world = world; ex->nq_max = nq_max; ex->k_max = k_max;
  ex->entries = static_cast<size_t>(nq_max) * k_max;
  ex->slot_stride = 4 * ex->entries;                       // an entry = 4 tagged words (score lo / hi, id lo / hi)
  ex->parity_stride = static_cast<size_t>(world) * ex->slot_stride;
  ex->bytes = 2 * ex->parity_stride * 8 + 256;
  cudaIpcMemHandle_t h;
  const cudaError_t e = [&]() -> cudaError_t {
    AUR_CU_RET(ex->local.reserve(ex->bytes / 8));
    AUR_CU_RET(cudaMemset(ex->local.p, 0, ex->bytes));
    AUR_CU_RET(ex->d_seq.reserve(1));
    AUR_CU_RET(cudaMemset(ex->d_seq.p, 0, 8));
    AUR_CU_RET(ex->d_done.reserve(4));      // [0] merge block counter, [1] status, [2] finalize block counter
    AUR_CU_RET(cudaMemset(ex->d_done.p, 0, 16));
    AUR_CU_RET(cudaDeviceSynchronize());
    return world > 1 ? cudaIpcGetMemHandle(&h, ex->local.p) : cudaSuccess;
  }();
  if (e != cudaSuccess) return fail(AUR_ERR_CUDA, "aur_exchange_create: %s", cudaGetErrorString(e));
  if (world > 1) memcpy(handle_out, &h, 64); else memset(handle_out, 0, 64);
  ex->peer[rank] = ex->local.p;
  ex->connected = world == 1;
  *out = ex.release();
  return AUR_OK;
}

int aur_exchange_connect(aur_exchange* ex, const uint8_t* all_handles /* [world][64], rank order */) {
  if (!ex || !all_handles) return fail(AUR_ERR_INVALID, "null argument");
  AUR_TRY(cudaSetDevice(ex->device));
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
  delete ex;
  return AUR_OK;
}

int aur_exchange_status(aur_exchange* ex, int64_t* exchanges_done, int32_t* status) {
  if (!ex) return fail(AUR_ERR_INVALID, "null argument");
  AUR_TRY(cudaSetDevice(ex->device));
  uint64_t seq = 0; uint32_t st[2] = {0, 0};
  AUR_TRY(cudaMemcpy(&seq, ex->d_seq.p, 8, cudaMemcpyDeviceToHost));
  AUR_TRY(cudaMemcpy(st, ex->d_done.p, 8, cudaMemcpyDeviceToHost));
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
  AUR_TRY(cudaSetDevice(ix->device));
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : ix->stream;
  SearchCtx* c = nullptr;
  if ((rc = bound_ctx(ix, s, &c)) != AUR_OK) return rc;
  std::lock_guard<std::mutex> cl(c->mu);
  FinalizeArgs::ExchangeOut eo{};
  eo.n_peers = ex->world;
  for (int r = 0; r < ex->world; ++r) eo.slot[r] = ex->peer[r] + static_cast<size_t>(ex->rank) * ex->slot_stride;
  eo.seq = ex->d_seq.p;
  eo.parity_stride = ex->parity_stride;
  const int64_t n_rows = ix->rows_pub.load(std::memory_order_acquire);
  Scope sc;
  if ((rc = stats_begin(c, s, nq, n_rows)) != AUR_OK) return rc;
  if ((rc = search_enqueue(ix, c, queries_dev, nq, k, sc, n_rows, nullptr, nullptr, nullptr, s, &eo)) != AUR_OK) return rc;
  if ((rc = stats_end(ix, c, s)) != AUR_OK) return rc;
  ExchangeParams p{};
  p.slots = ex->local.p;
  p.seq = ex->d_seq.p; p.done = ex->d_done.p; p.status = ex->d_done.p + 1;
  p.world = ex->world; p.rank = ex->rank; p.nq = nq; p.k = k;
  p.parity_stride = ex->parity_stride; p.slot_stride = ex->slot_stride;
  p.out_scores = scores_dev; p.out_ids = ids_dev;
  AUR_TRY(launch_exchange_merge(p, s));
  c->last_launches += 1;
  AUR_TRY(cudaEventRecord(c->ev_end, s));
  return AUR_OK;
}

int aur_cosine_pairs(int32_t device, const float* a_host, const float* b_host, int64_t n, int32_t dim, int32_t clamp,
                     double* out_host) {
  if (n < 0 || dim < 0) return fail(AUR_ERR_INVALID, "negative size");
  if (n == 0) return AUR_OK;
  if (!a_host || !b_host || !out_host) return fail(AUR_ERR_INVALID, "null argument");
  if (aur_device_count() == 0) return fail(AUR_ERR_NO_DEVICE, "no CUDA device: aurora_b200 has no CPU fallback");
  AUR_TRY(cudaSetDevice(device));
  if (dim == 0) { for (int64_t i = 0; i < n; ++i) out_host[i] = 0.0; return AUR_OK; }
  DevBuf<float> da, db; DevBuf<double> dout;
  const size_t elems = static_cast<size_t>(n) * dim, bytes = elems * 4;
  std::vector<double> tmp(static_cast<size_t>(n));
  const cudaError_t e = [&]() -> cudaError_t {
    AUR_CU_RET(da.reserve(elems));
    AUR_CU_RET(db.reserve(elems));
    AUR_CU_RET(dout.reserve(static_cast<size_t>(n)));
    AUR_CU_RET(cudaMemcpy(da.p, a_host, bytes, cudaMemcpyHostToDevice));
    AUR_CU_RET(cudaMemcpy(db.p, b_host, bytes, cudaMemcpyHostToDevice));
    AUR_CU_RET(launch_cosine_pairs(da.p, db.p, n, dim, clamp, dout.p, nullptr));
    return cudaMemcpy(tmp.data(), dout.p, static_cast<size_t>(n) * 8, cudaMemcpyDeviceToHost);
  }();
  if (e != cudaSuccess) return fail(AUR_ERR_CUDA, "cosine_pairs: %s", cudaGetErrorString(e));
  memcpy(out_host, tmp.data(), static_cast<size_t>(n) * 8);
  return AUR_OK;
}

int aur_dev_malloc(int32_t device, uint64_t bytes, void** out) {
  if (!out) return fail(AUR_ERR_INVALID, "null argument");
  *out = nullptr;
  if (aur_device_count() == 0) return fail(AUR_ERR_NO_DEVICE, "no CUDA device");
  AUR_TRY(cudaSetDevice(device));
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, bytes ? bytes : 1);
  if (e != cudaSuccess) return fail(AUR_ERR_NOMEM, "cudaMalloc(%llu): %s", (unsigned long long)bytes, cudaGetErrorString(e));
  *out = p;
  return AUR_OK;
}
int aur_dev_free(int32_t device, void* p) {
  if (!p) return AUR_OK;
  AUR_TRY(cudaSetDevice(device));
  AUR_TRY(cudaFree(p));
  return AUR_OK;
}
int aur_memcpy_h2d(int32_t device, void* dst_dev, const void* src_host, uint64_t bytes) {
  if (bytes == 0) return AUR_OK;
  if (!dst_dev || !src_host) return fail(AUR_ERR_INVALID, "null argument");
  AUR_TRY(cudaSetDevice(device));
  AUR_TRY(cudaMemcpy(dst_dev, src_host, bytes, cudaMemcpyHostToDevice));
  return AUR_OK;
}
int aur_memcpy_d2h(int32_t device, void* dst_host, const void* src_dev, uint64_t bytes) {
  if (bytes == 0) return AUR_OK;
  if (!dst_host || !src_dev) return fail(AUR_ERR_INVALID, "null argument");
  AUR_TRY(cudaSetDevice(device));
  AUR_TRY(cudaDeviceSynchronize());
  AUR_TRY(cudaMemcpy(dst_host, src_dev, bytes, cudaMemcpyDeviceToHost));
  return AUR_OK;
}

int aur_debug_tc_scores(aur_index* ix, const void* queries_dev, int32_t nq, int32_t cta_group, float* out_dev,
                        int64_t out_cap, int32_t* n_ctas_out, int32_t* tile_n_out, void* stream) {
  if (!ix || !queries_dev || !out_dev) return fail(AUR_ERR_INVALID, "null argument");
  std::shared_lock<std::shared_mutex> rl(ix->rw);
  AUR_TRY(cudaSetDevice(ix->device));
  if (!ix->tmap_ok) return fail(AUR_ERR_UNSUPPORTED, "index shape has no tensor-core path");
  if (nq <= 0 || nq > 2 * kTcQRows) return fail(AUR_ERR_INVALID, "1..%d queries", 2 * kTcQRows);
  const int ksel = 32 + kSlack;
  const int n_ctas = ix->sm_count & ~1;   // run_tc_block's grid for up to 2 * kTcQRows queries, either cta_group
  const int tile_n = tc_tile(ix, ksel, false, true);
  const int64_t need = static_cast<int64_t>(n_ctas) * kTcQRows * tile_n;
  if (out_cap < need)
    return fail(AUR_ERR_INVALID, "out_dev holds %lld floats; the dump needs %d CTAs x %d x %d = %lld", (long long)out_cap, n_ctas,
                kTcQRows, tile_n, (long long)need);
  int n_lists = 0;
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : ix->stream;
  SearchCtx* c = nullptr;
  int rc = bound_ctx(ix, s, &c);
  if (rc != AUR_OK) return rc;
  std::lock_guard<std::mutex> cl(c->mu);
  rc = run_tc_block(ix, c, cta_group, queries_dev, nq, ksel, ix->rows_pub.load(std::memory_order_acquire), out_dev,
                    &n_lists, s);
  if (rc != AUR_OK) return rc;
  AUR_TRY(cudaMemsetAsync(c->cand_count.p, 0, 8 * kTcQRows * 4, s));  // no finalize ran to reset them
  if (n_ctas_out) *n_ctas_out = n_ctas;
  if (tile_n_out) *tile_n_out = tile_n;
  return AUR_OK;
}

int aur_debug_simt_scores(aur_index* ix, const void* queries_host, int32_t nq, const int32_t* q_user, const int32_t* q_org,
                          float* out_host, int64_t out_cap, int64_t* n_rows_out) {
  int rc = check_search_args(ix, queries_host, nq, 1, out_host, out_host);
  if (rc != AUR_OK) return rc;
  if (nq > kSimtQBlock) return fail(AUR_ERR_INVALID, "1..%d queries: one block of a search", kSimtQBlock);
  HostCall call(ix);
  if ((rc = call.open()) != AUR_OK) return rc;
  const int64_t n = call.n_rows;
  if (n_rows_out) *n_rows_out = n;
  if (out_cap < nq * n) return fail(AUR_ERR_INVALID, "out holds %lld floats; the dump needs %d x %lld", (long long)out_cap, nq, (long long)n);
  SearchCtx* c = call.c;
  if ((rc = call.stage(queries_host, nq, 1, nullptr, nullptr)) != AUR_OK) return rc;
  Scope sc;
  int32_t scope[2];
  if (q_user && (rc = stage_tenant_scope(c, call.s, nq, q_user, q_org, scope, &sc)) != AUR_OK) return rc;
  AUR_TRY(c->score_chunk.reserve(static_cast<size_t>(nq) * kSimtChunk));
  std::vector<float> chunk;
  for (int64_t r0 = 0; r0 < n; r0 += kSimtChunk) {   // the chunks and launches of search_enqueue's generic path
    const int64_t nr = std::min(n - r0, kSimtChunk);
    chunk.resize(static_cast<size_t>(nq) * nr);
    AUR_TRY(cudaMemsetAsync(c->score_chunk.p, 0xFF, chunk.size() * 4, call.s));   // NaN wherever the kernel writes nothing
    AUR_TRY(launch_simt_scores(c->stage_q.p, ix->d_rows.p, ix->dtype, ix->dim, nq, r0, nr, n, ix->d_inv_norm.p,
                               simt_filter(ix, sc, nullptr, 0), c->score_chunk.p, call.s));
    AUR_TRY(cudaMemcpyAsync(chunk.data(), c->score_chunk.p, chunk.size() * 4, cudaMemcpyDeviceToHost, call.s));
    AUR_TRY(cudaStreamSynchronize(call.s));
    for (int32_t q = 0; q < nq; ++q)
      std::copy(chunk.begin() + q * nr, chunk.begin() + (q + 1) * nr, out_host + q * n + r0);
  }
  return AUR_OK;
}

int aur_debug_list_scores(aur_index* ix, const void* queries_host, int32_t nq, const int64_t* list_ids,
                          const int64_t* list_offsets, int32_t n_lists, const int32_t* q_list, float* out_host, int64_t out_cap,
                          int64_t* n_rows_out) {
  int rc = check_list_args(ix, queries_host, nq, 1, out_host, out_host);
  if (rc != AUR_OK) return rc;
  if ((rc = check_lists(nq, list_ids, list_offsets, n_lists, q_list)) != AUR_OK) return rc;
  DenseQuery q{queries_host, nq, 1};
  q.list_ids = list_ids; q.list_offsets = list_offsets; q.n_lists = n_lists; q.q_list = q_list;
  DensePart pt;
  pt.call.reset(new HostCall(ix));
  HostCall& call = *pt.call;
  if ((rc = call.open()) != AUR_OK) return rc;
  const int64_t n = call.n_rows;
  if (n_rows_out) *n_rows_out = n;
  if (out_cap < nq * n) return fail(AUR_ERR_INVALID, "out holds %lld floats; the dump needs %d x %lld", (long long)out_cap, nq, (long long)n);
  SearchCtx* c = call.c;
  if ((rc = call.stage(queries_host, nq, 1, nullptr, nullptr)) != AUR_OK) return rc;
  if ((rc = prepare_scope(q, &pt)) != AUR_OK) return rc;   // the lists resolved and planned as aur_search_lists does
  const ListPlan& pl = pt.pl;
  AUR_TRY(c->list_stage.reserve(pl.stage.size()));
  AUR_TRY(c->list_scores.reserve(std::max<size_t>(pl.max_slots, 1) * kSimtSeg));
  AUR_TRY(c->cand_a.reserve(pl.max_cand));
  AUR_TRY(cudaMemcpyAsync(c->list_stage.p, pl.stage.data(), pl.stage.size() * 4, cudaMemcpyHostToDevice, call.s));
  std::fill(out_host, out_host + nq * n, nanf(""));
  std::vector<float> sc;
  for (const ListPlan::Block& b : pl.blocks)
    for (const ListPlan::Launch& ln : b.launches) {
      // every work item's scores: query b.q0 + qidx[q0 + g] against row list_rows[row0 + j] (the plan's host copy)
      const ListItem* items = reinterpret_cast<const ListItem*>(pl.stage.data() + ln.items);
      sc.resize(static_cast<size_t>(items[ln.n_items - 1].out + items[ln.n_items - 1].nq) * kSimtSeg);
      AUR_TRY(cudaMemsetAsync(c->list_scores.p, 0xFF, sc.size() * 4, call.s));   // NaN wherever the kernel writes nothing
      AUR_TRY(launch_list_search(list_params(ix, c, b, ln, nullptr, 1 + kSlack), ln.max_nq, call.s));
      AUR_TRY(cudaMemcpyAsync(sc.data(), c->list_scores.p, sc.size() * 4, cudaMemcpyDeviceToHost, call.s));
      AUR_TRY(cudaStreamSynchronize(call.s));
      for (int i = 0; i < ln.n_items; ++i) {
        const ListItem& it = items[i];
        for (int g = 0; g < it.nq; ++g) {
          float* row = out_host + (b.q0 + pl.stage[static_cast<size_t>(it.q0 + g)]) * n;
          const float* src = sc.data() + static_cast<size_t>(it.out + g) * kSimtSeg;
          for (int j = 0; j < it.n_rows; ++j) row[pl.stage[static_cast<size_t>(it.row0 + j)]] = src[j];
        }
      }
    }
  return AUR_OK;
}

}  // extern "C"
