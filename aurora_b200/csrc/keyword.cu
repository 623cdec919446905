// Device-resident BM25 keyword store (aur_kw_*, include/aurora_b200.h): the keyword leg of the hybrid query.
//
// Layout (one store on one GPU, standalone from aur_index but keyed by the same caller ids and tenant codes):
//   off   [cap + 1] i64   row r's postings are post[off[r] .. off[r + 1])
//   post  [grow]    uint2 (term id, tf), ascending term id within a row
//   len   [cap] i32 doc length (sum of tf);  ids [cap] i64;  user / org [cap] i32;  live [cap] u8
// Append-only with a published prefix, like the vector shard (capi.cu): a writer lands rows behind the prefix and then
// publishes the row count together with N (live docs), total_len and df[term] under one short host lock, so a search
// snapshots all four at once and scores exactly the prefix whose statistics it uses.  Tombstoning a published row
// (remove, upsert of an existing id) and growing the posting array take the store's exclusive lock: searches are
// host-synchronous and hold the shared lock until their results are back, so no search ever sees a tombstone its
// statistics do not account for.
//
// Scoring (DESIGN.md section 10) reproduces bm25.BM25Index.search's loop path bit for bit:
//   contribution = idf * tf * (K1 + 1) / (tf + K1 * (1 - B + B * dl / avgdl)), fp64, operation by operation
//   (__dmul_rn / __dadd_rn / __ddiv_rn: no FMA contraction), summed from 0.0 in the query's term order;
//   idf and avgdl come from the host (std::log, the libm call CPython's math.log makes).
// One pass over the postings serves a block of up to 256 queries: every warp walks one row's postings, looks each
// term up in the launch's term table and parks the row's contribution per unique term; then every lane sums its
// queries' terms in their order.  Selection is exact on (fp64 score desc, id asc) throughout: per-block candidate
// buffers pruned by the block's own k-th best, sorted lists per block, then sorted folds down to one list per query.
// aur_kw_search_multi runs the same search over several stores (one per GPU) as one corpus: N, df and total_len are
// summed over the stores' snapshots, every store scores its own prefix with the resulting idf / avgdl, and the per-store
// lists are merged on the host (DESIGN.md section 10, "Sharded store").  The hybrid query (hybrid.cu) runs the same
// steps through kw_legs and merges the per-store lists on the device instead.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>

#include <cmath>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <memory>
#include <mutex>
#include <shared_mutex>
#include <unordered_map>
#include <vector>

#include "../../include/aurora_b200.h"
#include "internal.h"

using namespace aur;

namespace {

constexpr double kK1 = 1.2, kB = 0.75;   // bm25.K1, bm25.B
constexpr int kKwThreads = 256;           // 8 warps per block
constexpr int kKwWarps = kKwThreads / 32;
constexpr int kKwRowsPerWarp = 4;         // rows a warp scores per round
constexpr int kKwRoundRows = kKwWarps * kKwRowsPerWarp;   // rows per round = most appends one query gets per round
constexpr int kKwBufCap = 256;            // candidate buffer per (block, query): flushed above kKwBufCap - kKwRoundRows
constexpr int kKwQBlock = 256;            // queries per launch
constexpr int kKwFoldCap = 2048;          // entries one fold block sorts
constexpr int64_t kKwMaxTerm = int64_t(1) << 28;
constexpr int kKwMaxStores = 64;         // stores one aur_kw_search_multi call takes

#define KW_TRY(expr)                                                                                             \
  do {                                                                                                           \
    cudaError_t e_ = (expr);                                                                                     \
    if (e_ != cudaSuccess)                                                                                       \
      return report_error(e_ == cudaErrorMemoryAllocation ? AUR_ERR_NOMEM : AUR_ERR_CUDA, "%s: %s (%s:%d)", #expr, \
                          cudaGetErrorString(e_), __FILE__, __LINE__);                                           \
  } while (0)

struct Cand { double s; int64_t id; };   // (score, id); worse = lower score, then higher id

__device__ __forceinline__ bool better(const Cand& a, const Cand& b) {
  return a.s > b.s || (a.s == b.s && a.id < b.id);
}
__device__ __forceinline__ Cand sentinel() { return Cand{-INFINITY, INT64_MAX}; }

// Bitonic sort of a[0..n) (n a power of two) best first, by threads t = 0..nt-1 of a group that sync() joins.
template <typename Sync>
__device__ void bitonic_sort(Cand* a, int n, int t, int nt, Sync sync) {
  for (int size = 2; size <= n; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = t; i < n / 2; i += nt) {
        const int lo = 2 * i - (i & (stride - 1));
        const int hi = lo + stride;
        const bool desc = (lo & size) == 0;   // best-first runs, alternating
        Cand x = a[lo], y = a[hi];
        if (desc ? better(y, x) : better(x, y)) { a[lo] = y; a[hi] = x; }
      }
      sync();
    }
  }
}

struct KwParams {
  // corpus (published prefix n_rows)
  const int64_t* off; const uint2* post; const int32_t* len; const int64_t* ids;
  const int32_t* user; const int32_t* org; const uint8_t* live; const uint8_t* allow;   // allow nullable
  int64_t n_rows;
  // launch term table
  const int32_t* hkey; const int32_t* hval; int hmask;   // open addressing: term id -> unique index (-1 = empty)
  const double* idf; int n_uniq;
  const int32_t* q_off; const int32_t* slot_u;           // query q's terms in summation order: slot_u[q_off[q] .. q_off[q+1])
  const int32_t* q_user; const int32_t* q_org;           // nullable: per-query tenant scope
  int nq, ksel;
  double avgdl;
  double* cval_global;   // when the per-warp contribution table does not fit shared memory: [grid * warps * n_uniq]
  Cand* buf;             // [grid][nq][kKwBufCap]
  Cand* lists;           // out: [nq][grid][ksel]
  int64_t rows_per_block;
};

__device__ __forceinline__ int lookup(const KwParams& p, int32_t term) {
  uint32_t h = (static_cast<uint32_t>(term) * 2654435761u) & static_cast<uint32_t>(p.hmask);
  for (;;) {
    const int32_t k = __ldg(p.hkey + h);
    if (k == term) return __ldg(p.hval + h);
    if (k < 0) return -1;
    h = (h + 1) & static_cast<uint32_t>(p.hmask);
  }
}

__device__ __forceinline__ double contribution(double idf, uint32_t tf_u, int32_t dl_i, double avgdl) {
  const double tf = static_cast<double>(tf_u), dl = static_cast<double>(dl_i);
  const double num = __dmul_rn(__dmul_rn(idf, tf), kK1 + 1.0);
  const double den = __dadd_rn(tf, __dmul_rn(kK1, __dadd_rn(1.0 - kB, __ddiv_rn(__dmul_rn(kB, dl), avgdl))));
  return __ddiv_rn(num, den);
}

// Warp w sorts buffer (block b, query q) of cnt entries in its shared area, keeps the best min(cnt, ksel) at the
// front of the buffer and returns how many.  thr_out: the ksel-th best when the buffer held at least ksel.
__device__ int warp_flush(const KwParams& p, Cand* area, Cand* gbuf, int cnt, int lane, Cand* thr_out) {
  for (int i = lane; i < kKwBufCap; i += 32) area[i] = i < cnt ? gbuf[i] : sentinel();
  __syncwarp();
  bitonic_sort(area, kKwBufCap, lane, 32, [] { __syncwarp(); });
  const int keep = cnt < p.ksel ? cnt : p.ksel;
  for (int i = lane; i < keep; i += 32) gbuf[i] = area[i];
  if (keep == p.ksel && thr_out) *thr_out = area[p.ksel - 1];
  __syncwarp();
  return keep;
}

__global__ void __launch_bounds__(kKwThreads) kw_score_kernel(KwParams p, int cval_in_smem) {
  extern __shared__ __align__(16) unsigned char smem[];
  Cand* thr = reinterpret_cast<Cand*>(smem);                         // [nq] block's ksel-th best so far
  Cand* sort_area = thr + p.nq;                                      // [warps][kKwBufCap]
  int* cnt = reinterpret_cast<int*>(sort_area + kKwWarps * kKwBufCap);   // [nq]
  double* cval_s = reinterpret_cast<double*>(smem + (((reinterpret_cast<size_t>(cnt + p.nq) - reinterpret_cast<size_t>(smem)) + 15) & ~size_t(15)));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double* cval = cval_in_smem ? cval_s + static_cast<size_t>(warp) * p.n_uniq
                              : p.cval_global + (static_cast<size_t>(blockIdx.x) * kKwWarps + warp) * p.n_uniq;
  for (int q = threadIdx.x; q < p.nq; q += blockDim.x) { thr[q] = sentinel(); cnt[q] = 0; }
  for (int u = lane; u < p.n_uniq; u += 32) cval[u] = 0.0;
  __syncthreads();
  Cand* gbuf = p.buf + static_cast<size_t>(blockIdx.x) * p.nq * kKwBufCap;
  const int64_t r_begin = static_cast<int64_t>(blockIdx.x) * p.rows_per_block;
  int64_t r_end = r_begin + p.rows_per_block;
  if (r_end > p.n_rows) r_end = p.n_rows;
  for (int64_t r0 = r_begin; r0 < r_end; r0 += kKwRoundRows) {
    for (int j = 0; j < kKwRowsPerWarp; ++j) {
      const int64_t row = r0 + warp * kKwRowsPerWarp + j;
      if (row >= r_end) break;
      if (!__ldg(p.live + row) || (p.allow && !__ldg(p.allow + row))) continue;
      const int64_t o0 = __ldg(p.off + row), o1 = __ldg(p.off + row + 1);
      const int32_t dl = __ldg(p.len + row);
      bool hit = false;
      for (int64_t i = o0 + lane; i < o1; i += 32) {
        const uint2 pt = __ldg(p.post + i);
        const int u = lookup(p, static_cast<int32_t>(pt.x));
        if (u >= 0) { cval[u] = contribution(__ldg(p.idf + u), pt.y, dl, p.avgdl); hit = true; }
      }
      if (!__any_sync(0xffffffffu, hit)) continue;
      __syncwarp();
      const int32_t ru = __ldg(p.user + row), ro = __ldg(p.org + row);
      const int64_t rid = __ldg(p.ids + row);
      for (int q = lane; q < p.nq; q += 32) {
        double s = 0.0;   // the loop path's defaultdict(float) start; adding a miss (0.0) leaves s bit-identical
        for (int g = __ldg(p.q_off + q), g1 = __ldg(p.q_off + q + 1); g < g1; ++g) s = __dadd_rn(s, cval[__ldg(p.slot_u + g)]);
        if (!(s > 0.0)) continue;
        if (p.q_user) {
          const int32_t qu = __ldg(p.q_user + q), qo = p.q_org ? __ldg(p.q_org + q) : -1;
          if (!(ru == qu || (qo >= 0 && ro == qo))) continue;
        }
        const Cand c{s, rid};
        if (!better(c, thr[q])) continue;
        const int pos = atomicAdd(cnt + q, 1);
        gbuf[static_cast<size_t>(q) * kKwBufCap + pos] = c;
      }
      __syncwarp();
      if (hit)
        for (int64_t i = o0 + lane; i < o1; i += 32) {
          const int u = lookup(p, static_cast<int32_t>(__ldg(p.post + i).x));
          if (u >= 0) cval[u] = 0.0;
        }
      __syncwarp();
    }
    __syncthreads();
    for (int q = warp; q < p.nq; q += kKwWarps) {
      const int c = cnt[q];
      if (c > kKwBufCap - kKwRoundRows) {
        Cand t = thr[q];
        const int keep = warp_flush(p, sort_area + warp * kKwBufCap, gbuf + static_cast<size_t>(q) * kKwBufCap, c, lane, &t);
        if (lane == 0) { cnt[q] = keep; thr[q] = t; }
      }
    }
    __syncthreads();
  }
  // the block's sorted best ksel per query
  for (int q = warp; q < p.nq; q += kKwWarps) {
    Cand* area = sort_area + warp * kKwBufCap;
    const int keep = warp_flush(p, area, gbuf + static_cast<size_t>(q) * kKwBufCap, cnt[q], lane, nullptr);
    Cand* out = p.lists + (static_cast<size_t>(q) * gridDim.x + blockIdx.x) * p.ksel;
    for (int i = lane; i < p.ksel; i += 32) out[i] = i < keep ? area[i] : sentinel();
  }
}

// [nq][n_lists][ksel] sorted lists -> [nq][ceil(n_lists / group)][ksel]; final: top-k as (fp64 score, id) with
// (-inf, -1) padding.  grid (n_groups, nq).
__global__ void __launch_bounds__(256) kw_fold_kernel(const Cand* in, int n_lists, int ksel, int group, int sort_n,
                                                      Cand* out, double* out_s, int64_t* out_ids, int k) {
  extern __shared__ __align__(16) unsigned char smem[];
  Cand* a = reinterpret_cast<Cand*>(smem);
  const int q = blockIdx.y, g = blockIdx.x;
  const int l0 = g * group, l1 = min(n_lists, l0 + group);
  const int n_in = (l1 - l0) * ksel;
  const Cand* src = in + (static_cast<size_t>(q) * n_lists + l0) * ksel;
  for (int i = threadIdx.x; i < sort_n; i += blockDim.x) a[i] = i < n_in ? src[i] : sentinel();
  __syncthreads();
  bitonic_sort(a, sort_n, threadIdx.x, blockDim.x, [] { __syncthreads(); });
  if (out) {
    Cand* dst = out + (static_cast<size_t>(q) * gridDim.x + g) * ksel;
    for (int i = threadIdx.x; i < ksel; i += blockDim.x) dst[i] = a[i];
  } else {
    for (int i = threadIdx.x; i < k; i += blockDim.x) {
      const Cand c = a[i];
      const bool pad = c.id == INT64_MAX;
      out_s[static_cast<size_t>(q) * k + i] = pad ? -INFINITY : c.s;
      out_ids[static_cast<size_t>(q) * k + i] = pad ? -1 : c.id;
    }
  }
}

// Compaction: postings of new row j (old row map[j]) -> new array at new_off[j]; one warp per row.
__global__ void kw_gather_postings(const uint2* post, const int64_t* old_off, const int32_t* map, const int64_t* new_off,
                                   int64_t n, uint2* out) {
  const int64_t w = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  const int64_t o0 = old_off[map[w]], o1 = old_off[map[w] + 1], d = new_off[w];
  for (int64_t i = lane; i < o1 - o0; i += 32) out[d + i] = post[o0 + i];
}

// Scratch of one in-flight search (a pool, so several host threads can search at once).
struct KwCtx {
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  DevBuf<unsigned char> tab;     // launch term table
  DevBuf<Cand> buf, lists_a, lists_b;
  DevBuf<double> cval, out_s;
  DevBuf<int64_t> out_ids;
  DevBuf<uint8_t> allow;
  DevBuf<int32_t> allow_rows;
  int launches = 0, terms = 0, spilled = 0;   // of the last search: kernels, most distinct terms in one launch,
                                              // launches whose contribution table spilled to global memory
  void release() {
    tab.release(); buf.release(); lists_a.release(); lists_b.release(); cval.release(); out_s.release(); out_ids.release();
    allow.release(); allow_rows.release();
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    if (stream) cudaStreamDestroy(stream);
  }
};

// flags[rows[i]] = v for the listed rows (allow-list rows of a search; tombstones)
__global__ void kw_scatter_flag(const int32_t* rows, int64_t n, uint8_t* flags, uint8_t v) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) flags[rows[i]] = v;
}

}  // namespace

struct aur_kw {
  std::shared_mutex rw;      // shared: searches and pure appends; exclusive: tombstones, posting growth, compaction
  std::mutex mu_write;       // one writer at a time (taken before rw)
  std::mutex mu_stat;        // the published prefix and its statistics, read and written together
  std::mutex mu_pool;
  int device = 0, sm_count = 0;
  size_t smem_optin = 0;
  int64_t capacity = 0;
  cudaStream_t stream = nullptr;
  // device
  int64_t* d_off = nullptr; int32_t* d_len = nullptr; int64_t* d_ids = nullptr;
  int32_t* d_user = nullptr; int32_t* d_org = nullptr; uint8_t* d_live = nullptr;
  uint2* d_post = nullptr; int64_t post_cap = 0;
  // host mirrors (the writer's bookkeeping; searches read only the published statistics)
  std::vector<int64_t> h_off{0};
  std::vector<int32_t> h_len, h_user, h_org;
  std::vector<int64_t> h_ids;
  std::vector<uint8_t> h_live;
  std::unordered_map<int64_t, int64_t> id2row;
  // published under mu_stat
  int64_t rows_pub = 0, post_pub = 0, n_live = 0, total_len = 0;
  std::vector<int64_t> df;
  // search pool + last search's stats
  std::vector<std::unique_ptr<KwCtx>> ctxs;
  std::vector<KwCtx*> idle;
  int last_launches = 0, last_terms = 0, last_spilled = 0;
  float last_ms = 0.f;
};

namespace {

int kw_ctx_acquire(aur_kw* kw, KwCtx** out) {
  {
    std::lock_guard<std::mutex> lk(kw->mu_pool);
    if (!kw->idle.empty()) { *out = kw->idle.back(); kw->idle.pop_back(); return AUR_OK; }
  }
  std::unique_ptr<KwCtx> c(new KwCtx());
  cudaError_t e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaEventCreate(&c->ev0);
  if (e == cudaSuccess) e = cudaEventCreate(&c->ev1);
  if (e != cudaSuccess) { c->release(); return report_error(AUR_ERR_CUDA, "search context: %s", cudaGetErrorString(e)); }
  std::lock_guard<std::mutex> lk(kw->mu_pool);
  *out = c.get();
  kw->ctxs.push_back(std::move(c));
  return AUR_OK;
}
void kw_ctx_release(aur_kw* kw, KwCtx* c) {
  std::lock_guard<std::mutex> lk(kw->mu_pool);
  kw->idle.push_back(c);
}

// Tombstone distinct published rows in one pass: their postings are gathered on the device and read back with one copy
// (their terms leave df), one kernel clears their live flags.  Caller holds the exclusive lock and mu_stat.
int tombstone_rows(aur_kw* kw, const std::vector<int64_t>& rows) {
  if (rows.empty()) return AUR_OK;
  const size_t m = rows.size();
  std::vector<int32_t> map(m);
  std::vector<int64_t> noff(m + 1, 0);
  for (size_t j = 0; j < m; ++j) {
    const size_t r = static_cast<size_t>(rows[j]);
    map[j] = static_cast<int32_t>(r);
    noff[j + 1] = noff[j] + (kw->h_off[r + 1] - kw->h_off[r]);
  }
  std::vector<uint2> terms(static_cast<size_t>(noff[m]));
  DevBuf<int32_t> d_map; DevBuf<int64_t> d_noff; DevBuf<uint2> d_terms;
  cudaStream_t s = kw->stream;
  cudaError_t e = d_map.reserve(m);
  if (e == cudaSuccess) e = d_noff.reserve(m + 1);
  if (e == cudaSuccess) e = d_terms.reserve(std::max<size_t>(terms.size(), 1));
  if (e == cudaSuccess) e = cudaMemcpyAsync(d_map.p, map.data(), m * 4, cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d_noff.p, noff.data(), (m + 1) * 8, cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) {
    kw_gather_postings<<<static_cast<unsigned>((static_cast<int64_t>(m) * 32 + 255) / 256), 256, 0, s>>>(
        kw->d_post, kw->d_off, d_map.p, d_noff.p, static_cast<int64_t>(m), d_terms.p);
    kw_scatter_flag<<<static_cast<unsigned>((m + 255) / 256), 256, 0, s>>>(d_map.p, static_cast<int64_t>(m), kw->d_live, 0);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess && !terms.empty())
    e = cudaMemcpyAsync(terms.data(), d_terms.p, terms.size() * 8, cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  d_map.release(); d_noff.release(); d_terms.release();
  if (e != cudaSuccess) return report_error(AUR_ERR_CUDA, "tombstone: %s", cudaGetErrorString(e));
  for (const uint2& p : terms) --kw->df[p.x];
  for (int64_t r : rows) {
    kw->h_live[static_cast<size_t>(r)] = 0;
    --kw->n_live;
    kw->total_len -= kw->h_len[static_cast<size_t>(r)];
  }
  return AUR_OK;
}

int grow_postings(aur_kw* kw, int64_t need) {
  if (need <= kw->post_cap) return AUR_OK;
  int64_t cap = std::max<int64_t>(need, kw->post_cap * 2);
  uint2* p = nullptr;
  KW_TRY(cudaMalloc(&p, static_cast<size_t>(cap) * 8));
  const int64_t used = kw->h_off.back();
  cudaError_t e = used ? cudaMemcpy(p, kw->d_post, static_cast<size_t>(used) * 8, cudaMemcpyDeviceToDevice) : cudaSuccess;
  if (e != cudaSuccess) { cudaFree(p); return report_error(AUR_ERR_CUDA, "posting growth: %s", cudaGetErrorString(e)); }
  cudaFree(kw->d_post);
  kw->d_post = p; kw->post_cap = cap;
  return AUR_OK;
}

// ---------------------------------------------------------------------------------------------------------- search
// One search, over one store or several stores taken as one corpus, in the steps both entry points share: every store's
// shared lock (in address order), a snapshot of each prefix and its statistics, the query blocks' launch tables built
// once from the summed statistics, every store's passes enqueued on its own device and stream, then each store's top-k
// collected.

struct KwQuery {   // the arguments of one search (aur_kw_search)
  const int32_t* terms; const int64_t* off; int32_t nq, k;
  const int32_t* user; const int32_t* org; const int64_t* allow; int64_t n_allow;
};

int kw_check_query(const KwQuery& q) {
  if (!q.off) return report_error(AUR_ERR_INVALID, "null argument");
  if (q.nq <= 0 || q.k <= 0) return report_error(AUR_ERR_INVALID, "nq and k must be positive");
  if (q.k > kMaxK) return report_error(AUR_ERR_UNSUPPORTED, "k > %d", kMaxK);
  if (q.off[0] != 0) return report_error(AUR_ERR_INVALID, "q_offsets[0] must be 0");
  for (int32_t i = 0; i < q.nq; ++i) if (q.off[i + 1] < q.off[i]) return report_error(AUR_ERR_INVALID, "q_offsets must be non-decreasing");
  if (q.off[q.nq] > 0 && !q.terms) return report_error(AUR_ERR_INVALID, "q_terms is required");
  if (q.n_allow < 0 || (q.n_allow > 0 && !q.allow)) return report_error(AUR_ERR_INVALID, "allow_ids / n_allow");
  return AUR_OK;
}

struct KwSnap { int64_t n_rows = 0, N = 0, total_len = 0; std::vector<int64_t> udf; };

// The published prefix and its statistics, df of the batch's distinct terms uniq, in one read.
void kw_snapshot(aur_kw* kw, const std::vector<int32_t>& uniq, KwSnap* s) {
  std::lock_guard<std::mutex> st(kw->mu_stat);
  s->n_rows = kw->rows_pub; s->N = kw->n_live; s->total_len = kw->total_len;
  s->udf.assign(uniq.size(), 0);
  for (size_t i = 0; i < uniq.size(); ++i)
    s->udf[i] = (uniq[i] >= 0 && uniq[i] < static_cast<int32_t>(kw->df.size())) ? kw->df[static_cast<size_t>(uniq[i])] : 0;
}

// One launch's query side, the same on every store: idf | hkey | hval | qoff | slot | q_user | q_org in one upload.
struct KwBlock {
  int q0 = 0, nqb = 0, nu = 0, hcap = 0;   // nu = 0: no query of the block has a live term
  size_t b_hk = 0, b_hv = 0, b_qo = 0, b_sl = 0, b_qu = 0, b_qg = 0;
  std::vector<unsigned char> tab;
};

// idf of every term with a live posting somewhere (N and udf: the corpus totals), then one table per kKwQBlock queries:
// the block's unique terms in an open-addressing hash, every query's terms as unique indices in summation order.
void kw_plan(const KwQuery& q, const std::vector<int32_t>& uniq, const std::vector<int64_t>& udf, int64_t N,
             std::vector<KwBlock>* blocks) {
  std::unordered_map<int32_t, double> idf;   // terms with a live posting (the loop path skips the others)
  for (size_t i = 0; i < uniq.size(); ++i)
    if (udf[i] > 0)
      idf[uniq[i]] = std::log(1.0 + (static_cast<double>(N - udf[i]) + 0.5) / (static_cast<double>(udf[i]) + 0.5));
  for (int32_t q0 = 0; q0 < q.nq; q0 += kKwQBlock) {
    KwBlock b;
    b.q0 = q0;
    b.nqb = std::min(kKwQBlock, q.nq - q0);
    const int nqb = b.nqb;
    std::vector<int32_t> ukeys;
    std::unordered_map<int32_t, int32_t> uidx;
    std::vector<int32_t> qoff(static_cast<size_t>(nqb) + 1, 0), slot;
    for (int i = 0; i < nqb; ++i) {
      std::vector<int32_t> seen;
      for (int64_t j = q.off[q0 + i]; j < q.off[q0 + i + 1]; ++j) {
        const int32_t t = q.terms[j];
        if (!idf.count(t) || std::find(seen.begin(), seen.end(), t) != seen.end()) continue;   // no live posting / repeated
        seen.push_back(t);
        auto it = uidx.find(t);
        if (it == uidx.end()) { it = uidx.emplace(t, static_cast<int32_t>(ukeys.size())).first; ukeys.push_back(t); }
        slot.push_back(it->second);
      }
      qoff[static_cast<size_t>(i) + 1] = static_cast<int32_t>(slot.size());
    }
    const int nu = b.nu = static_cast<int>(ukeys.size());
    if (nu == 0) { blocks->push_back(std::move(b)); continue; }
    int hcap = 16;
    while (hcap < 2 * nu) hcap <<= 1;
    b.hcap = hcap;
    std::vector<int32_t> hkey(static_cast<size_t>(hcap), -1), hval(static_cast<size_t>(hcap), -1);
    for (int u = 0; u < nu; ++u) {
      uint32_t h = (static_cast<uint32_t>(ukeys[static_cast<size_t>(u)]) * 2654435761u) & static_cast<uint32_t>(hcap - 1);
      while (hkey[h] >= 0) h = (h + 1) & static_cast<uint32_t>(hcap - 1);
      hkey[h] = ukeys[static_cast<size_t>(u)]; hval[h] = u;
    }
    std::vector<double> uidf(static_cast<size_t>(nu));
    for (int u = 0; u < nu; ++u) uidf[static_cast<size_t>(u)] = idf[ukeys[static_cast<size_t>(u)]];
    b.b_hk = 8 * static_cast<size_t>(nu); b.b_hv = b.b_hk + 4 * static_cast<size_t>(hcap);
    b.b_qo = b.b_hv + 4 * static_cast<size_t>(hcap); b.b_sl = b.b_qo + 4 * qoff.size();
    b.b_qu = b.b_sl + 4 * std::max<size_t>(slot.size(), 1); b.b_qg = b.b_qu + 4 * static_cast<size_t>(nqb);
    b.tab.assign(b.b_qg + 4 * static_cast<size_t>(nqb), 0);
    unsigned char* tab = b.tab.data();
    memcpy(tab, uidf.data(), 8 * static_cast<size_t>(nu));
    memcpy(tab + b.b_hk, hkey.data(), 4 * static_cast<size_t>(hcap));
    memcpy(tab + b.b_hv, hval.data(), 4 * static_cast<size_t>(hcap));
    memcpy(tab + b.b_qo, qoff.data(), 4 * qoff.size());
    if (!slot.empty()) memcpy(tab + b.b_sl, slot.data(), 4 * slot.size());
    if (q.user) memcpy(tab + b.b_qu, q.user + q0, 4 * static_cast<size_t>(nqb));
    std::vector<int32_t> qorg(static_cast<size_t>(nqb), -1);
    if (q.org) std::copy(q.org + q0, q.org + q0 + nqb, qorg.begin());
    memcpy(tab + b.b_qg, qorg.data(), 4 * static_cast<size_t>(nqb));
    blocks->push_back(std::move(b));
  }
}

// Enqueue one store's part of the search on c's stream: allow-list flags, then per block the table upload, the scoring
// pass over the store's prefix n_rows and the folds into c's [nq][k] output.  Nothing waits.
int kw_launch(aur_kw* kw, KwCtx* c, const KwQuery& q, const std::vector<KwBlock>& blocks, int64_t n_rows, int64_t N,
              double avgdl) {
  KW_TRY(cudaSetDevice(kw->device));
  cudaStream_t s = c->stream;
  const int k = q.k;
  c->launches = 0; c->terms = 0; c->spilled = 0;
  KW_TRY(cudaEventRecord(c->ev0, s));
  const uint8_t* d_allow = nullptr;
  if (q.allow) {
    std::vector<int32_t> rows;
    {
      std::lock_guard<std::mutex> st(kw->mu_stat);    // writers change id2row under it (and tombstone only exclusively)
      for (int64_t i = 0; i < q.n_allow; ++i) {
        auto it = kw->id2row.find(q.allow[i]);
        if (it != kw->id2row.end() && it->second < n_rows) rows.push_back(static_cast<int32_t>(it->second));
      }
    }
    KW_TRY(c->allow.reserve(static_cast<size_t>(std::max<int64_t>(n_rows, 1))));
    KW_TRY(c->allow_rows.reserve(std::max<size_t>(rows.size(), 1)));
    KW_TRY(cudaMemsetAsync(c->allow.p, 0, static_cast<size_t>(std::max<int64_t>(n_rows, 1)), s));
    if (!rows.empty()) {
      KW_TRY(cudaMemcpyAsync(c->allow_rows.p, rows.data(), rows.size() * 4, cudaMemcpyHostToDevice, s));
      kw_scatter_flag<<<static_cast<unsigned>((rows.size() + 255) / 256), 256, 0, s>>>(c->allow_rows.p, static_cast<int64_t>(rows.size()), c->allow.p, 1);
      KW_TRY(cudaGetLastError());
      c->launches += 1;
    }
    d_allow = c->allow.p;
  }
  const size_t nout = static_cast<size_t>(q.nq) * k;
  KW_TRY(c->out_s.reserve(nout));
  KW_TRY(c->out_ids.reserve(nout));
  for (const KwBlock& b : blocks) {
    const int nqb = b.nqb, nu = b.nu;
    double* o_s = c->out_s.p + static_cast<size_t>(b.q0) * k;
    int64_t* o_i = c->out_ids.p + static_cast<size_t>(b.q0) * k;
    if (nu == 0 || n_rows == 0 || N == 0) {   // nothing can match: padding only
      std::vector<double> ps(static_cast<size_t>(nqb) * k, -INFINITY);
      std::vector<int64_t> pi(static_cast<size_t>(nqb) * k, -1);
      KW_TRY(cudaMemcpyAsync(o_s, ps.data(), ps.size() * 8, cudaMemcpyHostToDevice, s));
      KW_TRY(cudaMemcpyAsync(o_i, pi.data(), pi.size() * 8, cudaMemcpyHostToDevice, s));
      continue;
    }
    KW_TRY(c->tab.reserve(b.tab.size()));
    KW_TRY(cudaMemcpyAsync(c->tab.p, b.tab.data(), b.tab.size(), cudaMemcpyHostToDevice, s));   // pageable: staged before return
    // geometry: blocks own contiguous row ranges of whole rounds
    const int64_t rounds = (n_rows + kKwRoundRows - 1) / kKwRoundRows;
    const int64_t grid = std::max<int64_t>(1, std::min<int64_t>(2 * kw->sm_count, rounds));
    const int64_t rpb = (rounds + grid - 1) / grid * kKwRoundRows;
    const int g = static_cast<int>((n_rows + rpb - 1) / rpb);
    const int ksel = k;
    size_t smem = static_cast<size_t>(nqb) * sizeof(Cand) + kKwWarps * kKwBufCap * sizeof(Cand) + 4 * static_cast<size_t>(nqb);
    smem = (smem + 15) & ~size_t(15);
    const size_t cval_smem = static_cast<size_t>(kKwWarps) * nu * 8;
    const bool in_smem = smem + cval_smem <= kw->smem_optin;
    c->terms = std::max(c->terms, nu);
    if (!in_smem) ++c->spilled;
    if (in_smem) smem += cval_smem;
    else KW_TRY(c->cval.reserve(static_cast<size_t>(g) * kKwWarps * nu));
    KW_TRY(c->buf.reserve(static_cast<size_t>(g) * nqb * kKwBufCap));
    KW_TRY(c->lists_a.reserve(static_cast<size_t>(nqb) * g * ksel));
    KwParams p{};
    p.off = kw->d_off; p.post = kw->d_post; p.len = kw->d_len; p.ids = kw->d_ids; p.user = kw->d_user; p.org = kw->d_org;
    p.live = kw->d_live; p.allow = d_allow; p.n_rows = n_rows;
    p.idf = reinterpret_cast<const double*>(c->tab.p); p.n_uniq = nu;
    p.hkey = reinterpret_cast<const int32_t*>(c->tab.p + b.b_hk); p.hval = reinterpret_cast<const int32_t*>(c->tab.p + b.b_hv);
    p.hmask = b.hcap - 1;
    p.q_off = reinterpret_cast<const int32_t*>(c->tab.p + b.b_qo); p.slot_u = reinterpret_cast<const int32_t*>(c->tab.p + b.b_sl);
    p.q_user = q.user ? reinterpret_cast<const int32_t*>(c->tab.p + b.b_qu) : nullptr;
    p.q_org = q.user ? reinterpret_cast<const int32_t*>(c->tab.p + b.b_qg) : nullptr;
    p.nq = nqb; p.ksel = ksel; p.avgdl = avgdl;
    p.cval_global = in_smem ? nullptr : c->cval.p;
    p.buf = c->buf.p; p.lists = c->lists_a.p; p.rows_per_block = rpb;
    kw_score_kernel<<<g, kKwThreads, smem, s>>>(p, in_smem ? 1 : 0);
    KW_TRY(cudaGetLastError());
    c->launches += 1;
    // fold the per-block lists until one sorted list per query remains
    int n_lists = g;
    Cand* cur = c->lists_a.p;
    bool in_a = true;
    const int group = std::max(1, kKwFoldCap / ksel);
    for (;;) {
      const int n_groups = (n_lists + group - 1) / group;
      const int gl = std::min(group, n_lists);
      int sort_n = 1;
      while (sort_n < gl * ksel) sort_n <<= 1;
      const size_t fsmem = static_cast<size_t>(sort_n) * sizeof(Cand);
      if (n_groups == 1) {
        kw_fold_kernel<<<dim3(1, nqb), 256, fsmem, s>>>(cur, n_lists, ksel, group, sort_n, nullptr, o_s, o_i, k);
        KW_TRY(cudaGetLastError());
        c->launches += 1;
        break;
      }
      DevBuf<Cand>& dst = in_a ? c->lists_b : c->lists_a;
      KW_TRY(dst.reserve(static_cast<size_t>(nqb) * n_groups * ksel));
      kw_fold_kernel<<<dim3(n_groups, nqb), 256, fsmem, s>>>(cur, n_lists, ksel, group, sort_n, dst.p, nullptr, nullptr, k);
      KW_TRY(cudaGetLastError());
      c->launches += 1;
      cur = dst.p; n_lists = n_groups; in_a = !in_a;
    }
  }
  KW_TRY(cudaEventRecord(c->ev1, s));
  return AUR_OK;
}

// Publish the last_* statistics of a search whose part on c's stream has completed.
int kw_publish(aur_kw* kw, KwCtx* c) {
  float ms = 0.f;
  KW_TRY(cudaEventElapsedTime(&ms, c->ev0, c->ev1));
  std::lock_guard<std::mutex> lk(kw->mu_pool);
  kw->last_launches = c->launches; kw->last_ms = ms;
  kw->last_terms = c->terms; kw->last_spilled = c->spilled;
  return AUR_OK;
}

// Wait for one store's part, copy its [nq][k] lists to the host and publish its last_* statistics.
int kw_collect(aur_kw* kw, KwCtx* c, const KwQuery& q, double* scores_out, int64_t* ids_out) {
  KW_TRY(cudaSetDevice(kw->device));
  cudaStream_t s = c->stream;
  const size_t nout = static_cast<size_t>(q.nq) * q.k;
  KW_TRY(cudaMemcpyAsync(scores_out, c->out_s.p, nout * 8, cudaMemcpyDeviceToHost, s));
  KW_TRY(cudaMemcpyAsync(ids_out, c->out_ids.p, nout * 8, cudaMemcpyDeviceToHost, s));
  KW_TRY(cudaStreamSynchronize(s));
  return kw_publish(kw, c);
}

// Each store's snapshot and the launch tables of a search over stores[0 .. n) taken as one corpus: the batch's distinct
// terms, idf and avgdl from the summed statistics.  Caller holds every store's shared lock.
struct KwPlan {
  std::vector<KwSnap> snaps;
  std::vector<KwBlock> blocks;
  int64_t N = 0;
  double avgdl = 1.0;
};
void kw_prepare(aur_kw* const* stores, int n, const KwQuery& q, KwPlan* pl) {
  std::vector<int32_t> uniq(q.terms, q.terms + q.off[q.nq]);
  std::sort(uniq.begin(), uniq.end());
  uniq.erase(std::unique(uniq.begin(), uniq.end()), uniq.end());
  pl->snaps.assign(static_cast<size_t>(n), KwSnap());
  std::vector<int64_t> udf(uniq.size(), 0);
  int64_t N = 0, total_len = 0;
  for (int s = 0; s < n; ++s) {
    kw_snapshot(stores[s], uniq, &pl->snaps[static_cast<size_t>(s)]);
    const KwSnap& sn = pl->snaps[static_cast<size_t>(s)];
    N += sn.N; total_len += sn.total_len;
    for (size_t i = 0; i < uniq.size(); ++i) udf[i] += sn.udf[i];
  }
  pl->N = N;
  pl->avgdl = total_len ? static_cast<double>(total_len) / static_cast<double>(N) : 1.0;
  kw_plan(q, uniq, udf, N, &pl->blocks);
}

// Search stores[0 .. n) (distinct, arguments checked) as one corpus and hand the enqueued parts to
// after(ctxs, snaps): ctxs[s] = store s's context, whose stream computes its top-k lists into out_s / out_ids, scored
// with the idf and avgdl of the union of the snapshots snaps.  Every store's shared lock is held, and every context
// stays out of its pool, until after() has returned and the context's stream is idle (also on an error).
template <typename After>
int kw_run(aur_kw* const* stores, int n, const KwQuery& q, After&& after) {
  // shared locks for the whole search, in one order (by address) so that searches over overlapping store sets cannot
  // deadlock behind a waiting writer
  std::vector<aur_kw*> order(stores, stores + n);
  std::sort(order.begin(), order.end(), std::less<aur_kw*>());
  std::vector<std::shared_lock<std::shared_mutex>> locks;
  locks.reserve(static_cast<size_t>(n));
  for (aur_kw* kw : order) locks.emplace_back(kw->rw);
  KwPlan pl;
  kw_prepare(stores, n, q, &pl);
  // every store's work enqueued before any is waited on; the contexts go back to their pools only once their streams
  // are idle (also on an error), before the locks are released
  struct Ctxs {
    std::vector<std::pair<aur_kw*, KwCtx*>> v;
    ~Ctxs() {
      for (auto& e : v) { cudaSetDevice(e.first->device); cudaStreamSynchronize(e.second->stream); kw_ctx_release(e.first, e.second); }
    }
  } ctxs;
  std::vector<KwCtx*> cs;
  for (int s = 0; s < n; ++s) {
    aur_kw* kw = stores[s];
    KW_TRY(cudaSetDevice(kw->device));
    KwCtx* c = nullptr;
    int rc = kw_ctx_acquire(kw, &c);
    if (rc != AUR_OK) return rc;
    ctxs.v.emplace_back(kw, c);
    cs.push_back(c);
    const KwSnap& sn = pl.snaps[static_cast<size_t>(s)];
    if ((rc = kw_launch(kw, c, q, pl.blocks, sn.n_rows, pl.N, pl.avgdl)) != AUR_OK) return rc;
  }
  return after(cs, pl.snaps);
}

// kw_run whose parts are copied to the host: store s's top-k lists land in out_s / out_i + s * nq * k.
int kw_search_stores(aur_kw* const* stores, int n, const KwQuery& q, double* out_s, int64_t* out_i, int64_t* snapshot_rows) {
  return kw_run(stores, n, q, [&](const std::vector<KwCtx*>& cs, const std::vector<KwSnap>& snaps) -> int {
    const size_t nout = static_cast<size_t>(q.nq) * q.k;
    for (int s = 0; s < n; ++s) {
      const int rc = kw_collect(stores[s], cs[static_cast<size_t>(s)], q, out_s + s * nout, out_i + s * nout);
      if (rc != AUR_OK) return rc;
    }
    if (snapshot_rows)
      for (int s = 0; s < n; ++s) snapshot_rows[s] = snaps[static_cast<size_t>(s)].n_rows;
    return AUR_OK;
  });
}

}  // namespace

namespace aur {
int kw_legs(aur_kw* const* stores, int n, const int32_t* q_terms, const int64_t* q_offsets, int32_t nq, int32_t k,
            const int32_t* q_user, const int32_t* q_org, const KwLegsThen& then) {
  const KwQuery q{q_terms, q_offsets, nq, k, q_user, q_org, nullptr, 0};
  return kw_run(stores, n, q, [&](const std::vector<KwCtx*>& cs, const std::vector<KwSnap>& snaps) -> int {
    std::vector<KwLeg> legs(static_cast<size_t>(n));
    for (int s = 0; s < n; ++s) {
      const KwCtx* c = cs[static_cast<size_t>(s)];
      legs[static_cast<size_t>(s)] = KwLeg{stores[s]->device, c->stream, c->out_s.p, c->out_ids.p, snaps[static_cast<size_t>(s)].n_rows};
    }
    int rc = then(legs);
    if (rc != AUR_OK) return rc;
    for (int s = 0; s < n; ++s) {
      KW_TRY(cudaSetDevice(stores[s]->device));
      KW_TRY(cudaStreamSynchronize(cs[static_cast<size_t>(s)]->stream));
      if ((rc = kw_publish(stores[s], cs[static_cast<size_t>(s)])) != AUR_OK) return rc;
    }
    return AUR_OK;
  });
}

int kw_check(const int32_t* q_terms, const int64_t* q_offsets, int32_t nq, int32_t k) {
  return kw_check_query(KwQuery{q_terms, q_offsets, nq, k, nullptr, nullptr, nullptr, 0});
}

int kw_device(const aur_kw* kw) { return kw->device; }
}  // namespace aur

extern "C" {

int aur_kw_open(int32_t device, int64_t doc_capacity, int64_t postings_capacity, aur_kw** out) {
  if (!out) return report_error(AUR_ERR_INVALID, "null argument");
  *out = nullptr;
  if (doc_capacity <= 0 || doc_capacity > 0x7FFFFFC0ll) return report_error(AUR_ERR_INVALID, "doc_capacity must be in 1 .. 2^31 - 64");
  if (postings_capacity < 0) return report_error(AUR_ERR_INVALID, "postings_capacity < 0");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess) { cudaGetLastError(); ndev = 0; }
  if (ndev == 0) return report_error(AUR_ERR_NO_DEVICE, "no CUDA device: aurora_b200 has no CPU fallback");
  if (device < 0 || device >= ndev) return report_error(AUR_ERR_INVALID, "device %d out of range", device);
  KW_TRY(cudaSetDevice(device));
  cudaDeviceProp prop;
  KW_TRY(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9) return report_error(AUR_ERR_UNSUPPORTED, "sm_%d%d device: this library is built for sm_90a only", prop.major, prop.minor);
  std::unique_ptr<aur_kw> kw(new aur_kw());
  kw->device = device; kw->capacity = doc_capacity;
  kw->sm_count = prop.multiProcessorCount; kw->smem_optin = prop.sharedMemPerBlockOptin;
  auto bail = [&](cudaError_t e) {
    aur_kw_close(kw.release());
    return report_error(e == cudaErrorMemoryAllocation ? AUR_ERR_NOMEM : AUR_ERR_CUDA, "aur_kw_open: %s", cudaGetErrorString(e));
  };
  cudaError_t e = cudaStreamCreateWithFlags(&kw->stream, cudaStreamNonBlocking);
  const size_t cap = static_cast<size_t>(doc_capacity);
  if (e == cudaSuccess) e = cudaMalloc(&kw->d_off, (cap + 1) * 8);
  if (e == cudaSuccess) e = cudaMalloc(&kw->d_len, cap * 4);
  if (e == cudaSuccess) e = cudaMalloc(&kw->d_ids, cap * 8);
  if (e == cudaSuccess) e = cudaMalloc(&kw->d_user, cap * 4);
  if (e == cudaSuccess) e = cudaMalloc(&kw->d_org, cap * 4);
  if (e == cudaSuccess) e = cudaMalloc(&kw->d_live, cap);
  kw->post_cap = postings_capacity ? postings_capacity : (int64_t(1) << 20);
  if (e == cudaSuccess) e = cudaMalloc(&kw->d_post, static_cast<size_t>(kw->post_cap) * 8);
  if (e == cudaSuccess) e = cudaMemset(kw->d_off, 0, 8);
  // once, at the device's limit: the attribute belongs to the kernel, not to a search, and searches run concurrently
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(kw_score_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kw->smem_optin));
  if (e != cudaSuccess) return bail(e);
  *out = kw.release();
  return AUR_OK;
}

int aur_kw_close(aur_kw* kw) {
  if (!kw) return AUR_OK;
  cudaSetDevice(kw->device);
  if (kw->stream) cudaStreamSynchronize(kw->stream);   // this store's work only: other users of the GPU are not waited on
  for (auto& c : kw->ctxs) cudaStreamSynchronize(c->stream);
  cudaFree(kw->d_off); cudaFree(kw->d_len); cudaFree(kw->d_ids); cudaFree(kw->d_user); cudaFree(kw->d_org);
  cudaFree(kw->d_live); cudaFree(kw->d_post);
  for (auto& c : kw->ctxs) c->release();
  if (kw->stream) cudaStreamDestroy(kw->stream);
  delete kw;
  return AUR_OK;
}

int aur_kw_add(aur_kw* kw, const int64_t* ids, const int32_t* user_codes, const int32_t* org_codes, const int32_t* term_ids,
               const int32_t* tfs, const int64_t* offsets, int64_t n) {
  if (!kw) return report_error(AUR_ERR_INVALID, "null store");
  if (n < 0) return report_error(AUR_ERR_INVALID, "n < 0");
  if (n == 0) return AUR_OK;
  if (!ids || !offsets) return report_error(AUR_ERR_INVALID, "ids and offsets are required");
  if (offsets[0] != 0) return report_error(AUR_ERR_INVALID, "offsets[0] must be 0");
  for (int64_t i = 0; i < n; ++i) {   // offsets first: they bound every read of term_ids / tfs below
    if (ids[i] < 0) return report_error(AUR_ERR_INVALID, "ids must be >= 0");
    if (offsets[i + 1] < offsets[i]) return report_error(AUR_ERR_INVALID, "offsets must be non-decreasing");
  }
  const int64_t total = offsets[n];
  if (total > 0 && (!term_ids || !tfs)) return report_error(AUR_ERR_INVALID, "term_ids and tfs are required");
  int32_t max_term = -1;
  for (int64_t i = 0; i < n; ++i) {
    int64_t dl = 0;
    for (int64_t j = offsets[i]; j < offsets[i + 1]; ++j) {
      if (term_ids[j] < 0 || term_ids[j] >= kKwMaxTerm) return report_error(AUR_ERR_INVALID, "term ids must be in 0 .. 2^28 - 1");
      if (j > offsets[i] && term_ids[j] <= term_ids[j - 1])
        return report_error(AUR_ERR_INVALID, "a document's term ids must be strictly increasing");
      if (tfs[j] < 1) return report_error(AUR_ERR_INVALID, "tf must be >= 1");
      dl += tfs[j];
      max_term = std::max(max_term, term_ids[j]);
    }
    if (dl > 0x7FFFFFFF) return report_error(AUR_ERR_INVALID, "document longer than 2^31 - 1 tokens");
  }
  std::lock_guard<std::mutex> wk(kw->mu_write);
  const int64_t base = static_cast<int64_t>(kw->h_len.size());
  if (base + n > kw->capacity)
    return report_error(AUR_ERR_NOMEM, "keyword store full: %lld + %lld > capacity %lld (aur_kw_compact reclaims tombstones)",
                        (long long)base, (long long)n, (long long)kw->capacity);
  const int64_t post0 = kw->h_off.back();
  bool replaces = false;
  for (int64_t i = 0; i < n && !replaces; ++i) replaces = kw->id2row.count(ids[i]) != 0;
  const bool exclusive = replaces || post0 + total > kw->post_cap;
  std::shared_lock<std::shared_mutex> rl(kw->rw, std::defer_lock);
  std::unique_lock<std::shared_mutex> xl(kw->rw, std::defer_lock);
  if (exclusive) xl.lock(); else rl.lock();
  KW_TRY(cudaSetDevice(kw->device));
  int rc = grow_postings(kw, post0 + total);
  if (rc != AUR_OK) return rc;
  std::vector<uint2> post(static_cast<size_t>(total));
  for (int64_t j = 0; j < total; ++j) post[static_cast<size_t>(j)] = make_uint2(static_cast<uint32_t>(term_ids[j]), static_cast<uint32_t>(tfs[j]));
  std::vector<int64_t> off(static_cast<size_t>(n));
  std::vector<int32_t> len(static_cast<size_t>(n)), user(static_cast<size_t>(n)), org(static_cast<size_t>(n));
  std::vector<uint8_t> live(static_cast<size_t>(n), 1);
  for (int64_t i = 0; i < n; ++i) {
    off[static_cast<size_t>(i)] = post0 + offsets[i + 1];
    int64_t dl = 0;
    for (int64_t j = offsets[i]; j < offsets[i + 1]; ++j) dl += tfs[j];
    len[static_cast<size_t>(i)] = static_cast<int32_t>(dl);
    user[static_cast<size_t>(i)] = user_codes ? user_codes[i] : 0;
    org[static_cast<size_t>(i)] = org_codes ? org_codes[i] : -1;
  }
  // an id repeated inside the batch: its last occurrence wins (the earlier rows land as tombstones)
  std::unordered_map<int64_t, int64_t> last;
  for (int64_t i = 0; i < n; ++i) last[ids[i]] = i;
  for (int64_t i = 0; i < n; ++i) if (last[ids[i]] != i) live[static_cast<size_t>(i)] = 0;
  cudaStream_t s = kw->stream;
  if (total) KW_TRY(cudaMemcpyAsync(kw->d_post + post0, post.data(), static_cast<size_t>(total) * 8, cudaMemcpyHostToDevice, s));
  KW_TRY(cudaMemcpyAsync(kw->d_off + base + 1, off.data(), static_cast<size_t>(n) * 8, cudaMemcpyHostToDevice, s));
  KW_TRY(cudaMemcpyAsync(kw->d_len + base, len.data(), static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, s));
  KW_TRY(cudaMemcpyAsync(kw->d_ids + base, ids, static_cast<size_t>(n) * 8, cudaMemcpyHostToDevice, s));
  KW_TRY(cudaMemcpyAsync(kw->d_user + base, user.data(), static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, s));
  KW_TRY(cudaMemcpyAsync(kw->d_org + base, org.data(), static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, s));
  KW_TRY(cudaMemcpyAsync(kw->d_live + base, live.data(), static_cast<size_t>(n), cudaMemcpyHostToDevice, s));
  KW_TRY(cudaStreamSynchronize(s));
  for (int64_t i = 0; i < n; ++i) {
    kw->h_off.push_back(off[static_cast<size_t>(i)]);
    kw->h_len.push_back(len[static_cast<size_t>(i)]);
    kw->h_ids.push_back(ids[i]);
    kw->h_user.push_back(user[static_cast<size_t>(i)]);
    kw->h_org.push_back(org[static_cast<size_t>(i)]);
    kw->h_live.push_back(live[static_cast<size_t>(i)]);
  }
  std::lock_guard<std::mutex> st(kw->mu_stat);
  if (static_cast<int64_t>(kw->df.size()) <= max_term) kw->df.resize(static_cast<size_t>(max_term) + 1, 0);
  if (replaces) {   // exclusive: no search is running, so the old rows and their statistics leave together
    std::vector<int64_t> old;
    for (int64_t i = 0; i < n; ++i) {
      if (last[ids[i]] != i) continue;
      auto it = kw->id2row.find(ids[i]);
      if (it != kw->id2row.end()) old.push_back(it->second);
    }
    if ((rc = tombstone_rows(kw, old)) != AUR_OK) return rc;
  }
  for (int64_t i = 0; i < n; ++i) {
    if (!live[static_cast<size_t>(i)]) continue;
    kw->id2row[ids[i]] = base + i;
    for (int64_t j = offsets[i]; j < offsets[i + 1]; ++j) ++kw->df[term_ids[j]];
    ++kw->n_live;
    kw->total_len += len[static_cast<size_t>(i)];
  }
  kw->rows_pub = base + n;
  kw->post_pub = post0 + total;
  return AUR_OK;
}

int aur_kw_remove(aur_kw* kw, const int64_t* ids, int64_t n, int64_t* removed) {
  if (!kw || (n > 0 && !ids) || n < 0) return report_error(AUR_ERR_INVALID, "null argument or n < 0");
  std::lock_guard<std::mutex> wk(kw->mu_write);
  std::unique_lock<std::shared_mutex> xl(kw->rw);
  KW_TRY(cudaSetDevice(kw->device));
  std::lock_guard<std::mutex> st(kw->mu_stat);
  std::vector<int64_t> dead;
  for (int64_t i = 0; i < n; ++i) {
    auto it = kw->id2row.find(ids[i]);
    if (it == kw->id2row.end()) continue;
    dead.push_back(it->second);
    kw->id2row.erase(it);
  }
  const int rc = tombstone_rows(kw, dead);
  if (rc != AUR_OK) return rc;
  if (removed) *removed = static_cast<int64_t>(dead.size());
  return AUR_OK;
}

int aur_kw_compact(aur_kw* kw, int64_t* reclaimed) {
  if (!kw) return report_error(AUR_ERR_INVALID, "null store");
  if (reclaimed) *reclaimed = 0;
  std::lock_guard<std::mutex> wk(kw->mu_write);
  std::unique_lock<std::shared_mutex> xl(kw->rw);
  KW_TRY(cudaSetDevice(kw->device));
  KW_TRY(cudaStreamSynchronize(kw->stream));        // searches are host-synchronous: the exclusive lock already drained them
  const int64_t rows = static_cast<int64_t>(kw->h_len.size());
  std::vector<int32_t> map;
  for (int64_t r = 0; r < rows; ++r) if (kw->h_live[static_cast<size_t>(r)]) map.push_back(static_cast<int32_t>(r));
  const int64_t nl = static_cast<int64_t>(map.size());
  if (nl == rows) return AUR_OK;
  // stable: live rows keep their order; postings go to a fresh array of the same capacity
  std::vector<int64_t> off(static_cast<size_t>(nl) + 1, 0), ids(static_cast<size_t>(nl));
  std::vector<int32_t> len(static_cast<size_t>(nl)), user(static_cast<size_t>(nl)), org(static_cast<size_t>(nl));
  for (int64_t j = 0; j < nl; ++j) {
    const size_t r = static_cast<size_t>(map[static_cast<size_t>(j)]);
    off[static_cast<size_t>(j) + 1] = off[static_cast<size_t>(j)] + (kw->h_off[r + 1] - kw->h_off[r]);
    ids[static_cast<size_t>(j)] = kw->h_ids[r]; len[static_cast<size_t>(j)] = kw->h_len[r];
    user[static_cast<size_t>(j)] = kw->h_user[r]; org[static_cast<size_t>(j)] = kw->h_org[r];
  }
  uint2* np_ = nullptr;
  int32_t* d_map = nullptr;
  int64_t* d_noff = nullptr;
  cudaError_t e = cudaMalloc(&np_, static_cast<size_t>(kw->post_cap) * 8);
  if (e == cudaSuccess) e = cudaMalloc(&d_map, std::max<size_t>(1, map.size()) * 4);
  if (e == cudaSuccess) e = cudaMalloc(&d_noff, off.size() * 8);
  if (e == cudaSuccess && nl) e = cudaMemcpy(d_map, map.data(), map.size() * 4, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(d_noff, off.data(), off.size() * 8, cudaMemcpyHostToDevice);
  if (e == cudaSuccess && nl) {
    const int64_t threads = nl * 32;
    kw_gather_postings<<<static_cast<unsigned>((threads + 255) / 256), 256, 0, kw->stream>>>(kw->d_post, kw->d_off, d_map, d_noff, nl, np_);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(kw->stream);
  cudaFree(d_map);
  if (e != cudaSuccess) { cudaFree(np_); cudaFree(d_noff); return report_error(AUR_ERR_CUDA, "aur_kw_compact: %s", cudaGetErrorString(e)); }
  cudaFree(kw->d_post);
  kw->d_post = np_;
  std::vector<uint8_t> live(static_cast<size_t>(nl), 1);
  e = cudaMemcpy(kw->d_off, off.data(), off.size() * 8, cudaMemcpyHostToDevice);
  cudaFree(d_noff);
  if (e == cudaSuccess && nl) e = cudaMemcpy(kw->d_len, len.data(), static_cast<size_t>(nl) * 4, cudaMemcpyHostToDevice);
  if (e == cudaSuccess && nl) e = cudaMemcpy(kw->d_ids, ids.data(), static_cast<size_t>(nl) * 8, cudaMemcpyHostToDevice);
  if (e == cudaSuccess && nl) e = cudaMemcpy(kw->d_user, user.data(), static_cast<size_t>(nl) * 4, cudaMemcpyHostToDevice);
  if (e == cudaSuccess && nl) e = cudaMemcpy(kw->d_org, org.data(), static_cast<size_t>(nl) * 4, cudaMemcpyHostToDevice);
  if (e == cudaSuccess && nl) e = cudaMemcpy(kw->d_live, live.data(), static_cast<size_t>(nl), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) return report_error(AUR_ERR_CUDA, "aur_kw_compact: %s (the store may be inconsistent: rebuild it)", cudaGetErrorString(e));
  kw->h_off = off; kw->h_len = len; kw->h_ids = ids; kw->h_user = user; kw->h_org = org; kw->h_live = live;
  kw->id2row.clear();
  for (int64_t j = 0; j < nl; ++j) kw->id2row[ids[static_cast<size_t>(j)]] = j;
  std::lock_guard<std::mutex> st(kw->mu_stat);
  kw->rows_pub = nl;
  kw->post_pub = off.back();
  if (reclaimed) *reclaimed = rows - nl;
  return AUR_OK;
}

int aur_kw_get_stats(aur_kw* kw, aur_kw_stats* out) {
  if (!kw || !out) return report_error(AUR_ERR_INVALID, "null argument");
  memset(out, 0, sizeof *out);
  {
    std::lock_guard<std::mutex> st(kw->mu_stat);
    out->docs = kw->rows_pub; out->live = kw->n_live; out->total_len = kw->total_len;
    out->postings_used = kw->post_pub;
  }
  std::lock_guard<std::mutex> lk(kw->mu_pool);
  out->postings_allocated = kw->post_cap;
  out->capacity = kw->capacity;
  out->last_launches = kw->last_launches;
  out->last_ms = kw->last_ms;
  out->last_terms = kw->last_terms;
  out->last_spilled = kw->last_spilled;
  return AUR_OK;
}

int aur_kw_search(aur_kw* kw, const int32_t* q_terms, const int64_t* q_offsets, int32_t nq, int32_t k, const int32_t* q_user,
                  const int32_t* q_org, const int64_t* allow_ids, int64_t n_allow, double* scores_out, int64_t* ids_out,
                  int64_t* snapshot_rows_out) {
  if (!kw || !scores_out || !ids_out) return report_error(AUR_ERR_INVALID, "null argument");
  const KwQuery q{q_terms, q_offsets, nq, k, q_user, q_org, allow_ids, n_allow};
  const int rc = kw_check_query(q);
  if (rc != AUR_OK) return rc;
  return kw_search_stores(&kw, 1, q, scores_out, ids_out, snapshot_rows_out);
}

int aur_kw_search_multi(aur_kw* const* stores, int32_t n_stores, const int32_t* q_terms, const int64_t* q_offsets, int32_t nq,
                        int32_t k, const int32_t* q_user, const int32_t* q_org, const int64_t* allow_ids, int64_t n_allow,
                        double* scores_out, int64_t* ids_out, int64_t* snapshot_rows_out) {
  if (!stores) return report_error(AUR_ERR_INVALID, "null argument");
  if (n_stores < 1 || n_stores > kKwMaxStores) return report_error(AUR_ERR_INVALID, "n_stores must be in 1 .. %d", kKwMaxStores);
  for (int32_t s = 0; s < n_stores; ++s) if (!stores[s]) return report_error(AUR_ERR_INVALID, "store %d is NULL", s);
  {
    std::vector<aur_kw*> sorted(stores, stores + n_stores);
    std::sort(sorted.begin(), sorted.end(), std::less<aur_kw*>());
    if (std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end())
      return report_error(AUR_ERR_INVALID, "a store is listed twice (its statistics would count double)");
  }
  if (!scores_out || !ids_out) return report_error(AUR_ERR_INVALID, "null argument");
  const KwQuery q{q_terms, q_offsets, nq, k, q_user, q_org, allow_ids, n_allow};
  int rc = kw_check_query(q);
  if (rc != AUR_OK) return rc;
  if (n_stores == 1) return kw_search_stores(stores, 1, q, scores_out, ids_out, snapshot_rows_out);
  const size_t nout = static_cast<size_t>(nq) * k;
  std::vector<double> ls(nout * n_stores);
  std::vector<int64_t> li(nout * n_stores);
  if ((rc = kw_search_stores(stores, n_stores, q, ls.data(), li.data(), snapshot_rows_out)) != AUR_OK) return rc;
  // every store's lists are sorted by (fp64 score desc, id asc) with (-inf, -1) padding last: one k-way merge per query
  return aur_merge_topk_host_f64(ls.data(), li.data(), n_stores, nq, k, k, scores_out, ids_out);
}

}  // extern "C"
