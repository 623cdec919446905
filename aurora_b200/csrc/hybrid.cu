// Hybrid query on the device (aur_hybrid_search, include/aurora_b200.h): collection.query.hybrid
// (weaviate_client.py:252-259) as one host call.  The keyword leg (keyword.cu, on the store's own context and stream) and
// the dense leg (capi.cu, on this call's stream) are enqueued into device buffers before either is waited on, an event
// joins them, one kernel fuses every query's two lists and one device-to-host copy returns the fused top-k_out.
//
// Fusion (DESIGN.md section 11) is bit for bit that of the host definitions in aurora_b200/bm25.py:
//   ranked          (ranked_fusion)         contribution = w / (rank + 60.0), rank 0-based within its leg;
//   relative score  (relative_score_fusion) contribution = w if hi == lo else w * ((s - lo) / (hi - lo)), lo / hi = the
//                                           leg's min / max score (dense: the fp32 cosine widened to fp64);
// fused = 0.0 + dense contribution (if listed) + keyword contribution (if listed), in that order, fp64 operation by
// operation (__dadd_rn / __dmul_rn / __ddiv_rn / __dsub_rn: no FMA contraction), sorted by (fused desc, id asc).  A leg
// whose weight is <= 0 takes no part at all.  Ids are distinct within a leg, as both engines return them.
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>

#include <cmath>
#include <memory>
#include <mutex>
#include <vector>

#include "../../include/aurora_b200.h"
#include "internal.h"

using namespace aur;

namespace {

#define HYB_TRY(expr)                                                                                            \
  do {                                                                                                           \
    cudaError_t e_ = (expr);                                                                                     \
    if (e_ != cudaSuccess)                                                                                       \
      return report_error(e_ == cudaErrorMemoryAllocation ? AUR_ERR_NOMEM : AUR_ERR_CUDA, "%s: %s (%s:%d)", #expr, \
                          cudaGetErrorString(e_), __FILE__, __LINE__);                                           \
  } while (0)

constexpr int kFuseThreads = kMaxK;        // thread t holds entry t of each leg (fetch <= kMaxK)
constexpr int kFuseEntries = 2 * kMaxK;    // the union of the two lists
constexpr double kRankConstant = 60.0;     // bm25.RANK_CONSTANT
constexpr size_t kOutBytes = 8 + 8 + 4;    // one fused entry: fp64 score, id, fp32 cosine

struct Ent { double s; int64_t id; float cos; };   // padding: (-inf, INT64_MAX, NaN)

__device__ __forceinline__ bool ent_better(const Ent& a, const Ent& b) { return a.s > b.s || (a.s == b.s && a.id < b.id); }

__device__ __forceinline__ double relative(double w, double s, double lo, double hi) {
  return hi == lo ? w : __dmul_rn(w, __ddiv_rn(__dsub_rn(s, lo), __dsub_rn(hi, lo)));
}

struct FuseParams {
  const int64_t* d_ids; const float* d_cos;   // dense leg [nq][fetch]: ids (-1 padding), fp32 cosines
  const int64_t* s_ids; const double* s_sc;   // keyword leg [nq][fetch]: ids (-1 padding), fp64 BM25 scores
  const double* w;                            // [nq][2]: dense weight, keyword weight
  int fetch, k_out, fusion, sort_n;           // sort_n: a power of two >= 2 * fetch
  double* o_s; int64_t* o_i; float* o_c;      // [nq][k_out]
};

// One CTA per query: the two lists, their contributions, the union (a keyword entry whose id the dense list holds adds
// onto that entry), a bitonic sort of the union and its best k_out out.
__global__ void __launch_bounds__(kFuseThreads) hybrid_fuse_kernel(FuseParams p) {
  __shared__ Ent e[kFuseEntries];
  __shared__ int64_t dense_id[kFuseThreads];
  __shared__ double red[4][kFuseThreads / 32];
  const int q = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const double wd = p.w[2 * q], ws = p.w[2 * q + 1];
  int64_t did = -1, sid = -1;
  float dc = nanf("");
  double ss = -INFINITY;
  if (t < p.fetch) {
    const size_t o = static_cast<size_t>(q) * p.fetch + t;
    if (wd > 0.0) { did = __ldg(p.d_ids + o); dc = __ldg(p.d_cos + o); }
    if (ws > 0.0) { sid = __ldg(p.s_ids + o); ss = __ldg(p.s_sc + o); }
  }
  const bool dv = did >= 0, sv = sid >= 0;
  const double ds = static_cast<double>(dc);
  double cd, cs;
  if (p.fusion == AUR_FUSION_RANKED) {
    const double den = static_cast<double>(t) + kRankConstant;
    cd = __ddiv_rn(wd, den);
    cs = __ddiv_rn(ws, den);
  } else {
    // each leg's min / max over its listed entries (fmin / fmax are exact)
    double v[4] = {dv ? ds : INFINITY, dv ? ds : -INFINITY, sv ? ss : INFINITY, sv ? ss : -INFINITY};
    for (int o = 16; o > 0; o >>= 1)
      for (int i = 0; i < 4; ++i) {
        const double x = __shfl_xor_sync(0xffffffffu, v[i], o);
        v[i] = (i & 1) ? fmax(v[i], x) : fmin(v[i], x);
      }
    if (lane == 0)
      for (int i = 0; i < 4; ++i) red[i][warp] = v[i];
    __syncthreads();
    for (int i = 0; i < 4; ++i)
      for (int w = 0; w < kFuseThreads / 32; ++w) v[i] = (i & 1) ? fmax(v[i], red[i][w]) : fmin(v[i], red[i][w]);
    cd = relative(wd, ds, v[0], v[1]);
    cs = relative(ws, ss, v[2], v[3]);
  }
  const Ent pad{-INFINITY, INT64_MAX, nanf("")};
  for (int i = t; i < p.sort_n; i += kFuseThreads) e[i] = pad;
  dense_id[t] = did;
  __syncthreads();
  // dense entry t in slot t, keyword entry t in slot fetch + t; every fused score starts from 0.0
  if (dv) e[t] = Ent{__dadd_rn(0.0, cd), did, dc};
  if (sv) e[p.fetch + t] = Ent{__dadd_rn(0.0, cs), sid, nanf("")};
  __syncthreads();
  if (sv)
    for (int j = 0; j < p.fetch; ++j)
      if (dense_id[j] == sid) {   // the only match: ids are distinct within the dense list
        e[j].s = __dadd_rn(e[j].s, cs);
        e[p.fetch + t] = pad;
        break;
      }
  __syncthreads();
  // bitonic sort, best first
  for (int size = 2; size <= p.sort_n; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = t; i < p.sort_n / 2; i += kFuseThreads) {
        const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
        const bool desc = (lo & size) == 0;
        const Ent x = e[lo], y = e[hi];
        if (desc ? ent_better(y, x) : ent_better(x, y)) { e[lo] = y; e[hi] = x; }
      }
      __syncthreads();
    }
  for (int i = t; i < p.k_out; i += kFuseThreads) {
    const Ent x = e[i];
    const bool none = x.id == INT64_MAX;
    const size_t o = static_cast<size_t>(q) * p.k_out + i;
    p.o_s[o] = none ? -INFINITY : x.s;
    p.o_i[o] = none ? -1 : x.id;
    p.o_c[o] = none ? nanf("") : x.cos;
  }
}

// Scratch of one hybrid call on one device: the stream the dense leg, the join and the fusion run on, and the buffers
// between them.  Idle contexts are pooled for the life of the process.
struct HybridCtx {
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t kw_done = nullptr;
  DevBuf<float> cos;
  DevBuf<int64_t> ids;
  DevBuf<double> w;
  DevBuf<unsigned char> out;        // fused [nq][k_out] scores | ids | cosines, copied back in one piece
  unsigned char* host = nullptr;    // page-locked landing area of that copy
  size_t host_n = 0;
};

std::mutex g_pool_mu;
std::vector<HybridCtx*> g_idle;

int hyb_acquire(int device, HybridCtx** out) {
  {
    std::lock_guard<std::mutex> lk(g_pool_mu);
    for (size_t i = 0; i < g_idle.size(); ++i)
      if (g_idle[i]->device == device) {
        *out = g_idle[i];
        g_idle.erase(g_idle.begin() + static_cast<std::ptrdiff_t>(i));
        return AUR_OK;
      }
  }
  std::unique_ptr<HybridCtx> h(new HybridCtx());
  h->device = device;
  int lo = 0, hi = 0;   // hi = numerically lowest = highest priority, as the search contexts' streams
  cudaError_t e = cudaDeviceGetStreamPriorityRange(&lo, &hi);
  if (e == cudaSuccess) e = cudaStreamCreateWithPriority(&h->stream, cudaStreamNonBlocking, hi);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->kw_done, cudaEventDisableTiming);
  if (e != cudaSuccess) {
    if (h->stream) cudaStreamDestroy(h->stream);
    return report_error(AUR_ERR_CUDA, "hybrid search context: %s", cudaGetErrorString(e));
  }
  *out = h.release();
  return AUR_OK;
}

void hyb_release(HybridCtx* h) {
  std::lock_guard<std::mutex> lk(g_pool_mu);
  g_idle.push_back(h);
}

// Inside the keyword leg: the dense leg, the join, the fusion and the copy into h->host.
int fuse_on_device(HybridCtx* h, aur_index* ix, const void* queries_host, int32_t nq, int32_t fetch, const int32_t* q_user,
                   const int32_t* q_org, const std::vector<double>& w, int32_t fusion, int32_t k_out, cudaStream_t ks,
                   const double* kw_s, const int64_t* kw_i, int64_t* dense_rows) {
  const size_t nl = static_cast<size_t>(nq) * fetch, no = static_cast<size_t>(nq) * k_out;
  cudaStream_t s = h->stream;
  HYB_TRY(h->cos.reserve(nl));
  HYB_TRY(h->ids.reserve(nl));
  HYB_TRY(h->w.reserve(w.size()));
  HYB_TRY(h->out.reserve(no * kOutBytes));
  if (h->host_n < no * kOutBytes) {
    if (h->host) cudaFreeHost(h->host);
    h->host = nullptr; h->host_n = 0;
    HYB_TRY(cudaHostAlloc(reinterpret_cast<void**>(&h->host), no * kOutBytes, cudaHostAllocDefault));
    h->host_n = no * kOutBytes;
  }
  HYB_TRY(cudaMemcpyAsync(h->w.p, w.data(), w.size() * 8, cudaMemcpyHostToDevice, s));   // pageable: staged before return
  int rc = dense_leg(ix, h->device, s, queries_host, nq, fetch, q_user, q_org, h->cos.p, h->ids.p, dense_rows);
  if (rc != AUR_OK) return rc;
  HYB_TRY(cudaEventRecord(h->kw_done, ks));
  HYB_TRY(cudaStreamWaitEvent(s, h->kw_done, 0));
  FuseParams p;
  p.d_ids = h->ids.p; p.d_cos = h->cos.p; p.s_ids = kw_i; p.s_sc = kw_s; p.w = h->w.p;
  p.fetch = fetch; p.k_out = k_out; p.fusion = fusion;
  p.sort_n = 2;
  while (p.sort_n < 2 * fetch) p.sort_n <<= 1;
  p.o_s = reinterpret_cast<double*>(h->out.p);
  p.o_i = reinterpret_cast<int64_t*>(h->out.p + no * 8);
  p.o_c = reinterpret_cast<float*>(h->out.p + no * 16);
  hybrid_fuse_kernel<<<static_cast<unsigned>(nq), kFuseThreads, 0, s>>>(p);
  HYB_TRY(cudaGetLastError());
  HYB_TRY(cudaMemcpyAsync(h->host, h->out.p, no * kOutBytes, cudaMemcpyDeviceToHost, s));
  HYB_TRY(cudaStreamSynchronize(s));
  return AUR_OK;
}

}  // namespace

extern "C" {

int aur_hybrid_search(aur_index* ix, aur_kw* kw, const void* queries_host, int32_t nq, int32_t fetch, const int32_t* q_terms,
                      const int64_t* q_offsets, const int32_t* q_user, const int32_t* q_org, const double* w_dense,
                      const double* w_sparse, int32_t fusion, int32_t k_out, double* scores_out, int64_t* ids_out,
                      float* cosine_out, int64_t* snapshot_rows_out) {
  if (!ix || !kw || !queries_host || !q_offsets || !w_dense || !w_sparse || !scores_out || !ids_out || !cosine_out)
    return report_error(AUR_ERR_INVALID, "null argument");
  if (nq <= 0) return report_error(AUR_ERR_INVALID, "nq must be positive");
  if (nq > 65535) return report_error(AUR_ERR_UNSUPPORTED, "nq > 65535: split the batch");
  if (fetch < 1) return report_error(AUR_ERR_INVALID, "fetch must be positive");
  if (fetch > kMaxK) return report_error(AUR_ERR_UNSUPPORTED, "fetch > %d", kMaxK);
  if (k_out < 1 || k_out > 2 * fetch) return report_error(AUR_ERR_INVALID, "k_out must be in 1 .. 2 * fetch (%d)", 2 * fetch);
  if (fusion != AUR_FUSION_RANKED && fusion != AUR_FUSION_RELATIVE_SCORE) return report_error(AUR_ERR_INVALID, "unknown fusion %d", fusion);
  std::vector<double> w(2 * static_cast<size_t>(nq));
  for (int32_t i = 0; i < nq; ++i) {
    if (!std::isfinite(w_dense[i]) || !std::isfinite(w_sparse[i])) return report_error(AUR_ERR_INVALID, "weights must be finite (query %d)", i);
    w[2 * static_cast<size_t>(i)] = w_dense[i];
    w[2 * static_cast<size_t>(i) + 1] = w_sparse[i];
  }
  HybridCtx* h = nullptr;
  int64_t rows[2] = {0, 0};
  const int rc = kw_leg(kw, q_terms, q_offsets, nq, fetch, q_user, q_org,
                        [&](int device, cudaStream_t ks, const double* kw_s, const int64_t* kw_i, int64_t kw_rows) {
                          rows[1] = kw_rows;
                          int r = hyb_acquire(device, &h);
                          if (r != AUR_OK) return r;
                          r = fuse_on_device(h, ix, queries_host, nq, fetch, q_user, q_org, w, fusion, k_out, ks, kw_s, kw_i, &rows[0]);
                          cudaStreamSynchronize(h->stream);   // nothing of this call stays in flight, also on an error
                          return r;
                        });
  if (rc == AUR_OK) {
    const size_t no = static_cast<size_t>(nq) * k_out;
    memcpy(scores_out, h->host, no * 8);
    memcpy(ids_out, h->host + no * 8, no * 8);
    memcpy(cosine_out, h->host + no * 16, no * 4);
    if (snapshot_rows_out) { snapshot_rows_out[0] = rows[0]; snapshot_rows_out[1] = rows[1]; }
  }
  if (h) hyb_release(h);
  return rc;
}

}  // extern "C"
