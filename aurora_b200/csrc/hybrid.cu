// Hybrid query on the device (aur_hybrid_search / aur_hybrid_search_multi, include/aurora_b200.h):
// collection.query.hybrid (weaviate_client.py:252-259) as one host call, over one vector shard and its keyword store or
// over n shards and n stores (one pair per GPU, engine.MultiIndex + engine.MultiKeywordIndex) taken as one corpus.
// aur_hybrid_search is the n = 1 case of the same path.  The keyword legs (keyword.cu, each on its store's own context
// and stream) and the dense legs (capi.cu, each on a pooled context of its shard's device) are enqueued into device
// buffers before any is waited on.  Events join them on shard 0's device, where the lists of shards 1 .. n-1 are
// gathered by peer copies; one kernel merges every query's per-shard lists into each leg's global top-fetch and fuses
// the two, and one device-to-host copy returns the fused top-k_out.
//
// Merge (DESIGN.md section 11): each leg's global list is the host merge's answer (aur_merge_topk_host on the dense
// legs' fp32 cosines, aur_merge_topk_host_f64 on the keyword legs' fp64 scores): a k-way merge that repeatedly takes
// the best list head by (score desc, id asc, list asc), a list ending at its first id < 0.
// Fusion is bit for bit that of the host definitions in aurora_b200/bm25.py:
//   ranked          (ranked_fusion)         contribution = w / (rank + 60.0), rank 0-based within its leg;
//   relative score  (relative_score_fusion) contribution = w if hi == lo else w * ((s - lo) / (hi - lo)), lo / hi = the
//                                           leg's min / max score (dense: the fp32 cosine widened to fp64);
// fused = 0.0 + dense contribution (if listed) + keyword contribution (if listed), in that order, fp64 operation by
// operation (__dadd_rn / __dmul_rn / __ddiv_rn / __dsub_rn: no FMA contraction), sorted by (fused desc, id asc).  A leg
// whose weight is <= 0 takes no part at all.  Ids are distinct within a leg, as both engines return them.
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>

#include <algorithm>
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

constexpr int kFuseThreads = kMaxK;        // thread t holds entry t of each merged leg (fetch <= kMaxK)
constexpr int kFuseWarps = kFuseThreads / 32;
constexpr int kFuseEntries = 2 * kMaxK;    // the union of the two lists
constexpr int kMaxLists = 64;              // shards / stores of one call (the host merge's limit)
constexpr double kRankConstant = 60.0;     // bm25.RANK_CONSTANT
constexpr size_t kOutBytes = 8 + 8 + 4;    // one fused entry: fp64 score, id, fp32 cosine

struct Ent { double s; int64_t id; float cos; };   // padding: (-inf, INT64_MAX, NaN)

__device__ __forceinline__ bool ent_better(const Ent& a, const Ent& b) { return a.s > b.s || (a.s == b.s && a.id < b.id); }

__device__ __forceinline__ double relative(double w, double s, double lo, double hi) {
  return hi == lo ? w : __dmul_rn(w, __ddiv_rn(__dsub_rn(s, lo), __dsub_rn(hi, lo)));
}

// One leg's n per-shard lists of the batch, each [nq][fetch] sorted best first with id -1 padding at its end.
struct LegLists {
  const int64_t* ids0; const void* sc0;     // list 0, where its leg wrote it
  const int64_t* ids_g; const void* sc_g;   // lists 1 .. n-1: gather buffers [n - 1][nq][fetch]
  int64_t* run_max;                         // scratch [nq][n][fetch] (n > 1)
};

struct FuseParams {
  LegLists dense, kw;                         // scores: fp32 cosines, fp64 BM25 scores
  const double* w;                            // [nq][2]: dense weight, keyword weight
  int n, nq, fetch, k_out, fusion, sort_n;    // sort_n: a power of two >= 2 * fetch
  double* o_s; int64_t* o_i; float* o_c;      // [nq][k_out]
};

template <typename S>
__device__ __forceinline__ const S* list_sc(const FuseParams& p, const LegLists& L, int l, int q) {
  const size_t o = static_cast<size_t>(q) * p.fetch;
  return l == 0 ? static_cast<const S*>(L.sc0) + o : static_cast<const S*>(L.sc_g) + static_cast<size_t>(l - 1) * p.nq * p.fetch + o;
}
__device__ __forceinline__ const int64_t* list_ids(const FuseParams& p, const LegLists& L, int l, int q) {
  const size_t o = static_cast<size_t>(q) * p.fetch;
  return l == 0 ? L.ids0 + o : L.ids_g + static_cast<size_t>(l - 1) * p.nq * p.fetch + o;
}
__device__ __forceinline__ int64_t* list_run_max(const FuseParams& p, const LegLists& L, int l, int q) {
  return L.run_max + (static_cast<size_t>(q) * p.n + l) * p.fetch;
}

// The host merge takes the best list head each step.  A list's scores never rise, but a dense list is sorted by its
// fp64 scores, so equal fp32 cosines need not come with ascending ids.  The head-by-head merge then emits the entries
// in the order of the key (score, m, list), m = the largest id of the entry's tie run in its list up to the entry
// (an entry cannot leave before the ones ahead of it, and they hold it back exactly by that key); within a list that
// key never gets better, so an entry's merged position is its index plus, for every other list, the length of the
// prefix whose keys are better -- one binary search each.
//
// Step 1 (warp per list): the valid length len[l] of every list (up to its first id < 0) and every entry's m, by a
// segmented max-scan over runs of equal scores (compared as numbers, so -0.0 == 0.0).
template <typename S>
__device__ __forceinline__ void leg_runs(const FuseParams& p, const LegLists& L, int q, int* len) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int l = warp; l < p.n; l += kFuseWarps) {
    const S* sc = list_sc<S>(p, L, l, q);
    const int64_t* id = list_ids(p, L, l, q);
    int64_t* m = list_run_max(p, L, l, q);
    int n_valid = p.fetch;
    S prev_s = 0;           // last entry of the previous chunk
    int64_t prev_m = 0;
    for (int c0 = 0; c0 < n_valid; c0 += 32) {
      const int j = c0 + lane;
      const bool in = j < p.fetch;
      const int64_t x = in ? __ldg(id + j) : -1;
      const S s = in ? __ldg(sc + j) : S(0);
      const unsigned bad = __ballot_sync(0xffffffffu, x < 0);
      if (bad) n_valid = min(n_valid, c0 + __ffs(bad) - 1);
      const S up = __shfl_up_sync(0xffffffffu, s, 1);
      bool head = lane == 0 ? (c0 == 0 || !(prev_s == s)) : !(up == s);
      int64_t v = x;
      if (lane == 0 && !head) v = prev_m > v ? prev_m : v;
      for (int d = 1; d < 32; d <<= 1) {
        const int64_t vu = __shfl_up_sync(0xffffffffu, v, d);
        const int hu = __shfl_up_sync(0xffffffffu, head ? 1 : 0, d);
        if (lane >= d) {
          if (!head) v = vu > v ? vu : v;
          head = head || hu;
        }
      }
      if (in) m[j] = v;
      prev_s = __shfl_sync(0xffffffffu, s, 31);
      prev_m = __shfl_sync(0xffffffffu, v, 31);
    }
    if (lane == 0) len[l] = n_valid;
  }
}

// Step 2: every entry's merged position; those below fetch land in out_id / out_s there.  Entry e is (index e / n,
// list e % n), so every thread gets a mix of depths; the search stops once the position reaches fetch.
template <typename S>
__device__ __forceinline__ void leg_place(const FuseParams& p, const LegLists& L, int q, const int* len, int64_t* out_id, S* out_s) {
  const int total = p.n * p.fetch;
  for (int e = threadIdx.x; e < total; e += kFuseThreads) {
    const int i = e / p.n, l = e - i * p.n;
    if (i >= len[l]) continue;
    const S s = __ldg(list_sc<S>(p, L, l, q) + i);
    const int64_t m = list_run_max(p, L, l, q)[i];   // written by this kernel: not through the read-only path
    int pos = i;
    for (int o = 0; o < p.n && pos < p.fetch; ++o) {
      if (o == l) continue;
      const S* so = list_sc<S>(p, L, o, q);
      const int64_t* mo = list_run_max(p, L, o, q);
      int lo = 0, hi = len[o];
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        const S t = __ldg(so + mid);
        const int64_t mm = mo[mid];
        if (t > s || (t == s && (mm < m || (mm == m && o < l)))) lo = mid + 1;
        else hi = mid;
      }
      pos += lo;
    }
    if (pos < p.fetch) { out_id[pos] = __ldg(list_ids(p, L, l, q) + i); out_s[pos] = s; }
  }
}

// One leg's global top-fetch of query q into out_id / out_s (id -1 past its end).  One list: itself.
template <typename S>
__device__ __forceinline__ void leg_merge(const FuseParams& p, const LegLists& L, int q, int* len, int64_t* out_id, S* out_s) {
  const int t = threadIdx.x;
  if (p.n == 1) {
    if (t < p.fetch) {
      out_id[t] = __ldg(list_ids(p, L, 0, q) + t);
      out_s[t] = __ldg(list_sc<S>(p, L, 0, q) + t);
    }
    return;
  }
  if (t < p.fetch) out_id[t] = -1;
  leg_runs<S>(p, L, q, len);
  __syncthreads();
  leg_place<S>(p, L, q, len, out_id, out_s);
}

// One CTA per query: each leg's merged list, the contributions, the union (a keyword entry whose id the dense list
// holds adds onto that entry), a bitonic sort of the union and its best k_out out.
__global__ void __launch_bounds__(kFuseThreads) hybrid_merge_fuse_kernel(FuseParams p) {
  __shared__ Ent e[kFuseEntries];
  __shared__ int64_t dense_id[kFuseThreads];
  __shared__ double red[4][kFuseWarps];
  __shared__ int64_t m_did[kMaxK], m_sid[kMaxK];   // the merged lists
  __shared__ float m_dcos[kMaxK];
  __shared__ double m_ss[kMaxK];
  __shared__ int len[2][kMaxLists];
  const int q = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  if (p.w[2 * q] > 0.0) leg_merge<float>(p, p.dense, q, len[0], m_did, m_dcos);
  if (p.w[2 * q + 1] > 0.0) leg_merge<double>(p, p.kw, q, len[1], m_sid, m_ss);
  __syncthreads();
  const double wd = p.w[2 * q], ws = p.w[2 * q + 1];   // read after the merges: held across them, they spill
  int64_t did = -1, sid = -1;
  float dc = nanf("");
  double ss = -INFINITY;
  if (t < p.fetch) {
    if (wd > 0.0) { did = m_did[t]; dc = m_dcos[t]; }
    if (ws > 0.0) { sid = m_sid[t]; ss = m_ss[t]; }
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
      for (int w = 0; w < kFuseWarps; ++w) v[i] = (i & 1) ? fmax(v[i], red[i][w]) : fmin(v[i], red[i][w]);
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

// Scratch of one shard's part of a hybrid call on one device: the stream its dense leg runs on and that leg's lists.
// The context of shard 0 also hosts the join, the gathered lists of the other shards, the merge + fusion kernel and the
// copy back.  Idle contexts are pooled for the life of the process.
struct HybridCtx {
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t kw_done = nullptr, dense_done = nullptr;
  DevBuf<float> cos;
  DevBuf<int64_t> ids;
  DevBuf<double> w;
  DevBuf<float> g_cos;              // gathered lists of shards 1 .. n-1: dense cosines and ids, keyword scores and ids
  DevBuf<int64_t> g_did, g_kid;
  DevBuf<double> g_ks;
  DevBuf<int64_t> run_max;          // the merge's scratch, both legs
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
  cudaError_t e = cudaSetDevice(device);
  if (e == cudaSuccess) e = cudaDeviceGetStreamPriorityRange(&lo, &hi);
  if (e == cudaSuccess) e = cudaStreamCreateWithPriority(&h->stream, cudaStreamNonBlocking, hi);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->kw_done, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->dense_done, cudaEventDisableTiming);
  if (e != cudaSuccess) {
    if (h->kw_done) cudaEventDestroy(h->kw_done);
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

// The arguments of one call, checked.
struct HybridArgs {
  aur_index* const* shards; int n;
  const void* queries_host; int32_t nq, fetch;
  const int32_t* q_user; const int32_t* q_org;
  std::vector<double> w;   // [nq][2]
  int32_t fusion, k_out;
};

// Inside the keyword legs: every shard's dense leg, the join and gather on shard 0's device, the merge + fusion and the
// copy into hs[0]->host.  hs[s] is on shard s's device; rows[s] receives shard s's snapshot.
int run_on_devices(const HybridArgs& a, const std::vector<HybridCtx*>& hs, const std::vector<KwLeg>& kl, int64_t* rows) {
  const int n = a.n;
  const size_t nl = static_cast<size_t>(a.nq) * a.fetch, no = static_cast<size_t>(a.nq) * a.k_out;
  HybridCtx* h = hs[0];
  cudaStream_t st = h->stream;
  HYB_TRY(cudaSetDevice(h->device));
  HYB_TRY(h->w.reserve(a.w.size()));
  HYB_TRY(h->out.reserve(no * kOutBytes));
  if (h->host_n < no * kOutBytes) {
    if (h->host) cudaFreeHost(h->host);
    h->host = nullptr; h->host_n = 0;
    HYB_TRY(cudaHostAlloc(reinterpret_cast<void**>(&h->host), no * kOutBytes, cudaHostAllocDefault));
    h->host_n = no * kOutBytes;
  }
  if (n > 1) {
    const size_t ng = static_cast<size_t>(n - 1) * nl;
    HYB_TRY(h->g_cos.reserve(ng));
    HYB_TRY(h->g_did.reserve(ng));
    HYB_TRY(h->g_ks.reserve(ng));
    HYB_TRY(h->g_kid.reserve(ng));
    HYB_TRY(h->run_max.reserve(2 * static_cast<size_t>(n) * nl));
  }
  HYB_TRY(cudaMemcpyAsync(h->w.p, a.w.data(), a.w.size() * 8, cudaMemcpyHostToDevice, st));
  // (pageable: staged before the call returns; behind the dense legs it would wait for their kernels)
  for (int s = 0; s < n; ++s) {
    HybridCtx* o = hs[static_cast<size_t>(s)];
    HYB_TRY(cudaSetDevice(o->device));
    HYB_TRY(o->cos.reserve(nl));
    HYB_TRY(o->ids.reserve(nl));
    const int rc = dense_leg(a.shards[s], o->device, o->stream, a.queries_host, a.nq, a.fetch, a.q_user, a.q_org, o->cos.p,
                             o->ids.p, &rows[s]);
    if (rc != AUR_OK) return rc;
    if (s > 0) HYB_TRY(cudaEventRecord(o->dense_done, o->stream));
    HYB_TRY(cudaEventRecord(o->kw_done, kl[static_cast<size_t>(s)].stream));   // the store shares the shard's device
  }
  HYB_TRY(cudaSetDevice(h->device));
  // the join: every keyword leg, every other shard's dense leg; their lists come over by peer copies (also between
  // shards of one device, so that every shard count runs the same code)
  for (int s = 0; s < n; ++s) {
    const HybridCtx* o = hs[static_cast<size_t>(s)];
    const KwLeg& k = kl[static_cast<size_t>(s)];
    HYB_TRY(cudaStreamWaitEvent(st, o->kw_done, 0));
    if (s == 0) continue;
    HYB_TRY(cudaStreamWaitEvent(st, o->dense_done, 0));
    const size_t at = static_cast<size_t>(s - 1) * nl;
    HYB_TRY(cudaMemcpyPeerAsync(h->g_cos.p + at, h->device, o->cos.p, o->device, nl * 4, st));
    HYB_TRY(cudaMemcpyPeerAsync(h->g_did.p + at, h->device, o->ids.p, o->device, nl * 8, st));
    HYB_TRY(cudaMemcpyPeerAsync(h->g_ks.p + at, h->device, k.scores, k.device, nl * 8, st));
    HYB_TRY(cudaMemcpyPeerAsync(h->g_kid.p + at, h->device, k.ids, k.device, nl * 8, st));
  }
  FuseParams p;
  p.dense = LegLists{h->ids.p, h->cos.p, h->g_did.p, h->g_cos.p, h->run_max.p};
  p.kw = LegLists{kl[0].ids, kl[0].scores, h->g_kid.p, h->g_ks.p, n > 1 ? h->run_max.p + static_cast<size_t>(n) * nl : nullptr};
  p.w = h->w.p;
  p.n = n; p.nq = a.nq; p.fetch = a.fetch; p.k_out = a.k_out; p.fusion = a.fusion;
  p.sort_n = 2;
  while (p.sort_n < 2 * a.fetch) p.sort_n <<= 1;
  p.o_s = reinterpret_cast<double*>(h->out.p);
  p.o_i = reinterpret_cast<int64_t*>(h->out.p + no * 8);
  p.o_c = reinterpret_cast<float*>(h->out.p + no * 16);
  hybrid_merge_fuse_kernel<<<static_cast<unsigned>(a.nq), kFuseThreads, 0, st>>>(p);
  HYB_TRY(cudaGetLastError());
  HYB_TRY(cudaMemcpyAsync(h->host, h->out.p, no * kOutBytes, cudaMemcpyDeviceToHost, st));
  HYB_TRY(cudaStreamSynchronize(st));
  return AUR_OK;
}

template <typename T>
bool has_repeat(T* const* v, int n) {
  std::vector<T*> sorted(v, v + n);
  std::sort(sorted.begin(), sorted.end(), std::less<T*>());
  return std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end();
}

// Both entry points: arguments already checked up to the handle lists (non-NULL, distinct, 1 <= n <= kMaxLists).
int hybrid_search(aur_index* const* shards, aur_kw* const* stores, int32_t n, const void* queries_host, int32_t nq,
                  int32_t fetch, const int32_t* q_terms, const int64_t* q_offsets, const int32_t* q_user,
                  const int32_t* q_org, const double* w_dense, const double* w_sparse, int32_t fusion, int32_t k_out,
                  double* scores_out, int64_t* ids_out, float* cosine_out, int64_t* snapshot_rows_out) {
  if (nq <= 0) return report_error(AUR_ERR_INVALID, "nq must be positive");
  if (nq > 65535) return report_error(AUR_ERR_UNSUPPORTED, "nq > 65535: split the batch");
  if (fetch < 1) return report_error(AUR_ERR_INVALID, "fetch must be positive");
  if (fetch > kMaxK) return report_error(AUR_ERR_UNSUPPORTED, "fetch > %d", kMaxK);
  if (k_out < 1 || k_out > 2 * fetch) return report_error(AUR_ERR_INVALID, "k_out must be in 1 .. 2 * fetch (%d)", 2 * fetch);
  if (fusion != AUR_FUSION_RANKED && fusion != AUR_FUSION_RELATIVE_SCORE) return report_error(AUR_ERR_INVALID, "unknown fusion %d", fusion);
  HybridArgs a{shards, n, queries_host, nq, fetch, q_user, q_org, std::vector<double>(2 * static_cast<size_t>(nq)), fusion, k_out};
  for (int32_t i = 0; i < nq; ++i) {
    if (!std::isfinite(w_dense[i]) || !std::isfinite(w_sparse[i])) return report_error(AUR_ERR_INVALID, "weights must be finite (query %d)", i);
    a.w[2 * static_cast<size_t>(i)] = w_dense[i];
    a.w[2 * static_cast<size_t>(i) + 1] = w_sparse[i];
  }
  int rc = kw_check(q_terms, q_offsets, nq, fetch);
  if (rc != AUR_OK) return rc;
  for (int s = 0; s < n; ++s) {
    if (!index_is_bf16(shards[s])) return report_error(AUR_ERR_UNSUPPORTED, "hybrid search needs bf16 shards (shard %d)", s);
    if (index_device(shards[s]) != kw_device(stores[s]))
      return report_error(AUR_ERR_INVALID, "keyword store %d is on device %d, its shard on device %d", s, kw_device(stores[s]),
                          index_device(shards[s]));
  }
  std::vector<HybridCtx*> hs;
  std::vector<int64_t> rows(2 * static_cast<size_t>(n), 0);
  rc = kw_legs(stores, n, q_terms, q_offsets, nq, fetch, q_user, q_org, [&](const std::vector<KwLeg>& kl) {
    int r = AUR_OK;
    for (int s = 0; s < n && r == AUR_OK; ++s) {
      HybridCtx* h = nullptr;
      if ((r = hyb_acquire(kl[static_cast<size_t>(s)].device, &h)) == AUR_OK) hs.push_back(h);
      rows[static_cast<size_t>(n + s)] = kl[static_cast<size_t>(s)].snapshot_rows;
    }
    if (r == AUR_OK) r = run_on_devices(a, hs, kl, rows.data());
    for (HybridCtx* h : hs) { cudaSetDevice(h->device); cudaStreamSynchronize(h->stream); }   // nothing stays in flight
    return r;
  });
  if (rc == AUR_OK) {
    const size_t no = static_cast<size_t>(nq) * k_out;
    memcpy(scores_out, hs[0]->host, no * 8);
    memcpy(ids_out, hs[0]->host + no * 8, no * 8);
    memcpy(cosine_out, hs[0]->host + no * 16, no * 4);
    if (snapshot_rows_out) memcpy(snapshot_rows_out, rows.data(), rows.size() * 8);
  }
  for (HybridCtx* h : hs) hyb_release(h);
  return rc;
}

}  // namespace

extern "C" {

int aur_hybrid_search(aur_index* ix, aur_kw* kw, const void* queries_host, int32_t nq, int32_t fetch, const int32_t* q_terms,
                      const int64_t* q_offsets, const int32_t* q_user, const int32_t* q_org, const double* w_dense,
                      const double* w_sparse, int32_t fusion, int32_t k_out, double* scores_out, int64_t* ids_out,
                      float* cosine_out, int64_t* snapshot_rows_out) {
  if (!ix || !kw || !queries_host || !q_offsets || !w_dense || !w_sparse || !scores_out || !ids_out || !cosine_out)
    return report_error(AUR_ERR_INVALID, "null argument");
  return hybrid_search(&ix, &kw, 1, queries_host, nq, fetch, q_terms, q_offsets, q_user, q_org, w_dense, w_sparse, fusion,
                       k_out, scores_out, ids_out, cosine_out, snapshot_rows_out);
}

int aur_hybrid_search_multi(aur_index* const* shards, aur_kw* const* stores, int32_t n, const void* queries_host, int32_t nq,
                            int32_t fetch, const int32_t* q_terms, const int64_t* q_offsets, const int32_t* q_user,
                            const int32_t* q_org, const double* w_dense, const double* w_sparse, int32_t fusion,
                            int32_t k_out, double* scores_out, int64_t* ids_out, float* cosine_out,
                            int64_t* snapshot_rows_out) {
  if (!shards || !stores || !queries_host || !q_offsets || !w_dense || !w_sparse || !scores_out || !ids_out || !cosine_out)
    return report_error(AUR_ERR_INVALID, "null argument");
  if (n < 1 || n > kMaxLists) return report_error(AUR_ERR_INVALID, "n must be in 1 .. %d", kMaxLists);
  for (int32_t s = 0; s < n; ++s)
    if (!shards[s] || !stores[s]) return report_error(AUR_ERR_INVALID, "shard or store %d is NULL", s);
  if (has_repeat(shards, n)) return report_error(AUR_ERR_INVALID, "a shard is listed twice");
  if (has_repeat(stores, n)) return report_error(AUR_ERR_INVALID, "a keyword store is listed twice (its statistics would count double)");
  return hybrid_search(shards, stores, n, queries_host, nq, fetch, q_terms, q_offsets, q_user, q_org, w_dense, w_sparse, fusion,
                       k_out, scores_out, ids_out, cosine_out, snapshot_rows_out);
}

}  // extern "C"
