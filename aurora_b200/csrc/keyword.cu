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
// A term-major index of the store's first R rows (DESIGN.md section 10, "Term-major index") lets a launch score those
// rows from its own terms' posting lists instead, into per-query accumulators, when the path rule estimates it cheaper;
// the rows behind R are always scanned forward, and both parts' lists are folded together.
// aur_kw_search_multi runs the same search over several stores (one per GPU) as one corpus: N, df and total_len are
// summed over the stores' snapshots, every store scores its own prefix with the resulting idf / avgdl, and the per-store
// lists are merged on the host (DESIGN.md section 10, "Sharded store").  The hybrid query (hybrid.cu) runs the same
// steps through kw_legs and merges the per-store lists on the device instead; its filtered form evaluates filter programs
// over the store's tenant codes and attribute columns (aur_kw_set_attrs, filter.cu) and scores only the matching rows.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>

#include <cmath>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <chrono>
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
// term-major index (DESIGN.md section 10, "Term-major index")
constexpr int64_t kKwMaxRows = 0x7FFFFFC0ll;              // aur_kw_open's capacity limit: every row id fits the index's u32
static_assert(kKwMaxRows <= 0xFFFFFFFFll, "indexed rows are u32");
constexpr int64_t kIxTailFrac = 8;                         // the writer rebuilds once the tail holds > 1/8 of the indexed postings
constexpr int kIxMaxTermPos = 64;                          // term positions (one launch each) a query group takes through the index
constexpr int64_t kIxAccBytes = int64_t(256) << 20;        // fp64 accumulators of one query group: more queries are split
constexpr int kIxSelBlocksPerSm = 4;                       // selection grid over the indexed rows
// the path rule's cost model, in ns of H100 time: forward scan per posting of [0, R); index per list posting, per
// accumulator entry scanned, per launch
constexpr double kFwdNsPerPosting = 0.02, kIxNsPerPosting = 0.05, kIxNsPerAcc = 0.005, kIxNsPerLaunch = 3000.0;

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
  // filtered launches (kw_score_kernel<true>): fmask [n_passes][fmask_stride] program match bits of every row (bit p of
  // word ps = program 32 ps + p), prog_used [n_passes] the programs this launch's queries name, q_prog [nq] each one's
  const uint32_t* fmask; const uint32_t* prog_used; const int32_t* q_prog;
  int64_t fmask_stride; int n_passes;
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

// Selection state of one block in shared memory (kw_score_kernel, kw_ix_select_kernel): thr [nq] the block's ksel-th
// best so far, sort_area [warps][kKwBufCap], cnt [nq] entries in each query's candidate buffer.
struct KwSel { Cand* thr; Cand* sort_area; int* cnt; };

// Query q's admission of a row with score s > 0 (row: index into the row-indexed arrays of p; ru / ro / rid: the row's
// tenant codes and id): the query's tenant scope, its filter program (kFilt), then the block's threshold; an admitted
// row joins the query's candidate buffer.
template <bool kFilt>
__device__ __forceinline__ void kw_offer(const KwParams& p, const KwSel& sl, Cand* gbuf, int q, int64_t row, int32_t ru,
                                         int32_t ro, int64_t rid, double s) {
  if (p.q_user) {
    const int32_t qu = __ldg(p.q_user + q), qo = p.q_org ? __ldg(p.q_org + q) : -1;
    if (!(ru == qu || (qo >= 0 && ro == qo))) return;
  }
  if constexpr (kFilt) {
    const int32_t pg = __ldg(p.q_prog + q);
    if (!((__ldg(p.fmask + (pg >> 5) * p.fmask_stride + row) >> (pg & 31)) & 1u)) return;
  }
  const Cand c{s, rid};
  if (!better(c, sl.thr[q])) return;
  const int pos = atomicAdd(sl.cnt + q, 1);
  gbuf[static_cast<size_t>(q) * kKwBufCap + pos] = c;
}

// End of a round (at most kKwRoundRows appends per query since the last): buffers that could overflow next round are
// cut to their best ksel, which raises the threshold.  Between two __syncthreads.
__device__ __forceinline__ void kw_round_flush(const KwParams& p, const KwSel& sl, Cand* gbuf, int warp, int lane) {
  for (int q = warp; q < p.nq; q += kKwWarps) {
    const int c = sl.cnt[q];
    if (c > kKwBufCap - kKwRoundRows) {
      Cand t = sl.thr[q];
      const int keep = warp_flush(p, sl.sort_area + warp * kKwBufCap, gbuf + static_cast<size_t>(q) * kKwBufCap, c, lane, &t);
      if (lane == 0) { sl.cnt[q] = keep; sl.thr[q] = t; }
    }
  }
}

// The block's sorted best ksel per query: query q's list is list `list` of n_lists at p.lists + (q * n_lists + list) * ksel.
__device__ __forceinline__ void kw_block_lists(const KwParams& p, const KwSel& sl, Cand* gbuf, int warp, int lane,
                                               unsigned n_lists, unsigned list) {
  for (int q = warp; q < p.nq; q += kKwWarps) {
    Cand* area = sl.sort_area + warp * kKwBufCap;
    const int keep = warp_flush(p, area, gbuf + static_cast<size_t>(q) * kKwBufCap, sl.cnt[q], lane, nullptr);
    Cand* out = p.lists + (static_cast<size_t>(q) * n_lists + list) * p.ksel;
    for (int i = lane; i < p.ksel; i += 32) out[i] = i < keep ? area[i] : sentinel();
  }
}

// kFilt: query q admits a row only when the row matches program q_prog[q]; a row that matches no program of the launch is
// skipped before its postings are read.
template <bool kFilt>
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
  const KwSel sl{thr, sort_area, cnt};
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
      if constexpr (kFilt) {
        uint32_t any = 0u;
        for (int ps = 0; ps < p.n_passes; ++ps) any |= __ldg(p.fmask + ps * p.fmask_stride + row) & __ldg(p.prog_used + ps);
        if (!any) continue;
      }
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
        kw_offer<kFilt>(p, sl, gbuf, q, row, ru, ro, rid, s);
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
    kw_round_flush(p, sl, gbuf, warp, lane);
    __syncthreads();
  }
  kw_block_lists(p, sl, gbuf, warp, lane, gridDim.x, blockIdx.x);
}

// ------------------------------------------------------------------------------------------- term-major index
// The store's first R rows, term by term: term t's postings are tpost[toff[t] .. toff[t + 1]) as (row, tf), in no
// particular order within a term.  Built by a counting sort of the forward postings of rows [0, R): kw_ix_count,
// kw_ix_scan, kw_ix_scatter.

// cnt[t] += postings of term t in rows [0, R); one warp per row.
__global__ void kw_ix_count(const int64_t* off, const uint2* post, int64_t R, unsigned* cnt) {
  const int64_t w = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (w >= R) return;
  for (int64_t i = off[w] + (threadIdx.x & 31); i < off[w + 1]; i += 32) atomicAdd(cnt + post[i].x, 1u);
}

// toff[0 .. T] = exclusive scan of cnt[0 .. T) (toff[T] = every posting), cur = toff[0 .. T); one block, each thread a
// contiguous chunk of terms.
__global__ void __launch_bounds__(1024) kw_ix_scan(const unsigned* cnt, int64_t T, int64_t* toff, unsigned long long* cur) {
  __shared__ int64_t part[1024];
  const int t = threadIdx.x;
  const int64_t chunk = (T + 1023) / 1024;
  const int64_t a = t * chunk, b = a + chunk < T ? a + chunk : T;
  int64_t s = 0;
  for (int64_t i = a; i < b; ++i) s += cnt[i];
  part[t] = s;
  __syncthreads();
  for (int d = 1; d < 1024; d <<= 1) {   // inclusive scan of the chunk sums
    const int64_t v = t >= d ? part[t - d] : 0;
    __syncthreads();
    part[t] += v;
    __syncthreads();
  }
  int64_t run = part[t] - s;
  for (int64_t i = a; i < b; ++i) { toff[i] = run; cur[i] = static_cast<unsigned long long>(run); run += cnt[i]; }
  if (t == 1023) toff[T] = part[1023];
}

// tpost[cur[t]++] = (row, tf) for every posting of rows [0, R); one warp per row.
__global__ void kw_ix_scatter(const int64_t* off, const uint2* post, int64_t R, unsigned long long* cur, uint2* tpost) {
  const int64_t w = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (w >= R) return;
  for (int64_t i = off[w] + (threadIdx.x & 31); i < off[w + 1]; i += 32) {
    const uint2 pt = post[i];
    tpost[atomicAdd(cur + pt.x, 1ull)] = make_uint2(static_cast<uint32_t>(w), pt.y);
  }
}

// One term position of a query group scored from the index: query q (blockIdx.y) of the group adds the contribution of
// its j-th term u (summation order) to acc[q * R + row] for every (row, tf) of u's list.  A list holds a row once and a
// query has one j-th term, so no two threads of a launch touch one entry; launches j = 0, 1, ... run in stream order,
// so acc[q][row] is summed in the query's term order, as kw_score_kernel sums it.
struct KwIxTerm {
  const uint2* tpost; const int64_t* toff; int64_t n_terms;   // the index (terms 0 .. n_terms - 1)
  const int32_t* len; const int32_t* ukey; const double* idf;   // ukey [n_uniq]: unique index -> term id
  const int32_t* q_off; const int32_t* slot_u;                  // the group's first query at q_off[0]
  double* acc; int64_t R; double avgdl; int j;
};

__global__ void __launch_bounds__(256) kw_ix_term_kernel(KwIxTerm t) {
  const int q = blockIdx.y;
  const int g = __ldg(t.q_off + q) + t.j;
  if (g >= __ldg(t.q_off + q + 1)) return;
  const int u = __ldg(t.slot_u + g);
  const int32_t term = __ldg(t.ukey + u);
  if (term >= t.n_terms) return;   // first seen after the build: no indexed row has it
  const int64_t hi = __ldg(t.toff + term + 1);
  const double idf = __ldg(t.idf + u);
  double* acc = t.acc + static_cast<size_t>(q) * t.R;
  for (int64_t i = __ldg(t.toff + term) + static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < hi;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const uint2 pt = __ldg(t.tpost + i);
    acc[pt.x] = __dadd_rn(acc[pt.x], contribution(idf, pt.y, __ldg(t.len + pt.x), t.avgdl));
  }
}

// Selection over the indexed rows [0, p.n_rows): query q's score of row r is acc[q * R + r] (0.0: none of its terms);
// every entry is read once and reset to 0.0 for the next search.  Rows are admitted by kw_score_kernel's tests and
// selected into the same per-block lists: query q's list of block b at p.lists + (q * n_lists + b) * ksel.  A round
// is kKwRoundRows rows, one per lane; warp w takes queries w, w + 8, ...
template <bool kFilt>
__global__ void __launch_bounds__(kKwThreads) kw_ix_select_kernel(KwParams p, double* acc, int64_t R, int n_lists) {
  extern __shared__ __align__(16) unsigned char smem[];
  Cand* thr = reinterpret_cast<Cand*>(smem);   // kw_score_kernel's layout, without the contribution table
  Cand* sort_area = thr + p.nq;
  int* cnt = reinterpret_cast<int*>(sort_area + kKwWarps * kKwBufCap);
  const KwSel sl{thr, sort_area, cnt};
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int q = threadIdx.x; q < p.nq; q += blockDim.x) { thr[q] = sentinel(); cnt[q] = 0; }
  __syncthreads();
  Cand* gbuf = p.buf + static_cast<size_t>(blockIdx.x) * p.nq * kKwBufCap;
  const int64_t r_begin = static_cast<int64_t>(blockIdx.x) * p.rows_per_block;
  int64_t r_end = r_begin + p.rows_per_block;
  if (r_end > p.n_rows) r_end = p.n_rows;
  for (int64_t r0 = r_begin; r0 < r_end; r0 += kKwRoundRows) {
    const int64_t row = r0 + lane;
    if (row < r_end) {
      int state = -1;   // the row's live / allow test, once a query scores it: 1 admitted, 0 not
      int32_t ru = 0, ro = 0;
      int64_t rid = 0;
      for (int q = warp; q < p.nq; q += kKwWarps) {
        double* a = acc + static_cast<size_t>(q) * R + row;
        const double s = *a;
        if (s == 0.0) continue;
        *a = 0.0;
        if (state < 0) {
          state = __ldg(p.live + row) && !(p.allow && !__ldg(p.allow + row));
          if (state) { ru = __ldg(p.user + row); ro = __ldg(p.org + row); rid = __ldg(p.ids + row); }
        }
        if (state && s > 0.0) kw_offer<kFilt>(p, sl, gbuf, q, row, ru, ro, rid, s);
      }
    }
    __syncthreads();
    kw_round_flush(p, sl, gbuf, warp, lane);
    __syncthreads();
  }
  kw_block_lists(p, sl, gbuf, warp, lane, static_cast<unsigned>(n_lists), blockIdx.x);
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
  Stream stream;
  Event ev0, ev1;
  DevBuf<unsigned char> tab;     // launch term table
  DevBuf<Cand> buf, lists_a, lists_b;
  DevBuf<double> cval, out_s;
  DevBuf<int64_t> out_ids;
  DevBuf<uint8_t> allow;
  DevBuf<int32_t> allow_rows;
  DevBuf<int32_t> fstage;        // filtered search: the programs' tokens, offsets and bitmaps (one upload)
  DevBuf<uint32_t> fmask;        // filtered search: [passes][rows] program match bits
  DevBuf<double> acc;            // index path: [group][R] per-query scores, all 0.0 between searches
  bool acc_clean = true;         // false while a search's index part is in flight (an error leaves it dirty)
  int launches = 0, terms = 0, spilled = 0;   // of the last search: kernels, most distinct terms in one launch,
                                              // launches whose contribution table spilled to global memory
  int path = 0;                  // of the last search: AUR_KW_PATH_* bits
  int64_t postings = 0;          // of the last search: postings it read

  int init(int /* device: current */) {
    const cudaError_t e = [&]() -> cudaError_t {
      AUR_CU_RET(stream.create(cudaStreamNonBlocking));
      AUR_CU_RET(ev0.create());
      return ev1.create();
    }();
    if (e != cudaSuccess) return report_error(AUR_ERR_CUDA, "search context: %s", cudaGetErrorString(e));
    return AUR_OK;
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
  std::mutex mu_last;        // the last search's statistics (last_*)
  int device = 0, sm_count = 0;
  size_t smem_optin = 0;
  std::atomic<int64_t> capacity{0};   // document rows; grows under mu_write and the exclusive lock (aur_kw_reserve)
  Stream stream;
  // device
  DevBuf<int64_t> d_off; DevBuf<int32_t> d_len; DevBuf<int64_t> d_ids;
  DevBuf<int32_t> d_user, d_org; DevBuf<uint8_t> d_live;
  DevBuf<uint2> d_post;      // d_post.n: the postings capacity
  AttrColumns attrs;         // program columns 2.., capacity rows each (aur_kw_set_attrs, writers hold mu_write)
  // host mirrors (the writer's bookkeeping; searches read only the published statistics)
  std::vector<int64_t> h_off{0};
  std::vector<int32_t> h_len, h_user, h_org;
  std::vector<int64_t> h_ids;
  std::vector<uint8_t> h_live;
  std::unordered_map<int64_t, int64_t> id2row;
  // published under mu_stat
  int64_t rows_pub = 0, post_pub = 0, n_live = 0, total_len = 0;
  std::vector<int64_t> df;
  // term-major index of rows [0, ix_rows) (ix_post postings), published under mu_stat and replaced only under the
  // exclusive lock: d_toff [ix_terms + 1], d_tpost [ix_post]; h_toff mirrors d_toff
  DevBuf<int64_t> d_toff; DevBuf<uint2> d_tpost;
  int64_t ix_rows = 0, ix_post = 0, ix_terms = 0, ix_builds = 0;
  std::vector<int64_t> h_toff;
  float ix_build_ms = 0.f;
  std::atomic<int> kw_path{0};   // aur_kw_set_option "kw_path": 0 auto, 1 forward, 2 index
  CtxPool<KwCtx> ctxs;           // search contexts
  int last_launches = 0, last_terms = 0, last_spilled = 0, last_path = 0;
  int64_t last_postings = 0;
  float last_ms = 0.f;
};

namespace {

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
  const cudaError_t e = [&]() -> cudaError_t {
    AUR_CU_RET(d_map.reserve(m));
    AUR_CU_RET(d_noff.reserve(m + 1));
    AUR_CU_RET(d_terms.reserve(std::max<size_t>(terms.size(), 1)));
    AUR_CU_RET(cudaMemcpyAsync(d_map.p, map.data(), m * 4, cudaMemcpyHostToDevice, s));
    AUR_CU_RET(cudaMemcpyAsync(d_noff.p, noff.data(), (m + 1) * 8, cudaMemcpyHostToDevice, s));
    kw_gather_postings<<<static_cast<unsigned>((static_cast<int64_t>(m) * 32 + 255) / 256), 256, 0, s>>>(
        kw->d_post.p, kw->d_off.p, d_map.p, d_noff.p, static_cast<int64_t>(m), d_terms.p);
    kw_scatter_flag<<<static_cast<unsigned>((m + 255) / 256), 256, 0, s>>>(d_map.p, static_cast<int64_t>(m), kw->d_live.p, 0);
    AUR_CU_RET(cudaGetLastError());
    if (!terms.empty()) AUR_CU_RET(cudaMemcpyAsync(terms.data(), d_terms.p, terms.size() * 8, cudaMemcpyDeviceToHost, s));
    return cudaStreamSynchronize(s);
  }();
  if (e != cudaSuccess) return report_error(AUR_ERR_CUDA, "tombstone: %s", cudaGetErrorString(e));
  for (const uint2& p : terms) --kw->df[p.x];
  for (int64_t r : rows) {
    kw->h_live[static_cast<size_t>(r)] = 0;
    --kw->n_live;
    kw->total_len -= kw->h_len[static_cast<size_t>(r)];
  }
  return AUR_OK;
}

// Drop the term-major index (rows are about to move).  Caller holds the exclusive lock.
void drop_index(aur_kw* kw) {
  DevBuf<int64_t> toff; DevBuf<uint2> tpost;   // the index, freed on return outside mu_stat
  std::lock_guard<std::mutex> st(kw->mu_stat);
  std::swap(toff, kw->d_toff); std::swap(tpost, kw->d_tpost);
  kw->ix_rows = kw->ix_post = kw->ix_terms = 0;
  kw->h_toff.clear();
}

// Build the term-major index of every appended row into fresh buffers on the store's stream and publish it.  The
// caller holds mu_write and no rw lock: the forward postings of the rows being indexed only change under mu_write, so
// searches go on while the index is built, and publishing waits for the searches in flight (exclusive lock).
int build_index(aur_kw* kw) {
  const auto t0 = std::chrono::steady_clock::now();
  const int64_t R = static_cast<int64_t>(kw->h_len.size()), P = kw->h_off.back();
  const int64_t T = static_cast<int64_t>(kw->df.size());   // every term id seen so far (writers resize df)
  AUR_TRY(cudaSetDevice(kw->device));
  cudaStream_t s = kw->stream;
  DevBuf<int64_t> toff; DevBuf<uint2> tpost;
  std::vector<int64_t> h_toff(static_cast<size_t>(T) + 1);
  const unsigned row_blocks = static_cast<unsigned>((R * 32 + 255) / 256);
  const cudaError_t e = [&]() -> cudaError_t {
    DevBuf<unsigned> cnt; DevBuf<unsigned long long> cur;
    AUR_CU_RET(toff.reserve(static_cast<size_t>(T) + 1));
    AUR_CU_RET(tpost.reserve(static_cast<size_t>(std::max<int64_t>(P, 1))));
    AUR_CU_RET(cnt.reserve(static_cast<size_t>(std::max<int64_t>(T, 1))));
    AUR_CU_RET(cur.reserve(static_cast<size_t>(std::max<int64_t>(T, 1))));
    AUR_CU_RET(cudaMemsetAsync(cnt.p, 0, static_cast<size_t>(T) * 4, s));
    if (R) kw_ix_count<<<row_blocks, 256, 0, s>>>(kw->d_off.p, kw->d_post.p, R, cnt.p);
    kw_ix_scan<<<1, 1024, 0, s>>>(cnt.p, T, toff.p, cur.p);
    if (R) kw_ix_scatter<<<row_blocks, 256, 0, s>>>(kw->d_off.p, kw->d_post.p, R, cur.p, tpost.p);
    AUR_CU_RET(cudaGetLastError());
    AUR_CU_RET(cudaMemcpyAsync(h_toff.data(), toff.p, h_toff.size() * 8, cudaMemcpyDeviceToHost, s));
    return cudaStreamSynchronize(s);
  }();
  if (e != cudaSuccess) {
    return report_error(e == cudaErrorMemoryAllocation ? AUR_ERR_NOMEM : AUR_ERR_CUDA, "keyword index build: %s",
                        cudaGetErrorString(e));
  }
  const float ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
  {
    std::unique_lock<std::shared_mutex> xl(kw->rw);
    std::lock_guard<std::mutex> st(kw->mu_stat);
    std::swap(toff, kw->d_toff); std::swap(tpost, kw->d_tpost);
    kw->h_toff.swap(h_toff);
    kw->ix_rows = R; kw->ix_post = P; kw->ix_terms = T;
    ++kw->ix_builds;
    kw->ix_build_ms = ms;
  }
  return AUR_OK;   // toff / tpost now hold the previous index, freed here: no search holds it any more
}

// The writer's rule: rebuild once the unindexed tail holds more than 1 / kIxTailFrac of the indexed postings (any
// postings at all when nothing is indexed).  Caller holds mu_write.
bool index_due(const aur_kw* kw) {
  const int64_t tail = kw->h_off.back() - kw->ix_post;
  return tail > 0 && tail * kIxTailFrac > kw->ix_post;
}

// ---------------------------------------------------------------------------------------------------------- search
// One search, over one store or several stores taken as one corpus, in the steps both entry points share: every store's
// shared lock (in address order), a snapshot of each prefix and its statistics, the query blocks' launch tables built
// once from the summed statistics, every store's passes enqueued on its own device and stream, then each store's top-k
// collected.

struct KwQuery {   // the arguments of one search (aur_kw_search; fp: the hybrid query's programs, nullable)
  const int32_t* terms; const int64_t* off; int32_t nq, k;
  const int32_t* user; const int32_t* org; const int64_t* allow; int64_t n_allow;
  const FiltProgs* fp;
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

struct KwSnap {
  int64_t n_rows = 0, N = 0, total_len = 0, post = 0;
  std::vector<int64_t> udf;
  // the term-major index of rows [0, ix_rows) (ix_post postings, terms 0 .. ix_terms - 1); ulen: list length of each
  // distinct term of the batch
  const int64_t* toff = nullptr; const uint2* tpost = nullptr;
  int64_t ix_rows = 0, ix_post = 0, ix_terms = 0;
  std::vector<int64_t> ulen;
};

// The published prefix, its statistics, df of the batch's distinct terms uniq and the index, in one read.
void kw_snapshot(aur_kw* kw, const std::vector<int32_t>& uniq, KwSnap* s) {
  std::lock_guard<std::mutex> st(kw->mu_stat);
  s->n_rows = kw->rows_pub; s->N = kw->n_live; s->total_len = kw->total_len; s->post = kw->post_pub;
  s->udf.assign(uniq.size(), 0);
  for (size_t i = 0; i < uniq.size(); ++i)
    s->udf[i] = (uniq[i] >= 0 && uniq[i] < static_cast<int32_t>(kw->df.size())) ? kw->df[static_cast<size_t>(uniq[i])] : 0;
  s->toff = kw->d_toff.p; s->tpost = kw->d_tpost.p;
  s->ix_rows = kw->ix_rows; s->ix_post = kw->ix_post; s->ix_terms = kw->ix_terms;
  s->ulen.assign(uniq.size(), 0);
  for (size_t i = 0; i < uniq.size(); ++i)
    if (uniq[i] >= 0 && uniq[i] < kw->ix_terms)
      s->ulen[i] = kw->h_toff[static_cast<size_t>(uniq[i]) + 1] - kw->h_toff[static_cast<size_t>(uniq[i])];
}

// One launch's query side, the same on every store: idf | hkey | hval | qoff | slot | q_user | q_org [| q_prog |
// programs used] in one upload.
struct KwBlock {
  int q0 = 0, nqb = 0, nu = 0, hcap = 0;   // nu = 0: no query of the block has a live term
  size_t b_hk = 0, b_hv = 0, b_qo = 0, b_sl = 0, b_qu = 0, b_qg = 0, b_qp = 0, b_pu = 0, b_uk = 0;
  std::vector<unsigned char> tab;
  std::vector<int32_t> qoff, slot, ug;     // host copies of qoff / slot; ug: unique index -> index into the batch's uniq
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
    b.b_qp = b.b_qg + 4 * static_cast<size_t>(nqb); b.b_pu = b.b_qp + 4 * static_cast<size_t>(nqb);
    const int n_passes = q.fp ? filter_passes(q.fp->n_programs) : 0;
    b.b_uk = q.fp ? b.b_pu + 4 * static_cast<size_t>(n_passes) : b.b_qp;
    b.tab.assign(b.b_uk + 4 * static_cast<size_t>(nu), 0);
    unsigned char* tab = b.tab.data();
    memcpy(tab + b.b_uk, ukeys.data(), 4 * static_cast<size_t>(nu));
    b.ug.resize(static_cast<size_t>(nu));
    for (int u = 0; u < nu; ++u)
      b.ug[static_cast<size_t>(u)] = static_cast<int32_t>(std::lower_bound(uniq.begin(), uniq.end(), ukeys[static_cast<size_t>(u)]) - uniq.begin());
    b.qoff = qoff; b.slot = slot;
    memcpy(tab, uidf.data(), 8 * static_cast<size_t>(nu));
    memcpy(tab + b.b_hk, hkey.data(), 4 * static_cast<size_t>(hcap));
    memcpy(tab + b.b_hv, hval.data(), 4 * static_cast<size_t>(hcap));
    memcpy(tab + b.b_qo, qoff.data(), 4 * qoff.size());
    if (!slot.empty()) memcpy(tab + b.b_sl, slot.data(), 4 * slot.size());
    if (q.user) memcpy(tab + b.b_qu, q.user + q0, 4 * static_cast<size_t>(nqb));
    std::vector<int32_t> qorg(static_cast<size_t>(nqb), -1);
    if (q.org) std::copy(q.org + q0, q.org + q0 + nqb, qorg.begin());
    memcpy(tab + b.b_qg, qorg.data(), 4 * static_cast<size_t>(nqb));
    if (q.fp) {
      std::vector<uint32_t> used(static_cast<size_t>(n_passes), 0u);
      for (int i = 0; i < nqb; ++i) {
        const int32_t pg = q.fp->q_program[q0 + i];
        used[static_cast<size_t>(pg / kFiltMaxPrograms)] |= 1u << (pg % kFiltMaxPrograms);
      }
      memcpy(tab + b.b_qp, q.fp->q_program + q0, 4 * static_cast<size_t>(nqb));
      memcpy(tab + b.b_pu, used.data(), 4 * used.size());
    }
    blocks->push_back(std::move(b));
  }
}

// Blocks that own contiguous ranges of whole rounds of n rows, at most max_blocks of them; *rpb = rows per block.
int kw_grid(int64_t n, int64_t max_blocks, int64_t* rpb) {
  const int64_t rounds = (n + kKwRoundRows - 1) / kKwRoundRows;
  const int64_t grid = std::max<int64_t>(1, std::min<int64_t>(max_blocks, rounds));
  *rpb = (rounds + grid - 1) / grid * kKwRoundRows;
  return static_cast<int>((n + *rpb - 1) / *rpb);
}

// How one launch (query block b) scores the indexed rows [0, rows) of the snapshot: rows = 0 leaves every row to the
// forward scan.  The index serves a block whose queries have at most kIxMaxTermPos terms, in groups of `group` queries
// whose accumulators fit kIxAccBytes, and (kw_path auto) when its estimated time -- a launch per term position and
// group, the lists it reads (`postings`, dead rows included), the accumulator scan -- is below the forward scan's of the
// same rows.
struct KwIxPlan { int64_t rows = 0, postings = 0; int group = 0; };
KwIxPlan kw_ix_plan(const aur_kw* kw, const KwSnap& sn, const KwBlock& b) {
  KwIxPlan x;
  const int mode = kw->kw_path.load(std::memory_order_relaxed);
  const int64_t R = sn.ix_rows;
  if (mode == 1 || R == 0) return x;
  int J = 0;
  for (int i = 0; i < b.nqb; ++i) J = std::max(J, b.qoff[static_cast<size_t>(i) + 1] - b.qoff[static_cast<size_t>(i)]);
  const int64_t gmax = kIxAccBytes / (8 * R);
  if (J > kIxMaxTermPos || gmax < 1) return x;
  const int group = static_cast<int>(std::min<int64_t>(b.nqb, gmax));
  int64_t L = 0;
  for (int32_t u : b.slot) L += sn.ulen[static_cast<size_t>(b.ug[static_cast<size_t>(u)])];
  if (mode == 0) {
    const int n_groups = (b.nqb + group - 1) / group;
    const double t_ix = n_groups * (J + 1) * kIxNsPerLaunch + static_cast<double>(L) * kIxNsPerPosting +
                        static_cast<double>(b.nqb) * static_cast<double>(R) * kIxNsPerAcc;
    if (!(t_ix < static_cast<double>(sn.ix_post) * kFwdNsPerPosting)) return x;
  }
  x.rows = R; x.postings = L; x.group = group;
  return x;
}

// Enqueue one store's part of the search on c's stream: allow-list flags, then per block the table upload, the scoring
// of the store's prefix sn.n_rows (index and / or forward scan) and the folds into c's [nq][k] output.  Nothing waits.
int kw_launch(aur_kw* kw, KwCtx* c, const KwQuery& q, const std::vector<KwBlock>& blocks, const KwSnap& sn, int64_t N,
              double avgdl) {
  AUR_TRY(cudaSetDevice(kw->device));
  cudaStream_t s = c->stream;
  const int k = q.k;
  const int64_t n_rows = sn.n_rows;
  c->launches = 0; c->terms = 0; c->spilled = 0; c->path = 0; c->postings = 0;
  AUR_TRY(cudaEventRecord(c->ev0, s));
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
    AUR_TRY(c->allow.reserve(static_cast<size_t>(std::max<int64_t>(n_rows, 1))));
    AUR_TRY(c->allow_rows.reserve(std::max<size_t>(rows.size(), 1)));
    AUR_TRY(cudaMemsetAsync(c->allow.p, 0, static_cast<size_t>(std::max<int64_t>(n_rows, 1)), s));
    if (!rows.empty()) {
      AUR_TRY(cudaMemcpyAsync(c->allow_rows.p, rows.data(), rows.size() * 4, cudaMemcpyHostToDevice, s));
      kw_scatter_flag<<<static_cast<unsigned>((rows.size() + 255) / 256), 256, 0, s>>>(c->allow_rows.p, static_cast<int64_t>(rows.size()), c->allow.p, 1);
      AUR_TRY(cudaGetLastError());
      c->launches += 1;
    }
    d_allow = c->allow.p;
  }
  // programs: every row's match bits over the snapshot, 32 programs a pass; the scoring kernel reads them in place
  const uint32_t* d_fmask = nullptr;
  int n_passes = 0;
  const bool scores = n_rows > 0 && N > 0 && std::any_of(blocks.begin(), blocks.end(), [](const KwBlock& b) { return b.nu > 0; });
  if (q.fp && scores) {
    n_passes = filter_passes(q.fp->n_programs);
    AUR_TRY(c->fmask.reserve(static_cast<size_t>(n_passes) * static_cast<size_t>(n_rows)));
    FiltParams p;
    AUR_TRY(filter_upload(*q.fp, kw->d_user.p, kw->d_org.p, kw->attrs, c->fstage, s, &p));
    p.live = kw->d_live.p; p.n_rows = n_rows;
    for (int ps = 0; ps < n_passes; ++ps) {
      AUR_TRY(launch_filter_mask(filter_pass(p, ps), c->fmask.p + static_cast<size_t>(ps) * n_rows, s));
      c->launches += 1;
    }
    d_fmask = c->fmask.p;
  }
  const size_t nout = static_cast<size_t>(q.nq) * k;
  AUR_TRY(c->out_s.reserve(nout));
  AUR_TRY(c->out_ids.reserve(nout));
  for (const KwBlock& b : blocks) {
    const int nqb = b.nqb, nu = b.nu;
    double* o_s = c->out_s.p + static_cast<size_t>(b.q0) * k;
    int64_t* o_i = c->out_ids.p + static_cast<size_t>(b.q0) * k;
    if (nu == 0 || n_rows == 0 || N == 0) {   // nothing can match: padding only
      std::vector<double> ps(static_cast<size_t>(nqb) * k, -INFINITY);
      std::vector<int64_t> pi(static_cast<size_t>(nqb) * k, -1);
      AUR_TRY(cudaMemcpyAsync(o_s, ps.data(), ps.size() * 8, cudaMemcpyHostToDevice, s));
      AUR_TRY(cudaMemcpyAsync(o_i, pi.data(), pi.size() * 8, cudaMemcpyHostToDevice, s));
      continue;
    }
    AUR_TRY(c->tab.reserve(b.tab.size()));
    AUR_TRY(cudaMemcpyAsync(c->tab.p, b.tab.data(), b.tab.size(), cudaMemcpyHostToDevice, s));   // pageable: staged before return
    const int ksel = k;
    c->terms = std::max(c->terms, nu);
    // rows [0, R) from the term-major index when the path rule picks it, rows [R, n_rows) by the forward scan; the
    // index part's per-block lists come first, the forward part's after them
    const KwIxPlan ix = kw_ix_plan(kw, sn, b);
    const int64_t R = ix.rows, tail = n_rows - R;
    int64_t rpb_i = 0, rpb_t = 0;
    const int gi = R > 0 ? kw_grid(R, kIxSelBlocksPerSm * static_cast<int64_t>(kw->sm_count), &rpb_i) : 0;
    const int gt = tail > 0 ? kw_grid(tail, 2 * static_cast<int64_t>(kw->sm_count), &rpb_t) : 0;
    int n_lists = gi + gt;   // folded below
    AUR_TRY(c->buf.reserve(static_cast<size_t>(std::max(gi, gt)) * nqb * kKwBufCap));
    AUR_TRY(c->lists_a.reserve(static_cast<size_t>(nqb) * n_lists * ksel));
    KwParams p{};
    p.off = kw->d_off.p; p.post = kw->d_post.p; p.len = kw->d_len.p; p.ids = kw->d_ids.p; p.user = kw->d_user.p; p.org = kw->d_org.p;
    p.live = kw->d_live.p; p.allow = d_allow; p.n_rows = n_rows;
    p.idf = reinterpret_cast<const double*>(c->tab.p); p.n_uniq = nu;
    p.hkey = reinterpret_cast<const int32_t*>(c->tab.p + b.b_hk); p.hval = reinterpret_cast<const int32_t*>(c->tab.p + b.b_hv);
    p.hmask = b.hcap - 1;
    p.q_off = reinterpret_cast<const int32_t*>(c->tab.p + b.b_qo); p.slot_u = reinterpret_cast<const int32_t*>(c->tab.p + b.b_sl);
    p.q_user = q.user ? reinterpret_cast<const int32_t*>(c->tab.p + b.b_qu) : nullptr;
    p.q_org = q.user ? reinterpret_cast<const int32_t*>(c->tab.p + b.b_qg) : nullptr;
    p.nq = nqb; p.ksel = ksel; p.avgdl = avgdl;
    p.buf = c->buf.p; p.lists = c->lists_a.p;
    if (d_fmask) {
      p.fmask = d_fmask; p.fmask_stride = n_rows; p.n_passes = n_passes;
      p.q_prog = reinterpret_cast<const int32_t*>(c->tab.p + b.b_qp);
      p.prog_used = reinterpret_cast<const uint32_t*>(c->tab.p + b.b_pu);
    }
    if (R > 0) {
      const size_t acc_n = static_cast<size_t>(ix.group) * static_cast<size_t>(R);
      if (c->acc.n < acc_n) { AUR_TRY(c->acc.reserve(acc_n)); c->acc_clean = false; }
      if (!c->acc_clean) AUR_TRY(cudaMemsetAsync(c->acc.p, 0, c->acc.n * 8, s));
      c->acc_clean = false;   // until every group's selection has been enqueued
      for (int g0 = 0; g0 < nqb; g0 += ix.group) {
        const int ng = std::min(ix.group, nqb - g0);
        int J = 0;
        for (int i = g0; i < g0 + ng; ++i) J = std::max(J, b.qoff[static_cast<size_t>(i) + 1] - b.qoff[static_cast<size_t>(i)]);
        KwIxTerm t{sn.tpost, sn.toff, sn.ix_terms, kw->d_len.p, reinterpret_cast<const int32_t*>(c->tab.p + b.b_uk), p.idf,
                   p.q_off + g0, p.slot_u, c->acc.p, R, avgdl, 0};
        for (int j = 0; j < J; ++j) {
          int64_t longest = 0;   // the longest list this launch reads
          for (int i = g0; i < g0 + ng; ++i) {
            const int32_t g = b.qoff[static_cast<size_t>(i)] + j;
            if (g < b.qoff[static_cast<size_t>(i) + 1])
              longest = std::max(longest, sn.ulen[static_cast<size_t>(b.ug[static_cast<size_t>(b.slot[static_cast<size_t>(g)])])]);
          }
          if (longest == 0) continue;   // nothing to add at this position
          t.j = j;
          const unsigned gx = static_cast<unsigned>(std::min<int64_t>((longest + 1023) / 1024, 65535));
          kw_ix_term_kernel<<<dim3(gx, static_cast<unsigned>(ng)), 256, 0, s>>>(t);
          AUR_TRY(cudaGetLastError());
          c->launches += 1;
        }
        KwParams ps = p;
        ps.n_rows = R; ps.nq = ng; ps.rows_per_block = rpb_i;
        ps.lists = c->lists_a.p + static_cast<size_t>(g0) * n_lists * ksel;
        if (p.q_user) { ps.q_user = p.q_user + g0; ps.q_org = p.q_org + g0; }
        if (p.q_prog) ps.q_prog = p.q_prog + g0;
        const size_t smem = static_cast<size_t>(ng) * sizeof(Cand) + kKwWarps * kKwBufCap * sizeof(Cand) + 4 * static_cast<size_t>(ng);
        if (d_fmask) kw_ix_select_kernel<true><<<gi, kKwThreads, smem, s>>>(ps, c->acc.p, R, n_lists);
        else kw_ix_select_kernel<false><<<gi, kKwThreads, smem, s>>>(ps, c->acc.p, R, n_lists);
        AUR_TRY(cudaGetLastError());
        c->launches += 1;
      }
      c->acc_clean = true;
      c->path |= AUR_KW_PATH_INDEX;
      c->postings += ix.postings;
    }
    if (tail > 0) {
      // kw_score_kernel over rows [R, n_rows): every row-indexed array starts at row R
      const int g = gt;
      size_t smem = static_cast<size_t>(nqb) * sizeof(Cand) + kKwWarps * kKwBufCap * sizeof(Cand) + 4 * static_cast<size_t>(nqb);
      smem = (smem + 15) & ~size_t(15);
      const size_t cval_smem = static_cast<size_t>(kKwWarps) * nu * 8;
      const bool in_smem = smem + cval_smem <= kw->smem_optin;
      if (!in_smem) ++c->spilled;
      if (in_smem) smem += cval_smem;
      else AUR_TRY(c->cval.reserve(static_cast<size_t>(g) * kKwWarps * nu));
      if (gi) AUR_TRY(c->lists_b.reserve(static_cast<size_t>(nqb) * g * ksel));
      KwParams pf = p;
      pf.off += R; pf.len += R; pf.ids += R; pf.user += R; pf.org += R; pf.live += R;
      if (pf.allow) pf.allow += R;
      if (pf.fmask) pf.fmask += R;
      pf.n_rows = tail; pf.rows_per_block = rpb_t;
      pf.cval_global = in_smem ? nullptr : c->cval.p;
      pf.lists = gi ? c->lists_b.p : c->lists_a.p;
      if (d_fmask) kw_score_kernel<true><<<g, kKwThreads, smem, s>>>(pf, in_smem ? 1 : 0);
      else kw_score_kernel<false><<<g, kKwThreads, smem, s>>>(pf, in_smem ? 1 : 0);
      AUR_TRY(cudaGetLastError());
      c->launches += 1;
      if (gi) {   // into lists gi .. n_lists - 1 of every query
        const size_t w = static_cast<size_t>(g) * ksel * sizeof(Cand);
        AUR_TRY(cudaMemcpy2DAsync(c->lists_a.p + static_cast<size_t>(gi) * ksel, static_cast<size_t>(n_lists) * ksel * sizeof(Cand),
                                  c->lists_b.p, w, w, static_cast<size_t>(nqb), cudaMemcpyDeviceToDevice, s));
      }
      c->path |= AUR_KW_PATH_FORWARD;
      c->postings += sn.post - (R > 0 ? sn.ix_post : 0);
    }
    // fold the per-block lists until one sorted list per query remains
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
        AUR_TRY(cudaGetLastError());
        c->launches += 1;
        break;
      }
      DevBuf<Cand>& dst = in_a ? c->lists_b : c->lists_a;
      AUR_TRY(dst.reserve(static_cast<size_t>(nqb) * n_groups * ksel));
      kw_fold_kernel<<<dim3(n_groups, nqb), 256, fsmem, s>>>(cur, n_lists, ksel, group, sort_n, dst.p, nullptr, nullptr, k);
      AUR_TRY(cudaGetLastError());
      c->launches += 1;
      cur = dst.p; n_lists = n_groups; in_a = !in_a;
    }
  }
  AUR_TRY(cudaEventRecord(c->ev1, s));
  return AUR_OK;
}

// Publish the last_* statistics of a search whose part on c's stream has completed.
int kw_publish(aur_kw* kw, KwCtx* c) {
  float ms = 0.f;
  AUR_TRY(cudaEventElapsedTime(&ms, c->ev0, c->ev1));
  std::lock_guard<std::mutex> lk(kw->mu_last);
  kw->last_launches = c->launches; kw->last_ms = ms;
  kw->last_terms = c->terms; kw->last_spilled = c->spilled;
  kw->last_path = c->path; kw->last_postings = c->postings;
  return AUR_OK;
}

// Wait for one store's part, copy its [nq][k] lists to the host and publish its last_* statistics.
int kw_collect(aur_kw* kw, KwCtx* c, const KwQuery& q, double* scores_out, int64_t* ids_out) {
  AUR_TRY(cudaSetDevice(kw->device));
  cudaStream_t s = c->stream;
  const size_t nout = static_cast<size_t>(q.nq) * q.k;
  AUR_TRY(cudaMemcpyAsync(scores_out, c->out_s.p, nout * 8, cudaMemcpyDeviceToHost, s));
  AUR_TRY(cudaMemcpyAsync(ids_out, c->out_ids.p, nout * 8, cudaMemcpyDeviceToHost, s));
  AUR_TRY(cudaStreamSynchronize(s));
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
// with the idf and avgdl of the union of the snapshots snaps.  Every store's shared lock and every context's lease are
// held until after() has returned; each lease drains its stream before the locks are released (also on an error).
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
  // every store's work enqueued before any is waited on; the leases come after the locks
  std::vector<CtxLease<KwCtx>> leases(static_cast<size_t>(n));
  std::vector<KwCtx*> cs;
  for (int s = 0; s < n; ++s) {
    aur_kw* kw = stores[s];
    AUR_TRY(cudaSetDevice(kw->device));
    int rc = kw->ctxs.lease(&leases[static_cast<size_t>(s)]);
    if (rc != AUR_OK) return rc;
    KwCtx* c = leases[static_cast<size_t>(s)];
    cs.push_back(c);
    const KwSnap& sn = pl.snaps[static_cast<size_t>(s)];
    if ((rc = kw_launch(kw, c, q, pl.blocks, sn, pl.N, pl.avgdl)) != AUR_OK) return rc;
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
            const int32_t* q_user, const int32_t* q_org, const FiltProgs* fp, const KwLegsThen& then) {
  const KwQuery q{q_terms, q_offsets, nq, k, q_user, q_org, nullptr, 0, fp};
  return kw_run(stores, n, q, [&](const std::vector<KwCtx*>& cs, const std::vector<KwSnap>& snaps) -> int {
    std::vector<KwLeg> legs(static_cast<size_t>(n));
    for (int s = 0; s < n; ++s) {
      const KwCtx* c = cs[static_cast<size_t>(s)];
      legs[static_cast<size_t>(s)] = KwLeg{stores[s]->device, c->stream, c->out_s.p, c->out_ids.p, snaps[static_cast<size_t>(s)].n_rows};
    }
    int rc = then(legs);
    if (rc != AUR_OK) return rc;
    for (int s = 0; s < n; ++s) {
      AUR_TRY(cudaSetDevice(stores[s]->device));
      AUR_TRY(cudaStreamSynchronize(cs[static_cast<size_t>(s)]->stream));
      if ((rc = kw_publish(stores[s], cs[static_cast<size_t>(s)])) != AUR_OK) return rc;
    }
    return AUR_OK;
  });
}

int kw_check(const int32_t* q_terms, const int64_t* q_offsets, int32_t nq, int32_t k) {
  return kw_check_query(KwQuery{q_terms, q_offsets, nq, k, nullptr, nullptr, nullptr, 0});
}

int kw_device(const aur_kw* kw) { return kw->device; }
AttrColumns& kw_attrs(aur_kw* kw) { return kw->attrs; }
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
  AUR_TRY(cudaSetDevice(device));
  cudaDeviceProp prop;
  AUR_TRY(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9) return report_error(AUR_ERR_UNSUPPORTED, "sm_%d%d device: this library is built for sm_90a only", prop.major, prop.minor);
  std::unique_ptr<aur_kw> kw(new aur_kw());
  kw->device = device; kw->capacity = doc_capacity;
  kw->ctxs.device = device;
  kw->sm_count = prop.multiProcessorCount; kw->smem_optin = prop.sharedMemPerBlockOptin;
  const cudaError_t e = [&]() -> cudaError_t {
    AUR_CU_RET(kw->stream.create(cudaStreamNonBlocking));
    const size_t cap = static_cast<size_t>(doc_capacity);
    AUR_CU_RET(kw->d_off.reserve(cap + 1));
    AUR_CU_RET(kw->d_len.reserve(cap));
    AUR_CU_RET(kw->d_ids.reserve(cap));
    AUR_CU_RET(kw->d_user.reserve(cap));
    AUR_CU_RET(kw->d_org.reserve(cap));
    AUR_CU_RET(kw->d_live.reserve(cap));
    AUR_CU_RET(kw->d_post.reserve(static_cast<size_t>(postings_capacity ? postings_capacity : (int64_t(1) << 20))));
    AUR_CU_RET(cudaMemset(kw->d_off.p, 0, 8));
    // once, at the device's limit: the attribute belongs to the kernel, not to a search, and searches run concurrently
    AUR_CU_RET(cudaFuncSetAttribute(kw_score_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kw->smem_optin)));
    return cudaFuncSetAttribute(kw_score_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kw->smem_optin));
  }();
  if (e != cudaSuccess)
    return report_error(e == cudaErrorMemoryAllocation ? AUR_ERR_NOMEM : AUR_ERR_CUDA, "aur_kw_open: %s", cudaGetErrorString(e));
  *out = kw.release();
  return AUR_OK;
}

int aur_kw_close(aur_kw* kw) {
  if (!kw) return AUR_OK;
  cudaSetDevice(kw->device);
  if (kw->stream) cudaStreamSynchronize(kw->stream);   // this store's work only: other users of the GPU are not waited on
  delete kw;                                           // (its search contexts are idle: each lease drained its stream)
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
  std::vector<uint2> post(static_cast<size_t>(total));
  for (int64_t j = 0; j < total; ++j) post[static_cast<size_t>(j)] = make_uint2(static_cast<uint32_t>(term_ids[j]), static_cast<uint32_t>(tfs[j]));
  std::vector<int32_t> len(static_cast<size_t>(n));
  for (int64_t i = 0; i < n; ++i) {
    int64_t dl = 0;
    for (int64_t j = offsets[i]; j < offsets[i + 1]; ++j) dl += tfs[j];
    len[static_cast<size_t>(i)] = static_cast<int32_t>(dl);
  }
  std::lock_guard<std::mutex> wk(kw->mu_write);
  const KwRows rows{ids, user_codes, org_codes, offsets, term_ids, len.data(), n, total, max_term};
  int rc = kw_check_room(kw, n);
  if (rc == AUR_OK)
    rc = kw_append_rows(kw, rows, [&](uint2* dst, cudaStream_t s) {
      return total ? cudaMemcpyAsync(dst, post.data(), static_cast<size_t>(total) * 8, cudaMemcpyHostToDevice, s) : cudaSuccess;
    });
  kw_after_append(kw, rc);
  return rc;
}

}  // extern "C"

namespace aur {
int kw_check_room(aur_kw* kw, int64_t n) {
  const int64_t base = static_cast<int64_t>(kw->h_len.size());
  if (base + n > kw->capacity)
    return report_error(AUR_ERR_NOMEM, "keyword store full: %lld + %lld > capacity %lld (aur_kw_compact reclaims tombstones)",
                        (long long)base, (long long)n, (long long)kw->capacity.load());
  return AUR_OK;
}

// The append and publication of r (checked, room checked) shared by aur_kw_add and aur_kw_add_text; the caller holds
// mu_write.  land(dst, stream) enqueues the copy of the rows' r.total postings to dst on the store's stream.
int kw_append_rows(aur_kw* kw, const KwRows& r, const KwLand& land) {
  const int64_t n = r.n, total = r.total;
  const int64_t* ids = r.ids;
  const int64_t base = static_cast<int64_t>(kw->h_len.size());
  const int64_t post0 = kw->h_off.back();
  bool replaces = false;
  for (int64_t i = 0; i < n && !replaces; ++i) replaces = kw->id2row.count(ids[i]) != 0;
  const bool exclusive = replaces || post0 + total > static_cast<int64_t>(kw->d_post.n);
  std::shared_lock<std::shared_mutex> rl(kw->rw, std::defer_lock);
  std::unique_lock<std::shared_mutex> xl(kw->rw, std::defer_lock);
  if (exclusive) xl.lock(); else rl.lock();
  AUR_TRY(cudaSetDevice(kw->device));
  const cudaError_t ge = kw->d_post.grow_keep(static_cast<size_t>(post0 + total), static_cast<size_t>(post0), kw->stream);
  if (ge != cudaSuccess)
    return report_error(ge == cudaErrorMemoryAllocation ? AUR_ERR_NOMEM : AUR_ERR_CUDA, "posting growth: %s", cudaGetErrorString(ge));
  std::vector<int64_t> off(static_cast<size_t>(n));
  std::vector<int32_t> user(static_cast<size_t>(n)), org(static_cast<size_t>(n));
  std::vector<uint8_t> live(static_cast<size_t>(n), 1);
  for (int64_t i = 0; i < n; ++i) {
    off[static_cast<size_t>(i)] = post0 + r.offsets[i + 1];
    user[static_cast<size_t>(i)] = r.user ? r.user[i] : 0;
    org[static_cast<size_t>(i)] = r.org ? r.org[i] : -1;
  }
  // an id repeated inside the batch: its last occurrence wins (the earlier rows land as tombstones)
  std::unordered_map<int64_t, int64_t> last;
  for (int64_t i = 0; i < n; ++i) last[ids[i]] = i;
  for (int64_t i = 0; i < n; ++i) if (last[ids[i]] != i) live[static_cast<size_t>(i)] = 0;
  cudaStream_t s = kw->stream;
  AUR_TRY(land(kw->d_post.p + post0, s));
  AUR_TRY(cudaMemcpyAsync(kw->d_off.p + base + 1, off.data(), static_cast<size_t>(n) * 8, cudaMemcpyHostToDevice, s));
  AUR_TRY(cudaMemcpyAsync(kw->d_len.p + base, r.len, static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, s));
  AUR_TRY(cudaMemcpyAsync(kw->d_ids.p + base, ids, static_cast<size_t>(n) * 8, cudaMemcpyHostToDevice, s));
  AUR_TRY(cudaMemcpyAsync(kw->d_user.p + base, user.data(), static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, s));
  AUR_TRY(cudaMemcpyAsync(kw->d_org.p + base, org.data(), static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, s));
  AUR_TRY(cudaMemcpyAsync(kw->d_live.p + base, live.data(), static_cast<size_t>(n), cudaMemcpyHostToDevice, s));
  AUR_TRY(cudaStreamSynchronize(s));
  for (int64_t i = 0; i < n; ++i) {
    kw->h_off.push_back(off[static_cast<size_t>(i)]);
    kw->h_len.push_back(r.len[i]);
    kw->h_ids.push_back(ids[i]);
    kw->h_user.push_back(user[static_cast<size_t>(i)]);
    kw->h_org.push_back(org[static_cast<size_t>(i)]);
    kw->h_live.push_back(live[static_cast<size_t>(i)]);
  }
  std::lock_guard<std::mutex> st(kw->mu_stat);
  if (static_cast<int64_t>(kw->df.size()) <= r.max_term) kw->df.resize(static_cast<size_t>(r.max_term) + 1, 0);
  if (replaces) {   // exclusive: no search is running, so the old rows and their statistics leave together
    std::vector<int64_t> old;
    for (int64_t i = 0; i < n; ++i) {
      if (last[ids[i]] != i) continue;
      auto it = kw->id2row.find(ids[i]);
      if (it != kw->id2row.end()) old.push_back(it->second);
    }
    const int rc = tombstone_rows(kw, old);
    if (rc != AUR_OK) return rc;
  }
  for (int64_t i = 0; i < n; ++i) {
    if (!live[static_cast<size_t>(i)]) continue;
    kw->id2row[ids[i]] = base + i;
    for (int64_t j = r.offsets[i]; j < r.offsets[i + 1]; ++j) ++kw->df[r.term_ids[j]];
    ++kw->n_live;
    kw->total_len += r.len[i];
  }
  kw->rows_pub = base + n;
  kw->post_pub = post0 + total;
  return AUR_OK;
}

void kw_after_append(aur_kw* kw, int rc) {
  // a failed rebuild (out of memory, say) keeps the previous index and leaves the appended rows to the forward scan:
  // the documents are in, and aur_kw_reindex reports the error
  if (rc == AUR_OK && index_due(kw)) build_index(kw);
}

std::mutex& kw_write_mutex(aur_kw* kw) { return kw->mu_write; }
int64_t kw_rows_appended(const aur_kw* kw) { return static_cast<int64_t>(kw->h_len.size()); }
}  // namespace aur

extern "C" {

int aur_kw_remove(aur_kw* kw, const int64_t* ids, int64_t n, int64_t* removed) {
  if (!kw || (n > 0 && !ids) || n < 0) return report_error(AUR_ERR_INVALID, "null argument or n < 0");
  std::lock_guard<std::mutex> wk(kw->mu_write);
  std::unique_lock<std::shared_mutex> xl(kw->rw);
  AUR_TRY(cudaSetDevice(kw->device));
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
  AUR_TRY(cudaSetDevice(kw->device));
  AUR_TRY(cudaStreamSynchronize(kw->stream));        // searches are host-synchronous: the exclusive lock already drained them
  const int64_t rows = static_cast<int64_t>(kw->h_len.size());
  std::vector<int32_t> map;
  for (int64_t r = 0; r < rows; ++r) if (kw->h_live[static_cast<size_t>(r)]) map.push_back(static_cast<int32_t>(r));
  const int64_t nl = static_cast<int64_t>(map.size());
  if (nl == rows) return AUR_OK;
  const bool reindex = kw->ix_rows > 0;   // rows move: the index is rebuilt over the compacted store
  drop_index(kw);
  // stable: live rows keep their order; postings go to a fresh array of the same capacity
  std::vector<int64_t> off(static_cast<size_t>(nl) + 1, 0), ids(static_cast<size_t>(nl));
  std::vector<int32_t> len(static_cast<size_t>(nl)), user(static_cast<size_t>(nl)), org(static_cast<size_t>(nl));
  for (int64_t j = 0; j < nl; ++j) {
    const size_t r = static_cast<size_t>(map[static_cast<size_t>(j)]);
    off[static_cast<size_t>(j) + 1] = off[static_cast<size_t>(j)] + (kw->h_off[r + 1] - kw->h_off[r]);
    ids[static_cast<size_t>(j)] = kw->h_ids[r]; len[static_cast<size_t>(j)] = kw->h_len[r];
    user[static_cast<size_t>(j)] = kw->h_user[r]; org[static_cast<size_t>(j)] = kw->h_org[r];
  }
  DevBuf<uint2> np;
  cudaStream_t st = kw->stream;
  cudaError_t e = [&]() -> cudaError_t {
    DevBuf<int32_t> d_map, bounce; DevBuf<int64_t> d_noff;
    AUR_CU_RET(np.reserve(kw->d_post.n));
    AUR_CU_RET(d_map.reserve(std::max<size_t>(1, map.size())));
    AUR_CU_RET(d_noff.reserve(off.size()));
    if (nl) AUR_CU_RET(cudaMemcpy(d_map.p, map.data(), map.size() * 4, cudaMemcpyHostToDevice));
    AUR_CU_RET(cudaMemcpy(d_noff.p, off.data(), off.size() * 8, cudaMemcpyHostToDevice));
    if (nl) {
      const int64_t threads = nl * 32;
      kw_gather_postings<<<static_cast<unsigned>((threads + 255) / 256), 256, 0, st>>>(kw->d_post.p, kw->d_off.p, d_map.p, d_noff.p, nl, np.p);
      AUR_CU_RET(cudaGetLastError());
    }
    // attribute codes move with their rows (through a bounce buffer); the rows compaction frees start absent again
    if (kw->attrs.any() && nl) AUR_CU_RET(bounce.reserve(static_cast<size_t>(nl)));
    AUR_CU_RET(kw->attrs.gather(d_map.p, nl, 0, bounce.p, st));
    AUR_CU_RET(kw->attrs.clear(nl, rows, st));
    return cudaStreamSynchronize(st);
  }();
  if (e != cudaSuccess) return report_error(AUR_ERR_CUDA, "aur_kw_compact: %s", cudaGetErrorString(e));
  kw->d_post = std::move(np);
  std::vector<uint8_t> live(static_cast<size_t>(nl), 1);
  e = [&]() -> cudaError_t {
    AUR_CU_RET(cudaMemcpy(kw->d_off.p, off.data(), off.size() * 8, cudaMemcpyHostToDevice));
    if (!nl) return cudaSuccess;
    AUR_CU_RET(cudaMemcpy(kw->d_len.p, len.data(), static_cast<size_t>(nl) * 4, cudaMemcpyHostToDevice));
    AUR_CU_RET(cudaMemcpy(kw->d_ids.p, ids.data(), static_cast<size_t>(nl) * 8, cudaMemcpyHostToDevice));
    AUR_CU_RET(cudaMemcpy(kw->d_user.p, user.data(), static_cast<size_t>(nl) * 4, cudaMemcpyHostToDevice));
    AUR_CU_RET(cudaMemcpy(kw->d_org.p, org.data(), static_cast<size_t>(nl) * 4, cudaMemcpyHostToDevice));
    return cudaMemcpy(kw->d_live.p, live.data(), static_cast<size_t>(nl), cudaMemcpyHostToDevice);
  }();
  if (e != cudaSuccess) return report_error(AUR_ERR_CUDA, "aur_kw_compact: %s (the store may be inconsistent: rebuild it)", cudaGetErrorString(e));
  kw->h_off = off; kw->h_len = len; kw->h_ids = ids; kw->h_user = user; kw->h_org = org; kw->h_live = live;
  kw->id2row.clear();
  for (int64_t j = 0; j < nl; ++j) kw->id2row[ids[static_cast<size_t>(j)]] = j;
  {
    std::lock_guard<std::mutex> st(kw->mu_stat);
    kw->rows_pub = nl;
    kw->post_pub = off.back();
  }
  if (reclaimed) *reclaimed = rows - nl;
  xl.unlock();
  return reindex ? build_index(kw) : AUR_OK;
}

int aur_kw_get_stats(aur_kw* kw, aur_kw_stats* out) {
  if (!kw || !out) return report_error(AUR_ERR_INVALID, "null argument");
  memset(out, 0, sizeof *out);
  {
    std::lock_guard<std::mutex> st(kw->mu_stat);
    out->docs = kw->rows_pub; out->live = kw->n_live; out->total_len = kw->total_len;
    out->postings_used = kw->post_pub;
  }
  std::lock_guard<std::mutex> lk(kw->mu_last);
  out->postings_allocated = static_cast<int64_t>(kw->d_post.n);
  out->capacity = kw->capacity;
  out->last_launches = kw->last_launches;
  out->last_ms = kw->last_ms;
  out->last_terms = kw->last_terms;
  out->last_spilled = kw->last_spilled;
  return AUR_OK;
}

int aur_kw_set_attrs(aur_kw* kw, int32_t col, const int64_t* ids, const int32_t* codes, int64_t n) {
  if (!kw || n < 0 || (n > 0 && (!ids || !codes))) return report_error(AUR_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> wk(kw->mu_write);
  std::shared_lock<std::shared_mutex> rl(kw->rw);
  AUR_TRY(cudaSetDevice(kw->device));
  std::vector<int32_t> pairs;   // (row, code); id2row changes only under mu_write, which this call holds
  pairs.reserve(2 * static_cast<size_t>(n));
  for (int64_t i = 0; i < n; ++i) {
    auto it = kw->id2row.find(ids[i]);
    if (it != kw->id2row.end()) { pairs.push_back(static_cast<int32_t>(it->second)); pairs.push_back(codes[i]); }
  }
  return kw->attrs.write(col, pairs, kw->capacity.load(), kw->stream);   // the store's capacity, like its tenant codes
}

int aur_kw_reserve(aur_kw* kw, int64_t doc_capacity) {
  if (!kw) return report_error(AUR_ERR_INVALID, "null store");
  if (doc_capacity > kKwMaxRows) return report_error(AUR_ERR_INVALID, "doc_capacity exceeds 2^31 - 64");
  std::lock_guard<std::mutex> wk(kw->mu_write);
  const int64_t old_cap = kw->capacity.load();
  if (doc_capacity <= old_cap) return AUR_OK;
  // the per-document arrays move: every keyword search is a host call under the shared lock, so none holds them now
  std::unique_lock<std::shared_mutex> xl(kw->rw);
  AUR_TRY(cudaSetDevice(kw->device));
  const size_t cap = static_cast<size_t>(doc_capacity), used = kw->h_len.size();
  cudaStream_t st = kw->stream;
  const cudaError_t e = [&]() -> cudaError_t {
    AUR_CU_RET(kw->d_off.grow_keep(cap + 1, used + 1, st));
    AUR_CU_RET(kw->d_len.grow_keep(cap, used, st));
    AUR_CU_RET(kw->d_ids.grow_keep(cap, used, st));
    AUR_CU_RET(kw->d_user.grow_keep(cap, used, st));
    AUR_CU_RET(kw->d_org.grow_keep(cap, used, st));
    AUR_CU_RET(kw->d_live.grow_keep(cap, used, st));
    return kw->attrs.grow(old_cap, doc_capacity, st);
  }();
  if (e != cudaSuccess)   // arrays that did grow keep their rows and the old capacity still holds
    return report_error(e == cudaErrorMemoryAllocation ? AUR_ERR_NOMEM : AUR_ERR_CUDA, "aur_kw_reserve(%lld): %s (the store keeps %lld rows)",
                        (long long)doc_capacity, cudaGetErrorString(e), (long long)old_cap);
  kw->h_off.reserve(cap + 1); kw->h_len.reserve(cap); kw->h_ids.reserve(cap);
  kw->h_user.reserve(cap); kw->h_org.reserve(cap); kw->h_live.reserve(cap);
  kw->capacity.store(doc_capacity);
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

int aur_kw_read_rows(aur_kw* kw, int64_t row0, int64_t n, int64_t* ids_out, int64_t* offsets_out, int32_t* term_ids_out,
                     int32_t* tfs_out, int64_t cap, int64_t* postings_out) {
  if (!kw || !offsets_out || !postings_out) return report_error(AUR_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> wk(kw->mu_write);   // the host mirrors change only under mu_write
  std::shared_lock<std::shared_mutex> rl(kw->rw);
  int64_t rows = 0;
  {
    std::lock_guard<std::mutex> st(kw->mu_stat);
    rows = kw->rows_pub;
  }
  if (row0 < 0 || n < 0 || row0 + n > rows)
    return report_error(AUR_ERR_INVALID, "rows [%lld, %lld) outside the published %lld", (long long)row0, (long long)(row0 + n),
                        (long long)rows);
  const int64_t p0 = kw->h_off[static_cast<size_t>(row0)], total = kw->h_off[static_cast<size_t>(row0 + n)] - p0;
  for (int64_t i = 0; i <= n; ++i) offsets_out[i] = kw->h_off[static_cast<size_t>(row0 + i)] - p0;
  if (ids_out) std::copy(kw->h_ids.begin() + row0, kw->h_ids.begin() + row0 + n, ids_out);
  *postings_out = total;
  if (!term_ids_out || !tfs_out || cap < total || total == 0) return AUR_OK;   // count mode
  AUR_TRY(cudaSetDevice(kw->device));
  std::vector<uint2> post(static_cast<size_t>(total));
  AUR_TRY(cudaMemcpyAsync(post.data(), kw->d_post.p + p0, static_cast<size_t>(total) * 8, cudaMemcpyDeviceToHost, kw->stream));
  AUR_TRY(cudaStreamSynchronize(kw->stream));
  for (int64_t j = 0; j < total; ++j) {
    term_ids_out[j] = static_cast<int32_t>(post[static_cast<size_t>(j)].x);
    tfs_out[j] = static_cast<int32_t>(post[static_cast<size_t>(j)].y);
  }
  return AUR_OK;
}

int aur_kw_reindex(aur_kw* kw) {
  if (!kw) return report_error(AUR_ERR_INVALID, "null store");
  std::lock_guard<std::mutex> wk(kw->mu_write);
  return build_index(kw);
}

int aur_kw_set_option(aur_kw* kw, const char* name, int64_t value) {
  if (!kw || !name) return report_error(AUR_ERR_INVALID, "null argument");
  if (strcmp(name, "kw_path") == 0) {
    if (value < 0 || value > 2) return report_error(AUR_ERR_INVALID, "kw_path must be 0 (auto), 1 (forward) or 2 (index)");
    kw->kw_path.store(static_cast<int>(value));
    return AUR_OK;
  }
  return report_error(AUR_ERR_INVALID, "unknown keyword store option '%s'", name);
}

int aur_kw_get_index_stats(aur_kw* kw, aur_kw_index_stats* out) {
  if (!kw || !out) return report_error(AUR_ERR_INVALID, "null argument");
  memset(out, 0, sizeof *out);
  {
    std::lock_guard<std::mutex> st(kw->mu_stat);
    out->indexed_rows = kw->ix_rows;
    out->index_postings = kw->ix_post;
    out->index_bytes = kw->d_toff.p ? kw->ix_post * 8 + (kw->ix_terms + 1) * 8 : 0;
    out->builds = kw->ix_builds;
    out->last_build_ms = kw->ix_build_ms;
  }
  std::lock_guard<std::mutex> lk(kw->mu_last);
  out->last_path = kw->last_path;
  out->last_postings = kw->last_postings;
  return AUR_OK;
}

}  // extern "C"
