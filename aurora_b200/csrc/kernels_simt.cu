// CUDA-core kernels of the retrieval path: ingest-time inverse norms, the generic
// (any dim / dtype / tenant-filter) similarity path, candidate-list reduction, the exact
// fp64 re-rank that fixes the final (score desc, id asc) order, the cross-shard merge and
// the pairwise cosine that mirrors SimilarityStrategy._cosine_similarity.
#include <math.h>
#include <string.h>
#include <type_traits>
#include "internal.h"

namespace aur {
namespace {

template <typename T> __device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <> __device__ __forceinline__ float to_f32<int8_t>(int8_t v) { return static_cast<float>(v); }

__device__ __forceinline__ double warp_sum_lane0(double v) {
  // shfl_down tree: lane 0 ends with a value whose association order is fixed, so the
  // result for a row depends only on the row's content.
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return __shfl_sync(0xffffffffu, v, 0);
}

__device__ __forceinline__ uint64_t ld_acquire_sys(const uint64_t* p) {
  uint64_t v; asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ void st_release_sys(uint64_t* p, uint64_t v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// --------------------------------------------------------------------------------------
// Inverse L2 norm per appended row (one warp per row).  Weaviate normalises vectors at
// import for the cosine metric; we keep the raw rows and this scale beside them.
template <typename T>
__global__ void row_inv_norm_kernel(const T* __restrict__ rows, int dim, int64_t n, float* __restrict__ inv_norm) {
  const int64_t row = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= n) return;
  const T* p = rows + row * dim;
  float ss = 0.f;
  for (int i = lane; i < dim; i += 32) { const float v = to_f32(p[i]); ss = fmaf(v, v, ss); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if (lane == 0) inv_norm[row] = ss > 0.f ? 1.0f / sqrtf(ss) : 0.f;
}

// Ingest into an int8 shard (AUR_I8), one warp per row: amax = max |x| (exact), q = rint(x * 127 / amax) with an exact
// fp64 product and one correctly rounded fp64 division (oracle/quantize.py), then the inverse norm of the int8 row in
// row_inv_norm_kernel's summation order, so an int8 row and the same values stored as bf16 get the same scale bit for
// bit.  An all-zero row stays zero with scale 0.  A row holding a NaN or +-inf is stored as zeros with scale +inf: its
// first-pass score 0 * inf is NaN on every path, which no selection admits -- never returned, as in a bf16 shard, where
// such a row scores NaN -- while it stays live for exports and filters (a tombstone is a NaN scale).
__global__ void quantize_rows_i8_kernel(const __nv_bfloat16* __restrict__ in, int dim, int64_t n, int8_t* __restrict__ out,
                                        float* __restrict__ inv_norm) {
  const int64_t row = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= n) return;
  const __nv_bfloat16* p = in + row * dim;
  int8_t* o = out + row * dim;
  float amax = 0.f;
  bool finite = true;
  for (int i = lane; i < dim; i += 32) {
    const float v = __bfloat162float(p[i]);
    finite = finite && isfinite(v);
    amax = fmaxf(amax, fabsf(v));
  }
#pragma unroll
  for (int o2 = 16; o2 > 0; o2 >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o2));
  finite = __all_sync(0xffffffffu, finite);
  const double a = static_cast<double>(amax);
  float ss = 0.f;
  for (int i = lane; i < dim; i += 32) {
    int8_t q = 0;
    if (finite && amax > 0.f)
      q = static_cast<int8_t>(rint(__ddiv_rn(__dmul_rn(static_cast<double>(__bfloat162float(p[i])), 127.0), a)));
    o[i] = q;
    const float v = static_cast<float>(q);
    ss = fmaf(v, v, ss);
  }
#pragma unroll
  for (int o2 = 16; o2 > 0; o2 >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o2);
  if (lane == 0) inv_norm[row] = !finite ? INFINITY : (ss > 0.f ? 1.0f / sqrtf(ss) : 0.f);
}

// The tensor-core kernel's query operand for an int8 shard, one warp per query: q16 = rint(q * 32512 / amax) (exact
// fp64 product, one rounded division; a zero query stays 0), split exactly as q16 = 256 hi + lo with hi = (q16 + 128) >> 8
// in [-127, 127] and lo in [-128, 127].  Row q of the output is [dim / 128][hi 128 B | lo 128 B]: dim * 2 bytes, the size
// of the bf16 query row the kernel's staging copies.  Rounding to 16 bits moves a cosine by at most about
// sqrt(dim) / 65024 relative to |q|: the re-rank's k + 8 slack covers it as it covers fp32 noise on bf16 rows.
__global__ void query_image_i8_kernel(const __nv_bfloat16* __restrict__ q, int dim, int nq, int8_t* __restrict__ out) {
  const int64_t qi = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (qi >= nq) return;
  const __nv_bfloat16* p = q + qi * dim;
  int8_t* o = out + qi * dim * 2;
  float amax = 0.f;
  for (int i = lane; i < dim; i += 32) amax = fmaxf(amax, fabsf(__bfloat162float(p[i])));
#pragma unroll
  for (int o2 = 16; o2 > 0; o2 >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o2));
  const double a = static_cast<double>(amax);
  for (int i = lane; i < dim; i += 32) {
    int v = 0;
    if (amax > 0.f && isfinite(amax))
      v = static_cast<int>(rint(__ddiv_rn(__dmul_rn(static_cast<double>(__bfloat162float(p[i])), 32512.0), a)));
    const int hi = (v + 128) >> 8, lo = v - 256 * hi;
    int8_t* blk = o + (i / 128) * 256 + (i % 128);
    blk[0] = static_cast<int8_t>(hi);
    blk[128] = static_cast<int8_t>(lo);
  }
}

// --------------------------------------------------------------------------------------
// Generic similarity: 64 queries x 64 rows per block, 4x4 per thread, fp32 FMA.
constexpr int kSB = 64, kSK = 16;
template <typename T, typename TR = T>
__global__ void __launch_bounds__(256)
simt_scores_kernel(const T* __restrict__ q, const TR* __restrict__ rows, int dim, int nq, int64_t row0,
                   int64_t nrows_chunk, int64_t n_rows, const float* __restrict__ inv_norm, FilterArgs f,
                   float* __restrict__ scores) {
  __shared__ float Qs[kSK][kSB + 1];
  __shared__ float Cs[kSK][kSB + 1];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int q0 = blockIdx.y * kSB;
  const int64_t c0 = static_cast<int64_t>(blockIdx.x) * kSB;  // within chunk
  float acc[4][4] = {};
  for (int k0 = 0; k0 < dim; k0 += kSK) {
    for (int i = threadIdx.x; i < kSB * kSK; i += 256) {
      const int rr = i / kSK, kk = i % kSK;
      const int k = k0 + kk;
      float qv = 0.f, cv = 0.f;
      if (k < dim) {
        if (q0 + rr < nq) qv = to_f32(q[static_cast<size_t>(q0 + rr) * dim + k]);
        const int64_t row = row0 + c0 + rr;
        if (c0 + rr < nrows_chunk && row < n_rows) cv = to_f32(rows[row * dim + k]);
      }
      Qs[kk][rr] = qv; Cs[kk][rr] = cv;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kSK; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = Qs[kk][ty * 4 + i]; b[i] = Cs[kk][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int qi = q0 + ty * 4 + i;
    if (qi >= nq) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int64_t cj = c0 + tx * 4 + j;
      if (cj >= nrows_chunk) continue;
      const int64_t row = row0 + cj;
      float s = -INFINITY;
      if (row < n_rows) {
        const float nv = inv_norm[row];
        bool ok = (nv == nv);  // NaN = tombstone
        if (ok && f.q_user != nullptr) {
          // weaviate_client.py:244-249: user_id == u OR (org given AND org_id == o)
          const int32_t qo = f.q_org ? f.q_org[qi] : -1;
          ok = (f.row_user[row] == f.q_user[qi]) || (qo >= 0 && f.row_org[row] == qo);
        }
        if (ok) s = acc[i][j] * nv;
      }
      scores[static_cast<size_t>(qi) * nrows_chunk + cj] = s;
    }
  }
}

// --------------------------------------------------------------------------------------
// Block-wide bitonic sort, descending, n a power of two >= 64, keys in shared memory.
// A step (k, j) compares elements i and i ^ j.  All steps with j <= 32 stay inside an aligned block of 64 keys: a warp
// takes such a block into registers (two keys per lane: i and i + 32), runs those steps with shuffles and writes the
// block back -- no block barrier in between.  Only the steps with j >= 64 go through shared memory with a barrier
// each.  A 512-key sort needs 10 barriers instead of 45; the exact-re-rank kernel is a latency chain and most of its
// time used to be spent waiting at them.
__device__ __forceinline__ uint64_t shfl_xor_u64(uint64_t v, int m) {
  const uint32_t lo = __shfl_xor_sync(0xffffffffu, static_cast<uint32_t>(v), m);
  const uint32_t hi = __shfl_xor_sync(0xffffffffu, static_cast<uint32_t>(v >> 32), m);
  return (static_cast<uint64_t>(hi) << 32) | lo;
}
// Keys are ordered by key_before (score desc, id asc); ids = the rows' external ids.
// Steps j = j_hi, j_hi / 2, ..., 1 of level k on every 64-key block (j_hi <= 32); with all_levels, levels 2 .. 64 in full.
__device__ void bitonic_local64(uint64_t* s, int n, int k, bool all_levels, const int64_t* ids) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (int base = warp * 64; base < n; base += nwarps * 64) {
    const int i0 = base + lane, i1 = i0 + 32;
    uint64_t e0 = s[i0], e1 = s[i1];
    auto step = [&](int kk, int j) {
      if (j == 32) {
        const bool desc = (i0 & kk) == 0;
        if (desc ? key_before(e1, e0, ids) : key_before(e0, e1, ids)) { const uint64_t t = e0; e0 = e1; e1 = t; }
      } else {
        const uint64_t o0 = shfl_xor_u64(e0, j), o1 = shfl_xor_u64(e1, j);
        const bool lower = (lane & j) == 0;
        const bool want_max0 = ((i0 & kk) == 0) == lower, want_max1 = ((i1 & kk) == 0) == lower;
        const bool b0 = key_before(e0, o0, ids), b1 = key_before(e1, o1, ids);
        e0 = want_max0 == b0 ? e0 : o0;
        e1 = want_max1 == b1 ? e1 : o1;
      }
    };
    if (all_levels) {
      for (int kk = 2; kk <= 64; kk <<= 1)
        for (int j = kk >> 1; j > 0; j >>= 1) step(kk, j);
    } else {
      for (int j = 32; j > 0; j >>= 1) step(k, j);
    }
    s[i0] = e0; s[i1] = e1;
  }
  __syncthreads();
}
__device__ void bitonic_desc(uint64_t* s, int n, const int64_t* ids) {
  bitonic_local64(s, n, 0, true, ids);
  for (int k = 128; k <= n; k <<= 1) {
    for (int j = k >> 1; j >= 64; j >>= 1) {
      for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int l = i ^ j;
        if (l > i) {
          const uint64_t a = s[i], b = s[l];
          const bool desc = (i & k) == 0;
          if (desc ? key_before(b, a, ids) : key_before(a, b, ids)) { s[i] = b; s[l] = a; }
        }
      }
      __syncthreads();
    }
    bitonic_local64(s, n, k, false, ids);
  }
}

// One block per (segment of kSimtSeg scores, query): keep the best ksel as keys.
__global__ void __launch_bounds__(256)
simt_select_kernel(const float* __restrict__ scores, int64_t row0, int64_t nrows_chunk, int ksel,
                   const int64_t* __restrict__ ids, uint64_t* __restrict__ cand, int n_lists, int list0) {
  __shared__ uint64_t keys[kSimtSeg];
  const int seg = blockIdx.x, qi = blockIdx.y;
  const int64_t base = static_cast<int64_t>(seg) * kSimtSeg;
  for (int i = threadIdx.x; i < kSimtSeg; i += blockDim.x) {
    const int64_t cj = base + i;
    uint64_t key = 0;
    if (cj < nrows_chunk) {
      const float s = scores[static_cast<size_t>(qi) * nrows_chunk + cj];
      key = (s == -INFINITY || s != s) ? kKeyEmpty : make_key(s, static_cast<int32_t>(row0 + cj));
    }
    keys[i] = key;
  }
  __syncthreads();
  bitonic_desc(keys, kSimtSeg, ids);
  uint64_t* out = cand + (static_cast<size_t>(qi) * n_lists + list0 + seg) * ksel;
  for (int t = threadIdx.x; t < ksel; t += blockDim.x) out[t] = keys[t] == 0 ? kKeyEmpty : keys[t];
}

constexpr int kSortCap = 4096;

// [nq, n_lists, ksel] -> [nq, n_groups, ksel]
__global__ void __launch_bounds__(512)
reduce_lists_kernel(const uint64_t* __restrict__ in, int n_lists, int ksel, int group, const int64_t* __restrict__ ids,
                    uint64_t* __restrict__ out, int n_groups) {
  extern __shared__ uint64_t skeys[];
  const int g = blockIdx.x, qi = blockIdx.y;
  const int l0 = g * group, l1 = min(n_lists, l0 + group);
  const int n = (l1 - l0) * ksel;
  int P = 64; while (P < n) P <<= 1;
  const uint64_t* src = in + (static_cast<size_t>(qi) * n_lists + l0) * ksel;
  for (int i = threadIdx.x; i < P; i += blockDim.x) skeys[i] = i < n ? src[i] : 0ull;
  __syncthreads();
  bitonic_desc(skeys, P, ids);
  uint64_t* dst = out + (static_cast<size_t>(qi) * n_groups + g) * ksel;
  for (int t = threadIdx.x; t < ksel; t += blockDim.x) dst[t] = (t < P && skeys[t] != 0) ? skeys[t] : kKeyEmpty;
}

// --------------------------------------------------------------------------------------
// Finalize: best ksel approximate candidates -> exact fp64 cosine -> (score desc, id asc).
// T: the query's element type, TR: the rows' (int8 rows take bf16 queries).
template <typename T, typename TR = T>
__global__ void __launch_bounds__(256, 2)
finalize_kernel(FinalizeArgs a) {
  extern __shared__ uint64_t skeys[];
  __shared__ double ex_score[kMaxK + kSlack];
  __shared__ int64_t ex_id[kMaxK + kSlack];
  __shared__ double s_qq;
  __shared__ uint64_t topkeys[kMaxK + kSlack];
  const int qi = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  // ---- prologue, independent of the similarity kernel (launched with programmatic dependent launch, so this part
  //      overlaps that kernel's tail): the query goes to shared memory once (as fp32, exact for bf16 / f32), |q|^2
  const TR* rows = static_cast<const TR*>(a.rows);
  const T* qv = static_cast<const T*>(a.q) + static_cast<size_t>(qi) * a.dim;
  float* qs = reinterpret_cast<float*>(skeys + a.sort_cap);      // [dim] behind the sort buffer
  for (int i = threadIdx.x; i < a.dim; i += blockDim.x) qs[i] = to_f32(qv[i]);
  __syncthreads();
  if (warp == 0) {
    double qq = 0.0;
    for (int i = lane; i < a.dim; i += 32) { const double v = static_cast<double>(qs[i]); qq = fma(v, v, qq); }
    qq = warp_sum_lane0(qq);
    if (lane == 0) s_qq = sqrt(qq);          // |q|: one fp64 square root per query, not one per candidate
  }
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");     // the candidate lists come from the previous kernel
  if (a.epoch_bump && blockIdx.x == 0 && threadIdx.x == 0) {   // that kernel is complete: next launch, next epoch
    const uint32_t e = *a.epoch_bump;
    *a.epoch_bump = e >= kSearchEpochMax ? 1u : e + 1u;
  }

  const int cap = a.n_lists * a.ksel;                       // row stride of cand
  const uint64_t* src = a.cand + static_cast<size_t>(qi) * cap;
  // the first keys of the row are requested together with the count that says how many of them are valid: one global
  // round trip instead of two (slots past the count hold stale keys of earlier searches and are masked below)
  uint64_t spec[2];
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const int i = threadIdx.x + u * 256;
    spec[u] = (a.counts && i < cap) ? src[i] : 0ull;
  }
  const int n = a.counts ? min(static_cast<int>(a.counts[qi]), cap) : cap;
  if (a.cand_read && threadIdx.x == 0) a.cand_read[qi] = static_cast<uint32_t>(n);
  // Sort in rounds of at most sort_cap keys; the best ksel of earlier rounds ride along
  // at the front.  (One round unless a compacted row overflows the sort buffer.)
  int P = 1;
  {
    int done = 0, carried = 0;
    do {
      const int take = min(n - done, a.sort_cap - carried);
      const int m = carried + take;
      P = 64; while (P < m) P <<= 1;
      if (a.counts && done == 0 && blockDim.x == 256) {      // first round: the speculative loads cover slots 0 .. 511
        if (static_cast<int>(threadIdx.x) < P) skeys[threadIdx.x] = (static_cast<int>(threadIdx.x) < m) ? spec[0] : 0ull;
        if (static_cast<int>(threadIdx.x) + 256 < P) skeys[threadIdx.x + 256] = (static_cast<int>(threadIdx.x) + 256 < m) ? spec[1] : 0ull;
        for (int i = threadIdx.x + 512; i < P; i += blockDim.x) skeys[i] = (i < m) ? src[i] : 0ull;
      } else {
        for (int i = carried + threadIdx.x; i < P; i += blockDim.x) skeys[i] = (i < m) ? src[done + i - carried] : 0ull;
      }
      __syncthreads();
      bitonic_desc(skeys, P, a.ids);
      done += take;
      carried = min(a.ksel, m);
    } while (done < n);
  }
  __syncthreads();
  if (a.counts && threadIdx.x == 0) a.counts[qi] = 0;      // ready for the next launch

  // Exact re-score: a warp takes one candidate: lanes stride over 16-byte pieces of the row, fp64 FMA, fixed
  // shuffle tree -- a row's score depends only on its content, never on where it is stored.
  const int ncand = min(a.ksel, P);
  for (int c = threadIdx.x; c < ncand; c += blockDim.x) topkeys[c] = skeys[c];
  __syncthreads();
  // elements per piece: a 16-byte piece of bf16 / f32 rows; int8 rows are read 8 bytes at a time, so that every lane
  // sums the same elements in the same order as for the row stored as bf16
  constexpr int kVec = sizeof(TR) == 1 ? 8 : 16 / static_cast<int>(sizeof(TR));
  using Piece = typename std::conditional<sizeof(TR) == 1, uint2, uint4>::type;
  const bool vec_ok = (a.dim % kVec) == 0;
  // kRe candidates per warp and step, strided by the warp count, with every row load (and the id load)
  // issued before any arithmetic: at k+slack = 40 and 8 warps x 5 all candidate rows of the query are in
  // flight at once, so the gather costs one HBM round trip instead of one per pass.
  constexpr int kRe = 5, kMaxCh = 4;                                // rows per step; 16-byte pieces per lane (dim <= 1024 bf16)
  const int n_chunks = vec_ok ? a.dim / kVec : 0;
  const bool reg_path = vec_ok && n_chunks <= 32 * kMaxCh;
  for (int c0 = warp; c0 < ncand; c0 += kRe * nwarps) {
    int32_t row[kRe]; const TR* rv[kRe]; int64_t idv[kRe];
    double dot[kRe], cc[kRe];
#pragma unroll
    for (int h = 0; h < kRe; ++h) {
      const int c = c0 + h * nwarps;
      const uint64_t key = (c < ncand) ? topkeys[c] : 0ull;
      row[h] = (key == 0) ? -1 : key_row(key);
      rv[h] = rows + static_cast<size_t>(row[h] < 0 ? 0 : row[h]) * a.dim;
      dot[h] = 0.0; cc[h] = 0.0;
    }
    if (reg_path) {
      Piece raw[kRe][kMaxCh];
#pragma unroll
      for (int h = 0; h < kRe; ++h)
#pragma unroll
        for (int i = 0; i < kMaxCh; ++i) {
          const int ch = lane + 32 * i;
          raw[h][i] = (row[h] >= 0 && ch < n_chunks) ? __ldg(reinterpret_cast<const Piece*>(rv[h]) + ch) : Piece{};
        }
#pragma unroll
      for (int h = 0; h < kRe; ++h) idv[h] = (row[h] >= 0) ? __ldg(a.ids + row[h]) : -1;
#pragma unroll
      for (int h = 0; h < kRe; ++h)
#pragma unroll
        for (int i = 0; i < kMaxCh; ++i) {
          const int ch = lane + 32 * i;
          if (ch < n_chunks) {
            TR el[kVec];
            memcpy(el, &raw[h][i], sizeof(Piece));
#pragma unroll
            for (int e = 0; e < kVec; ++e) {
              const double x = static_cast<double>(qs[ch * kVec + e]), y = static_cast<double>(to_f32(el[e]));
              dot[h] = fma(x, y, dot[h]); cc[h] = fma(y, y, cc[h]);
            }
          }
        }
    } else {
#pragma unroll
      for (int h = 0; h < kRe; ++h) idv[h] = (row[h] >= 0) ? __ldg(a.ids + row[h]) : -1;
      for (int i = lane; i < a.dim; i += 32) {
#pragma unroll
        for (int h = 0; h < kRe; ++h) {
          if (row[h] < 0) continue;
          const double x = static_cast<double>(qs[i]), y = static_cast<double>(to_f32(rv[h][i]));
          dot[h] = fma(x, y, dot[h]); cc[h] = fma(y, y, cc[h]);
        }
      }
    }
    // the kRe reduced (dot, |row|^2) pairs land in lanes 0 .. kRe-1, which then do the fp64 square root and division
    // side by side (software sequences of a few hundred cycles each: one after the other on lane 0 they were a
    // tenth of this kernel)
    double my_d = 0.0, my_n2 = 0.0; int64_t my_id = -1; int my_row = -1;
#pragma unroll
    for (int h = 0; h < kRe; ++h) {
      double d = 0.0, n2 = 0.0;
      if (row[h] >= 0) { d = warp_sum_lane0(dot[h]); n2 = warp_sum_lane0(cc[h]); }   // warp-uniform
      d = __shfl_sync(0xffffffffu, d, 0); n2 = __shfl_sync(0xffffffffu, n2, 0);
      if (lane == h) { my_d = d; my_n2 = n2; my_id = idv[h]; my_row = row[h]; }
    }
    if (lane < kRe) {
      const int c = c0 + lane * nwarps;
      if (c < ncand) {
        double sc = -INFINITY; int64_t id = -1;
        if (my_row >= 0) {
          const double den = s_qq * sqrt(my_n2);
          sc = den > 0.0 ? my_d / den : 0.0;  // zero norm -> 0.0 (similarity.py:94-95)
          id = my_id;
        }
        ex_score[c] = sc; ex_id[c] = id;
      }
    }
  }
  __syncthreads();
  // where a result row goes: local arrays and / or this rank's slot in every rank's exchange buffer (peer stores)
  const uint64_t ex_seq = (a.ex.n_peers > 0) ? (*a.ex.seq + 1) : 0ull;
  const uint64_t ex_par = (ex_seq & 1ull) * a.ex.parity_stride;
  const uint64_t ex_tag = (ex_seq & 0xFFFFFFFFull) << 32;
  auto emit = [&](int pos, double s, int64_t id) {
    const size_t o = static_cast<size_t>(qi) * a.k + pos;
    if (a.out_scores) { a.out_scores[o] = static_cast<float>(s); a.out_ids[o] = id; }
    if (a.out_scores64) a.out_scores64[o] = s;
    if (a.ex.n_peers > 0) {
      const size_t w = ex_par + (static_cast<size_t>(a.ex.q0 + qi) * a.k + pos) * 4;
      const uint64_t sb = static_cast<uint64_t>(__double_as_longlong(s)), ib = static_cast<uint64_t>(id);
      const uint64_t w0 = ex_tag | (sb & 0xFFFFFFFFull), w1 = ex_tag | (sb >> 32);
      const uint64_t w2 = ex_tag | (ib & 0xFFFFFFFFull), w3 = ex_tag | (ib >> 32);
#pragma unroll 1
      for (int r = 0; r < a.ex.n_peers; ++r) {
        ulonglong2* dst = reinterpret_cast<ulonglong2*>(a.ex.slot[r] + w);      // two 16-byte stores (each word valid on its own)
        dst[0] = make_ulonglong2(w0, w1);
        dst[1] = make_ulonglong2(w2, w3);
      }
    }
  };
  // rank by counting: ids are unique, so (score desc, id asc) is a total order.  The ncand^2 comparisons are spread
  // over the whole block (candidate t = thread / 4, every 4th opponent), partial counts meet in a quad shuffle.
  const int nvalid = __syncthreads_count(static_cast<int>(threadIdx.x) < ncand && ex_id[threadIdx.x < ncand ? threadIdx.x : 0] >= 0);
  for (int t0 = 0; t0 < ncand; t0 += blockDim.x / 4) {
    const int t = t0 + (threadIdx.x >> 2), part = threadIdx.x & 3;
    const bool live = t < ncand;
    const double s = live ? ex_score[t] : 0.0; const int64_t id = live ? ex_id[t] : -1;
    int rank = 0;
    if (id >= 0)
      for (int u = part; u < ncand; u += 4) {
        const double su = ex_score[u]; const int64_t iu = ex_id[u];
        if (iu >= 0 && (su > s || (su == s && iu < id))) ++rank;
      }
    rank += __shfl_xor_sync(0xffffffffu, rank, 1);
    rank += __shfl_xor_sync(0xffffffffu, rank, 2);
    if (part == 0 && id >= 0 && rank < a.k) emit(rank, s, id);
  }
  for (int t = nvalid + threadIdx.x; t < a.k; t += blockDim.x) emit(t, -INFINITY, -1);
}

// Cross-shard merge of exact (fp64 score, id) lists: [n_shards, nq, k] -> [nq, k].
__global__ void __launch_bounds__(256)
merge_topk_kernel(const double* __restrict__ in_s, const int64_t* __restrict__ in_ids, size_t shard_stride, int n_shards,
                  int nq, int k, float* out_s, int64_t* out_ids, double* out_s64) {
  extern __shared__ uint8_t sm[];
  double* sc = reinterpret_cast<double*>(sm);
  int64_t* id = reinterpret_cast<int64_t*>(sc + n_shards * k);
  __shared__ int s_nvalid;
  const int qi = blockIdx.x, n = n_shards * k;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int sh = i / k, t = i % k;
    const size_t o = static_cast<size_t>(sh) * shard_stride + static_cast<size_t>(qi) * k + t;
    sc[i] = in_s[o]; id[i] = in_ids[o];
  }
  if (threadIdx.x == 0) s_nvalid = 0;
  __syncthreads();
  int local_valid = 0;
  for (int t = threadIdx.x; t < n; t += blockDim.x) {
    const double s = sc[t]; const int64_t me = id[t];
    if (me < 0) continue;
    ++local_valid;
    int rank = 0;
    for (int u = 0; u < n; ++u) {
      const double su = sc[u]; const int64_t iu = id[u];
      if (iu >= 0 && (su > s || (su == s && iu < me))) ++rank;
    }
    if (rank < k) {
      const size_t o = static_cast<size_t>(qi) * k + rank;
      out_s[o] = static_cast<float>(s); out_ids[o] = me;
      if (out_s64) out_s64[o] = s;
    }
  }
  atomicAdd(&s_nvalid, local_valid);
  __syncthreads();
  for (int t = s_nvalid + threadIdx.x; t < k; t += blockDim.x) {
    const size_t o = static_cast<size_t>(qi) * k + t;
    out_s[o] = -INFINITY; out_ids[o] = -1;
    if (out_s64) out_s64[o] = -INFINITY;
  }
}

// Fused exchange, receiving side.  Every rank's finalize kernels store their (fp64 score, id) rows into slot
// [parity][rank] of EVERY rank's buffer as tagged 8-byte words (see FinalizeArgs::ExchangeOut).  This kernel, next in
// the stream, has block q poll query q's world x k entries until all four words of each carry this exchange's tag,
// then merges them by (score desc, id asc); the last block to finish bumps the sequence word, so a replayed CUDA graph
// advances by itself.  Two parities: rank A can only write exchange s+2 after its own merge s+1, which waited for B's
// rows of s+1, which B produced after finishing its merge s -- so a slot is never overwritten while someone reads it.
__device__ __forceinline__ uint64_t ld_relaxed_sys(const uint64_t* p) {
  uint64_t v; asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory"); return v;
}

__global__ void __launch_bounds__(256)
exchange_merge_kernel(ExchangeParams p) {
  extern __shared__ uint8_t sm[];
  double* sc = reinterpret_cast<double*>(sm);
  int64_t* id = reinterpret_cast<int64_t*>(sc + p.world * p.k);
  __shared__ int s_nvalid;
  const uint64_t seq = *p.seq + 1;
  const uint32_t tag = static_cast<uint32_t>(seq);
  const uint64_t* base = p.slots + (seq & 1ull) * p.parity_stride;
  const int qi = blockIdx.x, n = p.world * p.k;
  if (threadIdx.x == 0) s_nvalid = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int sh = i / p.k, t = i % p.k;
    const uint64_t* e = base + static_cast<size_t>(sh) * p.slot_stride + (static_cast<size_t>(qi) * p.k + t) * 4;
    uint64_t w0, w1, w2, w3;
    const long long t0 = clock64();
    for (;;) {
      w0 = ld_relaxed_sys(e); w1 = ld_relaxed_sys(e + 1); w2 = ld_relaxed_sys(e + 2); w3 = ld_relaxed_sys(e + 3);
      if (static_cast<uint32_t>(w0 >> 32) == tag && static_cast<uint32_t>(w1 >> 32) == tag &&
          static_cast<uint32_t>(w2 >> 32) == tag && static_cast<uint32_t>(w3 >> 32) == tag) break;
      if (clock64() - t0 > 4000000000ll) { atomicExch(p.status, 1u + sh); w0 = w1 = 0; w2 = w3 = 0xFFFFFFFFull; break; }   // ~2 s: a peer died
      __nanosleep(20);
    }
    sc[i] = __longlong_as_double(static_cast<long long>((w1 << 32) | (w0 & 0xFFFFFFFFull)));
    id[i] = static_cast<int64_t>((w3 << 32) | (w2 & 0xFFFFFFFFull));
  }
  __syncthreads();
  int local_valid = 0;
  for (int t = threadIdx.x; t < n; t += blockDim.x) {
    const double s = sc[t]; const int64_t me = id[t];
    if (me < 0) continue;
    ++local_valid;
    int rank = 0;
    for (int u = 0; u < n; ++u) {
      const double su = sc[u]; const int64_t iu = id[u];
      if (iu >= 0 && (su > s || (su == s && iu < me))) ++rank;
    }
    if (rank < p.k) {
      const size_t o = static_cast<size_t>(qi) * p.k + rank;
      p.out_scores[o] = static_cast<float>(s); p.out_ids[o] = me;
    }
  }
  atomicAdd(&s_nvalid, local_valid);
  __syncthreads();
  for (int t = s_nvalid + threadIdx.x; t < p.k; t += blockDim.x) {
    const size_t o = static_cast<size_t>(qi) * p.k + t;
    p.out_scores[o] = -INFINITY; p.out_ids[o] = -1;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(p.done, 1u) == gridDim.x - 1) { *p.done = 0; __threadfence(); *p.seq = seq; }
  }
}

// Cosine of x and y [dim] by one warp, fp64 accumulate, optional [0,1] clamp (similarity.py:84-98); lane 0 writes
// out[pair].  The one statement of this arithmetic: cosine_pairs_kernel and cosine_gather_kernel agree bit for bit
// through it.
__device__ __forceinline__ void cosine_pair_warp(const float* __restrict__ x, const float* __restrict__ y, int dim,
                                                 int clamp, int lane, double* __restrict__ out, int64_t pair) {
  double dot = 0.0, xx = 0.0, yy = 0.0;
  for (int i = lane; i < dim; i += 32) {
    const double u = x[i], v = y[i];
    dot = fma(u, v, dot); xx = fma(u, u, xx); yy = fma(v, v, yy);
  }
  dot = warp_sum_lane0(dot); xx = warp_sum_lane0(xx); yy = warp_sum_lane0(yy);
  if (lane == 0) {
    const double den = sqrt(xx) * sqrt(yy);
    double c = (dim > 0 && den > 0.0) ? dot / den : 0.0;
    if (clamp) c = fmax(0.0, fmin(1.0, c));
    out[pair] = c;
  }
}

// Pairwise cosine of row i of a with row i of b.
__global__ void cosine_pairs_kernel(const float* __restrict__ a, const float* __restrict__ b, int64_t n, int dim,
                                    int clamp, double* __restrict__ out) {
  const int64_t pair = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (pair >= n) return;
  cosine_pair_warp(a + pair * dim, b + pair * dim, dim, clamp, lane, out, pair);
}

// Pair p = rows pa[p] and pb[p] of vecs [*, dim], one warp each (aur_encode_pair_cosines).
__global__ void cosine_gather_kernel(const float* __restrict__ vecs, const int32_t* __restrict__ pa,
                                     const int32_t* __restrict__ pb, int64_t n, int dim, int clamp,
                                     double* __restrict__ out) {
  const int64_t pair = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (pair >= n) return;
  cosine_pair_warp(vecs + static_cast<int64_t>(pa[pair]) * dim, vecs + static_cast<int64_t>(pb[pair]) * dim, dim, clamp,
                   lane, out, pair);
}

__global__ void fill_f32_kernel(float* p, float v, int64_t n) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

}  // namespace

cudaError_t launch_row_inv_norms(const void* rows, int dtype, int dim, int64_t n, float* inv_norm, cudaStream_t s) {
  if (n <= 0) return cudaSuccess;
  const int threads = 256;
  const int64_t blocks = (n * 32 + threads - 1) / threads;
  if (dtype == 2) return cudaErrorInvalidValue;   // int8 rows get their scale from launch_quantize_rows_i8
  if (dtype == 0)
    row_inv_norm_kernel<__nv_bfloat16><<<static_cast<unsigned>(blocks), threads, 0, s>>>(
        static_cast<const __nv_bfloat16*>(rows), dim, n, inv_norm);
  else
    row_inv_norm_kernel<float><<<static_cast<unsigned>(blocks), threads, 0, s>>>(static_cast<const float*>(rows), dim, n,
                                                                               inv_norm);
  return cudaGetLastError();
}

cudaError_t launch_query_image_i8(const __nv_bfloat16* q, int dim, int nq, int8_t* out, cudaStream_t s) {
  if (nq <= 0) return cudaSuccess;
  const int64_t blocks = (static_cast<int64_t>(nq) * 32 + 255) / 256;
  query_image_i8_kernel<<<static_cast<unsigned>(blocks), 256, 0, s>>>(q, dim, nq, out);
  return cudaGetLastError();
}

cudaError_t launch_quantize_rows_i8(const __nv_bfloat16* in, int dim, int64_t n, int8_t* out, float* inv_norm, cudaStream_t s) {
  if (n <= 0) return cudaSuccess;
  const int64_t blocks = (n * 32 + 255) / 256;
  quantize_rows_i8_kernel<<<static_cast<unsigned>(blocks), 256, 0, s>>>(in, dim, n, out, inv_norm);
  return cudaGetLastError();
}

cudaError_t launch_simt_scores(const void* q, const void* rows, int dtype, int dim, int nq, int64_t row0,
                               int64_t nrows_chunk, int64_t n_rows, const float* inv_norm, FilterArgs f, float* scores,
                               cudaStream_t s) {
  dim3 grid(static_cast<unsigned>((nrows_chunk + kSB - 1) / kSB), static_cast<unsigned>((nq + kSB - 1) / kSB));
  if (dtype == 2)
    simt_scores_kernel<__nv_bfloat16, int8_t><<<grid, 256, 0, s>>>(static_cast<const __nv_bfloat16*>(q),
                                                                  static_cast<const int8_t*>(rows), dim, nq, row0,
                                                                  nrows_chunk, n_rows, inv_norm, f, scores);
  else if (dtype == 0)
    simt_scores_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(static_cast<const __nv_bfloat16*>(q),
                                                          static_cast<const __nv_bfloat16*>(rows), dim, nq, row0,
                                                          nrows_chunk, n_rows, inv_norm, f, scores);
  else
    simt_scores_kernel<float><<<grid, 256, 0, s>>>(static_cast<const float*>(q), static_cast<const float*>(rows), dim, nq,
                                                  row0, nrows_chunk, n_rows, inv_norm, f, scores);
  return cudaGetLastError();
}

cudaError_t launch_simt_select(const float* scores, int nq, int64_t row0, int64_t nrows_chunk, int ksel, const int64_t* ids,
                               uint64_t* cand, int n_lists, int list0, cudaStream_t s) {
  dim3 grid(static_cast<unsigned>((nrows_chunk + kSimtSeg - 1) / kSimtSeg), static_cast<unsigned>(nq));
  simt_select_kernel<<<grid, 256, 0, s>>>(scores, row0, nrows_chunk, ksel, ids, cand, n_lists, list0);
  return cudaGetLastError();
}

cudaError_t launch_reduce_lists(const uint64_t* in, int nq, int n_lists, int ksel, int group, const int64_t* ids,
                                uint64_t* out, cudaStream_t s) {
  const int n_groups = (n_lists + group - 1) / group;
  int P = 64; while (P < group * ksel) P <<= 1;
  dim3 grid(static_cast<unsigned>(n_groups), static_cast<unsigned>(nq));
  reduce_lists_kernel<<<grid, 512, static_cast<size_t>(P) * 8, s>>>(in, n_lists, ksel, group, ids, out, n_groups);
  return cudaGetLastError();
}

cudaError_t launch_finalize(const FinalizeArgs& a_in, cudaStream_t s) {
  FinalizeArgs a = a_in;
  int P = 64; while (P < a.n_lists * a.ksel) P <<= 1;
  if (P > kSortCap) {
    if (!a.counts) return cudaErrorInvalidValue;   // dense rows must be folded first
    P = kSortCap;
  }
  a.sort_cap = P;
  const size_t smem = static_cast<size_t>(P) * 8 + static_cast<size_t>(a.dim) * 4;
  if (smem > 48 * 1024) {
    // raised only: concurrent searches on one device ask for different sizes (raise_smem_limit)
    cudaError_t e = raise_smem_limit(a.dtype == 0 ? (const void*)finalize_kernel<__nv_bfloat16>
                                     : a.dtype == 2 ? (const void*)finalize_kernel<__nv_bfloat16, int8_t>
                                                    : (const void*)finalize_kernel<float>, smem);
    if (e != cudaSuccess) return e;
  }
  // programmatic dependent launch: blocks start (query -> shared memory, |q|^2) while the similarity kernel drains
  if (a.dtype == 0) return launch_pdl(finalize_kernel<__nv_bfloat16>, dim3(a.nq), dim3(256), smem, s, 1, a);
  if (a.dtype == 2) return launch_pdl(finalize_kernel<__nv_bfloat16, int8_t>, dim3(a.nq), dim3(256), smem, s, 1, a);
  return launch_pdl(finalize_kernel<float>, dim3(a.nq), dim3(256), smem, s, 1, a);
}

cudaError_t launch_merge_topk(const double* in_s, const int64_t* in_ids, size_t shard_stride, int n_shards, int nq, int k,
                              float* out_s, int64_t* out_ids, double* out_s64, cudaStream_t s) {
  const size_t smem = static_cast<size_t>(n_shards) * k * 16;
  if (smem > 48 * 1024) return cudaErrorInvalidValue;
  merge_topk_kernel<<<nq, 256, smem, s>>>(in_s, in_ids, shard_stride, n_shards, nq, k, out_s, out_ids, out_s64);
  return cudaGetLastError();
}

cudaError_t launch_exchange_merge(const ExchangeParams& p, cudaStream_t s) {
  const size_t smem = static_cast<size_t>(p.world) * p.k * 16;
  if (smem > 48 * 1024 || p.world > 8) return cudaErrorInvalidValue;
  exchange_merge_kernel<<<p.nq, 256, smem, s>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_cosine_pairs(const float* a, const float* b, int64_t n, int dim, int clamp, double* out,
                                cudaStream_t s) {
  if (n <= 0) return cudaSuccess;
  const int threads = 256;
  const int64_t blocks = (n * 32 + threads - 1) / threads;
  cosine_pairs_kernel<<<static_cast<unsigned>(blocks), threads, 0, s>>>(a, b, n, dim, clamp, out);
  return cudaGetLastError();
}

cudaError_t launch_cosine_gather(const float* vecs, const int32_t* pa, const int32_t* pb, int64_t n, int dim, int clamp,
                                 double* out, cudaStream_t s) {
  if (n <= 0) return cudaSuccess;
  const int threads = 256;
  const int64_t blocks = (n * 32 + threads - 1) / threads;
  cosine_gather_kernel<<<static_cast<unsigned>(blocks), threads, 0, s>>>(vecs, pa, pb, n, dim, clamp, out);
  return cudaGetLastError();
}

// Tenant scope folded into the row scale: rows the (user, org) pair may not see get NaN, which the
// tensor-core kernel treats exactly like a tombstone (never admitted, never published).  Same predicate
// as simt_scores_kernel: row_user == u OR (o >= 0 AND row_org == o)  (weaviate_client.py:244-249).
__global__ void mask_inv_norm_kernel(const float* __restrict__ inv, const int32_t* __restrict__ row_user,
                                     const int32_t* __restrict__ row_org, int32_t u, int32_t o, int64_t n,
                                     float* __restrict__ out) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const bool ok = (row_user[i] == u) || (o >= 0 && row_org[i] == o);
  out[i] = ok ? inv[i] : __uint_as_float(0x7FC00000u);
}

cudaError_t launch_mask_inv_norm(const float* inv, const int32_t* row_user, const int32_t* row_org, int32_t u, int32_t o,
                                 int64_t n, float* out, cudaStream_t s) {
  if (n <= 0) return cudaSuccess;
  mask_inv_norm_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(inv, row_user, row_org, u, o, n, out);
  return cudaGetLastError();
}

// Subset search: out was filled with NaN; the listed rows get their inverse norm back (a tombstone stays NaN).
__global__ void scatter_inv_norm_kernel(const float* __restrict__ inv, const int32_t* __restrict__ rows, int64_t n, int64_t n_rows,
                                        float* __restrict__ out) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int32_t r = rows[i];
  if (r >= 0 && r < n_rows) out[r] = inv[r];
}

cudaError_t launch_scatter_inv_norm(const float* inv, const int32_t* rows, int64_t n, int64_t n_rows, float* out, cudaStream_t s) {
  if (n <= 0) return cudaSuccess;
  scatter_inv_norm_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(inv, rows, n, n_rows, out);
  return cudaGetLastError();
}

// Deletes: the listed rows become tombstones (NaN inverse norm, or NaN scale on an int8 shard), one thread per row.
__global__ void tombstone_rows_kernel(const int32_t* __restrict__ rows, int64_t n, float* __restrict__ inv) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) inv[rows[i]] = __uint_as_float(0x7FC00000u);
}

cudaError_t launch_tombstone_rows(const int32_t* rows, int64_t n, float* inv, cudaStream_t s) {
  if (n <= 0) return cudaSuccess;
  tombstone_rows_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(rows, n, inv);
  return cudaGetLastError();
}

// Checkpoints: liveness of rows [0, n) packed 32 to a word, one warp per word.  A row is live when its inverse norm is
// not NaN; on an int8 shard an infinite one (a row stored from a NaN or inf) is also set in nonfinite, as aur_export
// reports it live = 2.  Lanes past n vote 0, so the last word's tail bits are clear.
__global__ void live_bits_kernel(const float* __restrict__ inv, int64_t n, int i8, uint32_t* __restrict__ live,
                                 uint32_t* __restrict__ nonfinite) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const float v = i < n ? __ldg(inv + i) : __uint_as_float(0x7FC00000u);
  const uint32_t l = __ballot_sync(0xFFFFFFFFu, v == v);
  const uint32_t f = __ballot_sync(0xFFFFFFFFu, i8 && isinf(v));
  if ((threadIdx.x & 31) == 0 && i < n) {
    live[i >> 5] = l;
    nonfinite[i >> 5] = f;
  }
}

cudaError_t launch_live_bits(const float* inv, int64_t n, int i8, uint32_t* live, uint32_t* nonfinite, cudaStream_t s) {
  if (n <= 0) return cudaSuccess;
  live_bits_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(inv, n, i8, live, nonfinite);
  return cudaGetLastError();
}

// Compaction: gather the rows listed in map (and their side arrays) into bounce buffers.  One warp per row,
// 16-byte pieces (row_bytes % 16 == 0 for bf16 dims % 8 == 0 and for f32 dims % 4 == 0; else byte loop).
__global__ void gather_rows_kernel(const uint8_t* __restrict__ rows, const float* __restrict__ inv, const int64_t* __restrict__ ids,
                                   const int32_t* __restrict__ user, const int32_t* __restrict__ org, const int32_t* __restrict__ map,
                                   int64_t n, int row_bytes, uint8_t* __restrict__ o_rows, float* __restrict__ o_inv,
                                   int64_t* __restrict__ o_ids, int32_t* __restrict__ o_user, int32_t* __restrict__ o_org) {
  const int64_t j = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (j >= n) return;
  const int64_t r = map[j];
  const uint8_t* src = rows + r * row_bytes;
  uint8_t* dst = o_rows + j * row_bytes;
  if ((row_bytes & 15) == 0) {
    for (int i = lane; i < row_bytes / 16; i += 32) reinterpret_cast<uint4*>(dst)[i] = __ldg(reinterpret_cast<const uint4*>(src) + i);
  } else {
    for (int i = lane; i < row_bytes; i += 32) dst[i] = src[i];
  }
  if (lane == 0) { o_inv[j] = inv[r]; o_ids[j] = ids[r]; o_user[j] = user[r]; o_org[j] = org[r]; }
}

cudaError_t launch_gather_rows(const void* rows, const float* inv, const int64_t* ids, const int32_t* user, const int32_t* org,
                               const int32_t* map, int64_t n, int row_bytes, void* o_rows, float* o_inv, int64_t* o_ids,
                               int32_t* o_user, int32_t* o_org, cudaStream_t s) {
  if (n <= 0) return cudaSuccess;
  const int64_t blocks = (n * 32 + 255) / 256;
  gather_rows_kernel<<<static_cast<unsigned>(blocks), 256, 0, s>>>(static_cast<const uint8_t*>(rows), inv, ids, user, org, map, n,
                                                                  row_bytes, static_cast<uint8_t*>(o_rows), o_inv, o_ids, o_user, o_org);
  return cudaGetLastError();
}

// Per-query tenant scopes on the tensor-core path: one bit per distinct scope of the batch (<= 32) and corpus row.
// Same predicate as simt_scores_kernel: row_user == u OR (o >= 0 AND row_org == o)  (weaviate_client.py:244-249).
__global__ void row_scope_mask_kernel(const int32_t* __restrict__ row_user, const int32_t* __restrict__ row_org,
                                      const int32_t* __restrict__ scopes, int n_scopes, int64_t n, uint32_t* __restrict__ out) {
  __shared__ int32_t su[32], so[32];
  if (threadIdx.x < n_scopes) { su[threadIdx.x] = scopes[2 * threadIdx.x]; so[threadIdx.x] = scopes[2 * threadIdx.x + 1]; }
  __syncthreads();
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int32_t u = row_user[i], o = row_org[i];
  uint32_t m = 0u;
  for (int s = 0; s < n_scopes; ++s) m |= static_cast<uint32_t>((u == su[s]) || (so[s] >= 0 && o == so[s])) << s;
  out[i] = m;
}

cudaError_t launch_row_scope_mask(const int32_t* row_user, const int32_t* row_org, const int32_t* scopes, int n_scopes, int64_t n,
                                  uint32_t* out, cudaStream_t s) {
  if (n <= 0) return cudaSuccess;
  row_scope_mask_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(row_user, row_org, scopes, n_scopes, n, out);
  return cudaGetLastError();
}

cudaError_t launch_fill_f32(float* p, float v, int64_t n, cudaStream_t s) {
  if (n <= 0) return cudaSuccess;
  fill_f32_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(p, v, n);
  return cudaGetLastError();
}

}  // namespace aur
