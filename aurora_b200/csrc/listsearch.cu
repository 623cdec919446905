// Per-query pre-filter lists (aur_search_lists): similarity of each query against only the rows its list names.
//
// One work item = (list, group of <= kListQMax queries naming it, segment of <= kSimtSeg of the list's rows).  Two
// kernels per batch of items:
//   list_scores_kernel  one CTA per 64-row tile of a segment gathers the tile's rows (cp.async, 16 B per thread and
//                       piece, row by row) into a shared-memory ring together with the matching k-chunk of the group's
//                       queries, and scores them on tensor cores (mma.sync m16n8k16, bf16 -> fp32), times inv_norm[row]
//                       (NaN = invisible);
//   list_select_kernel  keeps the best ksel = k + slack keys of every (query, segment) in key_before order, into the
//                       dense candidate rows [nq, n_lists, ksel] that launch_reduce_lists / launch_finalize take.
// The scores of a segment (64 queries x 2048 rows x 4 B = 512 KB) do not fit in shared memory, so they pass through a
// global scratch between the two kernels; it is 8 B per (query, listed row) against the 2 * dim B per listed row the
// gather reads once per query group.
#include <math.h>
#include "internal.h"
#include "ptx.cuh"

namespace aur {
namespace {

constexpr int kLTile = 64;                 // listed rows per MMA tile
constexpr int kLKc = 64;                   // bf16 of a row per k-chunk (128 B)
constexpr int kLPitch = kLKc + 8;          // smem row pitch in bf16 (144 B): the 8 rows an ldmatrix reads sit in 8
                                           // different 16-byte bank groups
constexpr int kLStages = 4;                // ring depth: 3 k-chunks of rows in flight while one is multiplied
constexpr int kLThreads = 128;             // 4 MMA warps, 16 listed rows of the tile each
constexpr int kLStageElems = (kListQMax + kLTile) * kLPitch;   // queries [0, 64), rows [64, 128) of a stage
constexpr size_t kLSmem = static_cast<size_t>(kLStages) * kLStageElems * 2;

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int src_bytes) {
  // src_bytes 0 zero-fills the 16 bytes (k beyond dim, rows beyond the segment, unused query rows)
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// One CTA per (item, 64-row tile of its segment): the tile's k-chunks stream through the ring, so a short list is
// spread over many SMs instead of being one CTA's chain of dependent loads.
__global__ void __launch_bounds__(kLThreads) list_scores_kernel(ListParams p) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __nv_bfloat16* ring = reinterpret_cast<__nv_bfloat16*>(smem_raw);
  __shared__ int32_t s_rows[kLTile];
  __shared__ int32_t s_q[kListQMax];
  const ListItem it = p.items[blockIdx.x];
  const int j0 = blockIdx.y * kLTile;                    // first row of the tile inside the segment
  const int t_rows = min(kLTile, it.n_rows - j0);
  if (t_rows <= 0) return;
  for (int i = threadIdx.x; i < t_rows; i += kLThreads) s_rows[i] = p.list_rows[it.row0 + j0 + i];
  for (int i = threadIdx.x; i < it.nq; i += kLThreads) s_q[i] = p.qidx[it.q0 + i];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_tiles = (it.nq + 15) >> 4;     // 16-query MMA row blocks in use
  const int qrows = m_tiles * 16;
  const int n_kc = (p.dim + kLKc - 1) / kLKc;

  auto load = [&](int kc) {
    if (kc < n_kc) {
      const int k0 = kc * kLKc;
      const uint32_t base = ptx::smem_u32(ring + (kc % kLStages) * kLStageElems);
      const int pieces = (qrows + t_rows) * (kLKc / 8);
      for (int i = threadIdx.x; i < pieces; i += kLThreads) {
        const int r = i >> 3, k = k0 + (i & 7) * 8;
        const __nv_bfloat16* src = p.q;   // a valid address even when nothing is read
        int bytes = 0, dst_row = r;
        if (r < qrows) {
          if (r < it.nq && k < p.dim) { src = p.q + static_cast<size_t>(s_q[r]) * p.dim + k; bytes = 16; }
        } else {
          dst_row = kListQMax + (r - qrows);
          if (k < p.dim) { src = p.rows + static_cast<size_t>(s_rows[r - qrows]) * p.dim + k; bytes = 16; }
        }
        cp_async16(base + (dst_row * kLPitch + (i & 7) * 8) * 2, src, bytes);
      }
    }
    cp_async_commit();   // one group per k-chunk, empty past the end: the wait below counts groups
  };

  float acc[4][2][4];
#pragma unroll
  for (int m = 0; m < 4; ++m)
#pragma unroll
    for (int f = 0; f < 2; ++f)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[m][f][c] = 0.f;

#pragma unroll
  for (int s = 0; s < kLStages - 1; ++s) load(s);
  for (int kc = 0; kc < n_kc; ++kc) {
    cp_async_wait<kLStages - 2>();
    __syncthreads();                       // chunk kc landed for every thread; kc - 1's stage is free
    load(kc + kLStages - 1);
    const __nv_bfloat16* st = ring + (kc % kLStages) * kLStageElems;
    const uint32_t sq = ptx::smem_u32(st), sr = ptx::smem_u32(st + kListQMax * kLPitch);
    // rows of the tile past t_rows hold stale data of an earlier chunk: their scores are never stored
#pragma unroll
    for (int kk = 0; kk < kLKc; kk += 16) {
      uint32_t b[4];   // rows warp*16 + 0..7 (k lo, k hi), rows + 8..15 (k lo, k hi)
      const int bn = warp * 16 + (lane & 7) + ((lane >> 4) << 3), bk = kk + (((lane >> 3) & 1) << 3);
      ldmatrix_x4(b, sr + (bn * kLPitch + bk) * 2);
#pragma unroll
      for (int m = 0; m < 4; ++m) {
        if (m < m_tiles) {
          uint32_t a[4];
          const int am = m * 16 + (lane & 7) + (((lane >> 3) & 1) << 3), ak = kk + ((lane >> 4) << 3);
          ldmatrix_x4(a, sq + (am * kLPitch + ak) * 2);
          mma_16816(acc[m][0], a, b[0], b[1]);
          mma_16816(acc[m][1], a, b[2], b[3]);
        }
      }
    }
  }
  cp_async_wait<0>();
#pragma unroll
  for (int f = 0; f < 2; ++f)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int j = warp * 16 + f * 8 + (lane & 3) * 2 + e;
      const float nv = j < t_rows ? __ldg(p.inv_norm + s_rows[j]) : 0.f;
#pragma unroll
      for (int m = 0; m < 4; ++m)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int qr = m * 16 + (lane >> 2) + h * 8;
          if (m < m_tiles && qr < it.nq && j < t_rows)
            p.scores[static_cast<size_t>(it.out + qr) * kSimtSeg + j0 + j] = acc[m][f][h * 2 + e] * nv;
        }
    }
}

// One block per (item, query of the item): the segment's keys sorted by key_before, the first ksel kept.
__global__ void __launch_bounds__(256) list_select_kernel(ListParams p) {
  __shared__ uint64_t keys[kSimtSeg];
  const ListItem it = p.items[blockIdx.x];
  const int g = blockIdx.y;
  if (g >= it.nq) return;
  const float* sc = p.scores + static_cast<size_t>(it.out + g) * kSimtSeg;
  int P = 64;
  while (P < it.n_rows) P <<= 1;
  for (int i = threadIdx.x; i < kSimtSeg; i += blockDim.x) {
    uint64_t key = 0;   // 0 sorts below every real key and is read as empty downstream
    if (i < it.n_rows) {
      const float s = sc[i];
      if (!(s == -INFINITY || s != s)) key = make_key(s, p.list_rows[it.row0 + i]);
    }
    keys[i] = key;
  }
  __syncthreads();
  for (int k = 2; k <= P; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < P; i += blockDim.x) {
        const int l = i ^ j;
        if (l > i) {
          const uint64_t a = keys[i], b = keys[l];
          const bool desc = (i & k) == 0;
          if (desc ? key_before(b, a, p.ids) : key_before(a, b, p.ids)) { keys[i] = b; keys[l] = a; }
        }
      }
      __syncthreads();
    }
  const int qb = p.qidx[it.q0 + g];
  uint64_t* out = p.cand + (static_cast<size_t>(qb) * p.n_lists + it.seg) * p.ksel;
  for (int t = threadIdx.x; t < p.ksel; t += blockDim.x) out[t] = keys[t] == 0 ? kKeyEmpty : keys[t];
}

}  // namespace

cudaError_t launch_list_search(const ListParams& p, int max_nq, cudaStream_t s) {
  if (p.n_items <= 0) return cudaSuccess;
  cudaError_t e = cudaFuncSetAttribute(list_scores_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kLSmem));
  if (e != cudaSuccess) return e;
  list_scores_kernel<<<dim3(p.n_items, kSimtSeg / kLTile), kLThreads, kLSmem, s>>>(p);
  list_select_kernel<<<dim3(p.n_items, max_nq), 256, 0, s>>>(p);
  return cudaGetLastError();
}

}  // namespace aur
