// Encoder self-attention on wgmma: packed variable-length sequences (<= 512 tokens), head dim 64.
//
// One CTA per (work item, head); a work item is 128 queries of one sequence.  Thread 0 issues every TMA load of the
// CTA at once -- the Q tile and, per 128-key block of the sequence, its K and V tiles, each block on its own
// mbarrier -- so the first block's MMAs start while the later blocks are still in flight.  Two warpgroups, 64 query
// rows each, walk the key blocks with an online softmax:
//   S = Q K^T          wgmma m64n128k16 x 4, both operands K-major from shared memory
//   P = exp2(S - m)    in registers (keys past the end of the sequence are masked to -inf, P = 0)
//   O += P V           wgmma m64n64k16 x 8, P straight from registers (the accumulator layout of S is the A-operand
//                      layout), V from shared memory read MN-major
// and store O / rowsum as bf16.  The max is exact (rescale every block); P is rounded to bf16 for the PV MMA.
// Restates eager_attention_forward + softmax of transformers' modeling_bert.py:115-140 (oracle/bert_encoder.py).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "internal.h"
#include "ptx.cuh"

namespace aur {
namespace {

using namespace ptx;

constexpr int kKB = 128, kDh = 64, kMaxKeyBlocks = 4;
constexpr int kTile = 128 * kDh * 2;          // 16 KB: 128 rows x 128 B
constexpr int kThreads = 256;
constexpr size_t kSmemBytes = 1024 + static_cast<size_t>(1 + 2 * kMaxKeyBlocks) * kTile + 128;

__device__ __forceinline__ float ex2_approx(float x) {
  float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y;
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  uint32_t d;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
  return d;
}

__global__ void __launch_bounds__(kThreads, 1)
attn_tc_kernel(const __grid_constant__ CUtensorMap tmap_qkv, const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sQ = smem;
  uint8_t* sK = smem + kTile;                          // [kMaxKeyBlocks] tiles
  uint8_t* sV = smem + (1 + kMaxKeyBlocks) * kTile;    // [kMaxKeyBlocks] tiles
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (1 + 2 * kMaxKeyBlocks) * kTile);   // q_full, kv_full[4]

  const AttnItem item = p.items[blockIdx.x / p.heads];
  const int head = blockIdx.x % p.heads;
  const int n_kb = (item.len + kKB - 1) / kKB;

  grid_dep_launch();
  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_qkv);
    for (int i = 0; i < 1 + kMaxKeyBlocks; ++i) mbar_init(&bars[i], 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    grid_dep_wait();     // the qkv projections come from the previous kernel
    mbar_arrive_expect_tx(&bars[0], kTile);
    tma_load_2d(sQ, &tmap_qkv, &bars[0], head * kDh, item.tok0 + item.q0, kEvictNormal);
    for (int j = 0; j < n_kb; ++j) {
      mbar_arrive_expect_tx(&bars[1 + j], 2 * kTile);
      tma_load_2d(sK + j * kTile, &tmap_qkv, &bars[1 + j], p.hidden + head * kDh, item.tok0 + j * kKB, kEvictNormal);
      tma_load_2d(sV + j * kTile, &tmap_qkv, &bars[1 + j], 2 * p.hidden + head * kDh, item.tok0 + j * kKB, kEvictNormal);
    }
  }

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127, w = t >> 5, l = t & 31;
  // accumulator layout (m64nN): register 4 j + {0, 1} = row 16 w + l / 4, columns 8 j + 2 (l % 4) + {0, 1};
  // 4 j + {2, 3} = the same columns of row + 8
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const float sc = p.scale_log2e;
  const uint64_t q_desc = wgmma_desc_sw128(smem_u32(sQ + wg * 64 * 128));
  mbar_wait(&bars[0], 0);
  for (int j = 0; j < n_kb; ++j) {
    mbar_wait(&bars[1 + j], 0);
    float s[64];
    const uint64_t k_desc = wgmma_desc_sw128(smem_u32(sK + j * kTile));
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < kDh / 16; ++ks) wgmma_m64n128_ss(s, q_desc + 2 * ks, k_desc + 2 * ks, ks > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    // mask, scale to log2 units, running max per row (a row lives in the 4 lanes of a quad)
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 64; ++i) {
      const int key = j * kKB + 8 * (i >> 2) + 2 * (l & 3) + (i & 1);
      const float v = key < item.len ? s[i] * sc : -INFINITY;
      s[i] = v;
      mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], v);
    }
    float alpha[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
      const float m_new = fmaxf(m_run[h], mx[h]);
      alpha[h] = ex2_approx(m_run[h] - m_new);
      m_run[h] = m_new;
      l_run[h] *= alpha[h];
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] *= alpha[(i >> 1) & 1];
    uint32_t pa[8][4];   // P as the A operand of 8 K=16 steps
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
      const int h = (i >> 1) & 1;
      const float p0 = ex2_approx(s[i] - m_run[h]), p1 = ex2_approx(s[i + 1] - m_run[h]);
      l_run[h] += p0 + p1;
      pa[i >> 3][(i >> 1) & 3] = pack_bf16x2(p0, p1);
    }
    const uint64_t v_desc = wgmma_desc_sw128(smem_u32(sV + j * kTile));
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < kKB / 16; ++ks) wgmma_m64n64_rs_tb(o, pa[ks], v_desc + (2048 >> 4) * ks);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
  }
  // normalise and store this thread's two rows
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 1);
    l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 2);
    const int qrow = item.q0 + wg * 64 + 16 * w + (l >> 2) + 8 * h;
    if (qrow >= item.len) continue;
    const float inv = 1.f / l_run[h];
    __nv_bfloat16* dst = p.ctx + static_cast<size_t>(item.tok0 + qrow) * p.ld_ctx + head * kDh + 2 * (l & 3);
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
      *reinterpret_cast<uint32_t*>(dst + 8 * jj) = pack_bf16x2(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
  }
}

}  // namespace

cudaError_t attn_tc_launch(const void* tmap_qkv, const AttnParams& p, cudaStream_t s) {
  if (p.n_items <= 0) return cudaSuccess;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(attn_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kSmemBytes));
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  return launch_pdl(attn_tc_kernel, dim3(static_cast<unsigned>(p.n_items * p.heads)), dim3(kThreads), kSmemBytes, s, 1,
                    *reinterpret_cast<const CUtensorMap*>(tmap_qkv), p);
}

}  // namespace aur
