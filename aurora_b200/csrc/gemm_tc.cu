// Encoder GEMM on wgmma:  out[M, N] = act( A[M, K] . W[N, K]^T + bias ) (+ residual), bf16 in,
// fp32 accumulate in registers, bf16 out.  Both operands are K-major (activations [tokens, K] and
// torch-Linear weights [N, K]), so one {64 x rows} SWIZZLE_128B TMA box feeds either side.
//
// Persistent kernel, one CTA per SM, (128*kCtaGroup) x BN output tiles handed out round-robin:
//   warpgroup 0   TMA producer (one thread; A 16 KB + W BN*128 B per 64-wide k-block, kStages ring)
//   warpgroups 1-2 consumers: each owns 64 rows of the 128-row tile, wgmma m64 x BN x k16 (4 per k-block) into
//                 registers, then bias / GELU / residual fused and bf16 pairs stored straight to the output
//                 while the producer already streams the next tile's k-blocks
// Two-CTA clusters (cta_group 2): one 256 x BN tile per pair, each CTA loads its own 128 rows of A and HALF of
// the weight tile, multicast to both CTAs -- the weight tile crosses L2 -> SM once per pair.
// SURVEY.md section 8 a11 (BERT-family encoder forward); structural oracle: oracle/bert_encoder.py.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "internal.h"
#include "ptx.cuh"

namespace aur {
namespace {

using namespace ptx;

constexpr int kBM = 128, kBK = 64, kGemmThreads = 3 * 128;

__device__ __forceinline__ float rcp_approx(float x) {
  float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y;
}
__device__ __forceinline__ float ex2_approx(float x) {
  float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y;
}
__device__ __forceinline__ float gelu_erf(float x) {
  const float z = fabsf(x) * 0.70710678118654752f;
  const float t = rcp_approx(fmaf(0.3275911f, z, 1.0f));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  const float e = ex2_approx(z * -1.4426950408889634f * z);
  const float erf_abs = fmaf(-poly * t, e, 1.0f);
  const float h = 0.5f * x;
  return fmaf(h, copysignf(erf_abs, x), h);
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  uint32_t d;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
  return d;
}

template <int BN>
struct GemmSmem {
  static constexpr int kABytes = kBM * kBK * 2;          // 16 KB: this CTA's 128 rows of A
  static constexpr int kBBytes = BN * kBK * 2;           // the whole weight tile (half of it from the peer when paired)
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = (192 * 1024) / kStageBytes > 8 ? 8 : (192 * 1024) / kStageBytes;
  static constexpr int kBarBytes = 256;
  static constexpr size_t kTotal = 1024 + static_cast<size_t>(kStages) * kStageBytes + kBarBytes;
};

template <int BN> struct Acc;
template <> struct Acc<128> {
  static __device__ __forceinline__ void mma(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) { wgmma_m64n128_ss(d, a, b, acc); }
};
template <> struct Acc<256> {
  static __device__ __forceinline__ void mma(float (&d)[128], uint64_t a, uint64_t b, uint32_t acc) { wgmma_m64n256_ss(d, a, b, acc); }
};

template <int BN, int EPI, int G>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, const GemmParams p) {
  using S = GemmSmem<BN>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (base & 1023u)) & 1023u);
  uint8_t* stage0 = smem;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S::kStages * S::kStageBytes);
  uint64_t* full = bars;                       // [kStages]
  uint64_t* empty = bars + S::kStages;         // [kStages]  both consumer warpgroups of every CTA the stage reaches

  const int wg = threadIdx.x >> 7;
  const uint32_t rank = G == 2 ? cluster_ctarank() : 0u;
  const int group = blockIdx.x / G, n_groups = gridDim.x / G;
  const int n_tiles_total = p.m_tiles * p.n_tiles;   // tiles of (128*G) x BN

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_a); prefetch_tmap(&tmap_b);
    for (int s = 0; s < S::kStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2 * G); }
    fence_mbar_init();
  }
  if constexpr (G == 2) cluster_sync_all(); else __syncthreads();
  grid_dep_launch();   // the next kernel may take over SMs as this grid's CTAs retire
  grid_dep_wait();     // everything above overlapped the previous kernel's tail; its output is needed from here on

  if (wg == 0) {
    // ------------------------------------------------------------ TMA producer
    if (threadIdx.x == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int tile = group; tile < n_tiles_total; tile += n_groups) {
        const int m_blk = tile / p.n_tiles, n_blk = tile % p.n_tiles;
        const int a_row = (m_blk * G + static_cast<int>(rank)) * kBM;
        const int b_row = n_blk * BN + static_cast<int>(rank) * (BN / G);
        for (int kb = 0; kb < p.k_blocks; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          uint8_t* sa = stage0 + stage * S::kStageBytes;
          mbar_arrive_expect_tx(&full[stage], S::kStageBytes);
          tma_load_2d(sa, &tmap_a, &full[stage], kb * kBK, a_row, kEvictNormal);
          if constexpr (G == 1)
            tma_load_2d(sa + S::kABytes, &tmap_b, &full[stage], kb * kBK, b_row, kEvictLast);
          else
            tma_load_2d_mc(sa + S::kABytes + rank * (S::kBBytes / 2), &tmap_b, &full[stage], kb * kBK, b_row, 0x3, kEvictLast);
          if (++stage == S::kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ------------------------------------------------------------ consumers: 64 rows each
    const int t = threadIdx.x - 128 * wg, w = t >> 5, l = t & 31;
    const int half = wg - 1;
    int stage = 0; uint32_t phase = 0;
    for (int tile = group; tile < n_tiles_total; tile += n_groups) {
      const int m_blk = tile / p.n_tiles, n_blk = tile % p.n_tiles;
      float d[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
      for (int kb = 0; kb < p.k_blocks; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint32_t sa = smem_u32(stage0 + stage * S::kStageBytes);
        const uint64_t a_desc = wgmma_desc_sw128(sa + half * 64 * 128), b_desc = wgmma_desc_sw128(sa + S::kABytes);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < kBK / 16; ++ks) Acc<BN>::mma(d, a_desc + 2 * ks, b_desc + 2 * ks, 1u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(d);
        if (t == 0) {
          mbar_arrive(&empty[stage]);
          if constexpr (G == 2) mbar_arrive_cluster(&empty[stage], rank ^ 1u);
        }
        if (++stage == S::kStages) { stage = 0; phase ^= 1; }
      }
      // epilogue: register i of the accumulator = row 16 w + l / 4 (+ 8 for i & 2), column 8 (i / 4) + 2 (l % 4) (+ 1)
      const int row_lo = (m_blk * G + static_cast<int>(rank)) * kBM + half * 64 + 16 * w + (l >> 2);
      const int col_base = n_blk * BN + 2 * (l & 3);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = col_base + 8 * j;
        const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + col));
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int row = row_lo + 8 * hh;
          float x0 = d[4 * j + 2 * hh] + b.x, x1 = d[4 * j + 2 * hh + 1] + b.y;
          if constexpr (EPI == kEpiBiasGelu) { x0 = gelu_erf(x0); x1 = gelu_erf(x1); }
          if constexpr (EPI == kEpiBiasResid) {
            const __nv_bfloat162 r = *reinterpret_cast<const __nv_bfloat162*>(p.resid + static_cast<size_t>(row) * p.ldr + col);
            x0 += __bfloat162float(r.x); x1 += __bfloat162float(r.y);
          }
          *reinterpret_cast<uint32_t*>(p.out + static_cast<size_t>(row) * p.ldo + col) = pack_bf16x2(x0, x1);
        }
      }
    }
  }
  // no CTA of a pair exits while its peer may still multicast into it or arrive on its barriers
  if constexpr (G == 2) cluster_sync_all();
}

template <int BN, int EPI, int G>
cudaError_t launch_one(int sm_count, const void* tmap_a, const void* tmap_b, const GemmParams& p, cudaStream_t s) {
  auto kern = gemm_tc_kernel<BN, EPI, G>;
  static bool attr_set = false;   // per instantiation
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(GemmSmem<BN>::kTotal));
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  const int tiles = p.m_tiles * p.n_tiles, groups = sm_count / G;
  return launch_pdl(kern, dim3(static_cast<unsigned>((tiles < groups ? tiles : groups) * G)), dim3(kGemmThreads),
                    GemmSmem<BN>::kTotal, s, G, *reinterpret_cast<const CUtensorMap*>(tmap_a),
                    *reinterpret_cast<const CUtensorMap*>(tmap_b), p);
}

}  // namespace

// cta_group: 1 = one CTA per 128 x bn tile, 2 = CTA pair per 256 x bn tile (p.m_tiles counts those).
// tmap_b must have a {64, bn / cta_group} box.
cudaError_t gemm_tc_launch(int cta_group, int bn, int epi, int sm_count, const void* tmap_a, const void* tmap_b,
                           const GemmParams& p, cudaStream_t s) {
  if (p.m_tiles * p.n_tiles <= 0) return cudaSuccess;
#define AUR_GEMM_CASE(BN, EPI, G) \
  if (bn == BN && epi == EPI && cta_group == G) return launch_one<BN, EPI, G>(sm_count, tmap_a, tmap_b, p, s)
  AUR_GEMM_CASE(256, kEpiBias, 2); AUR_GEMM_CASE(256, kEpiBiasGelu, 2); AUR_GEMM_CASE(256, kEpiBiasResid, 2);
  AUR_GEMM_CASE(128, kEpiBias, 2); AUR_GEMM_CASE(128, kEpiBiasGelu, 2); AUR_GEMM_CASE(128, kEpiBiasResid, 2);
  AUR_GEMM_CASE(256, kEpiBias, 1); AUR_GEMM_CASE(256, kEpiBiasGelu, 1); AUR_GEMM_CASE(256, kEpiBiasResid, 1);
  AUR_GEMM_CASE(128, kEpiBias, 1); AUR_GEMM_CASE(128, kEpiBiasGelu, 1); AUR_GEMM_CASE(128, kEpiBiasResid, 1);
#undef AUR_GEMM_CASE
  return cudaErrorInvalidValue;
}

}  // namespace aur
