// CUDA-core kernels of the encoder forward: the HBM-bound row operations around the wgmma GEMMs
// and attention.  One warp owns one token row (hidden <= 1024 lives in registers: hidden/8 16-byte
// chunks striped over the lanes), LayerNorm statistics by warp shuffle in fp32 with the two-pass
// variance torch.nn.LayerNorm uses (oracle/bert_encoder.py:layer_norm).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "internal.h"
#include "ptx.cuh"

namespace aur {
namespace {

constexpr int kMaxChunksPerLane = 4;   // hidden <= 8 * 32 * 4 = 1024

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    f[2 * i] = __uint_as_float(w[i] << 16);
    f[2 * i + 1] = __uint_as_float(w[i] & 0xFFFF0000u);
  }
}
__device__ __forceinline__ uint32_t pack2(float lo, float hi) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&h);
}

// Normalise the row held in x[][] (n_chunks chunks per lane) and store it as bf16.
__device__ __forceinline__ void ln_store(float (&x)[kMaxChunksPerLane][8], int lane, int chunks, int hidden,
                                         const float* __restrict__ g, const float* __restrict__ b, float eps,
                                         __nv_bfloat16* __restrict__ out_row) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < kMaxChunksPerLane; ++i)
    if (lane + 32 * i < chunks)
#pragma unroll
      for (int e = 0; e < 8; ++e) s += x[i][e];
  const float mean = warp_sum(s) / hidden;
  float v = 0.f;
#pragma unroll
  for (int i = 0; i < kMaxChunksPerLane; ++i)
    if (lane + 32 * i < chunks)
#pragma unroll
      for (int e = 0; e < 8; ++e) { const float d = x[i][e] - mean; v += d * d; }
  const float rstd = rsqrtf(warp_sum(v) / hidden + eps);
#pragma unroll
  for (int i = 0; i < kMaxChunksPerLane; ++i) {
    const int ch = lane + 32 * i;
    if (ch < chunks) {
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(g) + 2 * ch), g1 = __ldg(reinterpret_cast<const float4*>(g) + 2 * ch + 1);
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(b) + 2 * ch), b1 = __ldg(reinterpret_cast<const float4*>(b) + 2 * ch + 1);
      const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
      float y[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) y[e] = (x[i][e] - mean) * rstd * gg[e] + bb[e];
      reinterpret_cast<uint4*>(out_row)[ch] = make_uint4(pack2(y[0], y[1]), pack2(y[2], y[3]), pack2(y[4], y[5]), pack2(y[6], y[7]));
    }
  }
}

// BertEmbeddings: word + position + token_type(0), LayerNorm (modeling_bert.py:72-112).
// Rows [n_tok, n_rows_pad) are zero-filled so the padded GEMM tiles read defined values.
__global__ void __launch_bounds__(256)
embed_ln_kernel(const int32_t* __restrict__ tok, const int32_t* __restrict__ pos, int n_tok, int n_rows_pad,
                const __nv_bfloat16* __restrict__ word, const __nv_bfloat16* __restrict__ pos_emb,
                const __nv_bfloat16* __restrict__ type_emb, const float* __restrict__ g, const float* __restrict__ b,
                float eps, int hidden, __nv_bfloat16* __restrict__ out) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  ptx::grid_dep_launch();
  ptx::grid_dep_wait();   // the previous forward may still be reading x
  if (row >= n_rows_pad) return;
  const int chunks = hidden >> 3;
  __nv_bfloat16* orow = out + static_cast<size_t>(row) * hidden;
  if (row >= n_tok) {
    for (int ch = lane; ch < chunks; ch += 32) reinterpret_cast<uint4*>(orow)[ch] = make_uint4(0, 0, 0, 0);
    return;
  }
  const uint4* wrow = reinterpret_cast<const uint4*>(word + static_cast<size_t>(__ldg(tok + row)) * hidden);
  const uint4* prow = reinterpret_cast<const uint4*>(pos_emb + static_cast<size_t>(__ldg(pos + row)) * hidden);
  const uint4* trow = reinterpret_cast<const uint4*>(type_emb);
  float x[kMaxChunksPerLane][8];
#pragma unroll
  for (int i = 0; i < kMaxChunksPerLane; ++i) {
    const int ch = lane + 32 * i;
    if (ch < chunks) {
      float a[8], c[8], d[8];
      unpack8(__ldg(wrow + ch), a); unpack8(__ldg(prow + ch), c); unpack8(__ldg(trow + ch), d);
#pragma unroll
      for (int e = 0; e < 8; ++e) x[i][e] = a[e] + d[e] + c[e];
    }
  }
  ln_store(x, lane, chunks, hidden, g, b, eps, orow);
}

// Two rows per warp: both rows' loads are in flight before any arithmetic starts.
__global__ void __launch_bounds__(256)
layernorm_kernel(const __nv_bfloat16* __restrict__ in, const float* __restrict__ g, const float* __restrict__ b,
                 float eps, int n_rows, int hidden, __nv_bfloat16* __restrict__ out) {
  const int row0 = ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 2, lane = threadIdx.x & 31;
  ptx::grid_dep_launch();
  ptx::grid_dep_wait();
  if (row0 >= n_rows) return;
  const bool two = row0 + 1 < n_rows;
  const int chunks = hidden >> 3;
  const uint4* irow0 = reinterpret_cast<const uint4*>(in + static_cast<size_t>(row0) * hidden);
  const uint4* irow1 = irow0 + chunks;
  uint4 raw0[kMaxChunksPerLane], raw1[kMaxChunksPerLane];
#pragma unroll
  for (int i = 0; i < kMaxChunksPerLane; ++i) {
    const int ch = lane + 32 * i;
    if (ch < chunks) { raw0[i] = __ldg(irow0 + ch); if (two) raw1[i] = __ldg(irow1 + ch); }
  }
  float x[kMaxChunksPerLane][8];
#pragma unroll
  for (int i = 0; i < kMaxChunksPerLane; ++i)
    if (lane + 32 * i < chunks) unpack8(raw0[i], x[i]);
  ln_store(x, lane, chunks, hidden, g, b, eps, out + static_cast<size_t>(row0) * hidden);
  if (two) {
#pragma unroll
    for (int i = 0; i < kMaxChunksPerLane; ++i)
      if (lane + 32 * i < chunks) unpack8(raw1[i], x[i]);
    ln_store(x, lane, chunks, hidden, g, b, eps, out + static_cast<size_t>(row0 + 1) * hidden);
  }
}

// Sentence vector per sequence: CLS row or mean over the real tokens, optional L2 normalisation
// (oracle/bert_encoder.py:pool).  One block per sequence, one thread per pair of dims.
__global__ void __launch_bounds__(512)
pool_kernel(const __nv_bfloat16* __restrict__ x, const int32_t* __restrict__ cu, int hidden, int pool_mode,
            int normalize, float* __restrict__ out_f32, __nv_bfloat16* __restrict__ out_bf16) {
  __shared__ float red[16];
  ptx::grid_dep_launch();
  ptx::grid_dep_wait();
  const int s = blockIdx.x, lo = cu[s], hi = cu[s + 1];
  const int d = 2 * threadIdx.x;
  float a0 = 0.f, a1 = 0.f;
  if (d < hidden && hi > lo) {
    const int n = pool_mode == 0 ? 1 : hi - lo;
    for (int t = 0; t < n; ++t) {
      const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(x + static_cast<size_t>(lo + t) * hidden + d));
      a0 += __uint_as_float(w << 16); a1 += __uint_as_float(w & 0xFFFF0000u);
    }
    a0 /= n; a1 /= n;
  }
  if (normalize) {
    float ss = warp_sum(a0 * a0 + a1 * a1);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    if (threadIdx.x < 32) {
      float t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
      t = warp_sum(t);
      if (threadIdx.x == 0) red[0] = t;
    }
    __syncthreads();
    const float inv = 1.0f / fmaxf(sqrtf(red[0]), 1e-12f);
    a0 *= inv; a1 *= inv;
  }
  if (d < hidden) {
    if (out_f32) { out_f32[static_cast<size_t>(s) * hidden + d] = a0; out_f32[static_cast<size_t>(s) * hidden + d + 1] = a1; }
    if (out_bf16) *reinterpret_cast<uint32_t*>(out_bf16 + static_cast<size_t>(s) * hidden + d) = pack2(a0, a1);
  }
}

// One vector per text from its windows' pooled fp32 vectors (aur_encode_texts in include/aurora_b200.h, restated by
// oracle/window_mean.py).  One warp per text; lane c owns dims c, c + 32, ..  The window sum runs in window order with
// one rounding per add; the fp64 sum of squares runs per lane in increasing dim, then over the 32 lane sums in lane
// order (every lane adds the same shuffled values in the same order, so every lane holds the same q).  The _rn
// intrinsics keep nvcc from contracting any of it.
__global__ void __launch_bounds__(128)
window_fold_kernel(const float* __restrict__ pool, const FoldItem* __restrict__ items, int n_items, int hidden,
                   int normalize, const float* __restrict__ carry_in, float* __restrict__ carry_out, float* __restrict__ out_f32,
                   __nv_bfloat16* __restrict__ out_bf16) {
  ptx::grid_dep_launch();
  ptx::grid_dep_wait();   // pool_kernel's rows
  const int item = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (item >= n_items) return;
  const FoldItem it = items[item];
  const bool from_carry = it.flags & kFoldCarryIn;
  const float winv = static_cast<float>(it.windows);
  double q = 0.0;
  for (int i = lane; i < hidden; i += 32) {
    float s = from_carry ? carry_in[i] : pool[static_cast<size_t>(it.first) * hidden + i];
    for (int r = it.first + (from_carry ? 0 : 1); r < it.end; ++r) s = __fadd_rn(s, pool[static_cast<size_t>(r) * hidden + i]);
    if (it.flags & kFoldOpen) { carry_out[i] = s; continue; }
    const float m = it.windows == 1 ? s : __fdiv_rn(s, winv);
    q = __dadd_rn(q, __dmul_rn(static_cast<double>(m), static_cast<double>(m)));
    out_f32[static_cast<size_t>(item) * hidden + i] = m;
  }
  if ((it.flags & kFoldOpen) || !normalize || it.windows == 1) {
    if (!(it.flags & kFoldOpen))
      for (int i = lane; i < hidden; i += 32)
        out_bf16[static_cast<size_t>(item) * hidden + i] = __float2bfloat16_rn(out_f32[static_cast<size_t>(item) * hidden + i]);
    return;
  }
  double tot = 0.0;
#pragma unroll
  for (int c = 0; c < 32; ++c) tot = __dadd_rn(tot, __shfl_sync(0xffffffffu, q, c));
  const double root = tot > 0.0 ? __dsqrt_rn(tot) : 1.0;
  for (int i = lane; i < hidden; i += 32) {
    float* o = out_f32 + static_cast<size_t>(item) * hidden + i;
    const float v = tot > 0.0 ? __double2float_rn(__ddiv_rn(static_cast<double>(*o), root)) : *o;
    *o = v;
    out_bf16[static_cast<size_t>(item) * hidden + i] = __float2bfloat16_rn(v);
  }
}

__global__ void f32_to_bf16_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out, int64_t n) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) out[i] = __float2bfloat16_rn(in[i]);
}

}  // namespace

cudaError_t launch_embed_ln(const int32_t* tok, const int32_t* pos, int n_tok, int n_rows_pad,
                            const __nv_bfloat16* word, const __nv_bfloat16* pos_emb, const __nv_bfloat16* type_emb,
                            const float* g, const float* b, float eps, int hidden, __nv_bfloat16* out, cudaStream_t s) {
  if (n_rows_pad <= 0) return cudaSuccess;
  return launch_pdl(embed_ln_kernel, dim3((n_rows_pad + 7) / 8), dim3(256), 0, s, 1, tok, pos, n_tok, n_rows_pad, word,
                    pos_emb, type_emb, g, b, eps, hidden, out);
}

cudaError_t launch_layernorm(const __nv_bfloat16* in, const float* g, const float* b, float eps, int n_rows, int hidden,
                             __nv_bfloat16* out, cudaStream_t s) {
  if (n_rows <= 0) return cudaSuccess;
  return launch_pdl(layernorm_kernel, dim3((n_rows + 15) / 16), dim3(256), 0, s, 1, in, g, b, eps, n_rows, hidden, out);
}

cudaError_t launch_pool(const __nv_bfloat16* x, const int32_t* cu, int n_seq, int hidden, int pool_mode, int normalize,
                        float* out_f32, __nv_bfloat16* out_bf16, cudaStream_t s) {
  if (n_seq <= 0) return cudaSuccess;
  const int threads = ((hidden / 2 + 31) / 32) * 32;
  return launch_pdl(pool_kernel, dim3(n_seq), dim3(threads), 0, s, 1, x, cu, hidden, pool_mode, normalize, out_f32, out_bf16);
}

cudaError_t launch_window_fold(const float* pool_f32, const FoldItem* items, int n_items, int hidden, int normalize,
                               const float* carry_in, float* carry_out, float* out_f32, __nv_bfloat16* out_bf16, cudaStream_t s) {
  if (n_items <= 0) return cudaSuccess;
  return launch_pdl(window_fold_kernel, dim3((n_items + 3) / 4), dim3(128), 0, s, 1, pool_f32, items, n_items, hidden,
                    normalize, carry_in, carry_out, out_f32, out_bf16);
}

cudaError_t launch_f32_to_bf16(const float* in, __nv_bfloat16* out, int64_t n, cudaStream_t s) {
  if (n <= 0) return cudaSuccess;
  f32_to_bf16_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(in, out, n);
  return cudaGetLastError();
}

}  // namespace aur
