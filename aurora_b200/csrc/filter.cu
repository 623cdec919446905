// Metadata pre-filters evaluated on the device (aur_search_filtered, aur_filter_ids, aur_hybrid_search_filtered).
//
// A program is a postfix sequence of leaves and AND / OR tokens (FiltToken).  A leaf (column, bitmap offset, bitmap length)
// is true for a row when bit code + 1 of its bitmap slice is set, code being the row's int32 value in that column (-1 =
// property absent).  Columns 0 / 1 are the shard's (or keyword store's) tenant codes, 2.. its attribute columns.  Three
// kernels:
//   filter_count_kernel  one pass over the snapshot's rows: every live row's match bits (bit p = program p, up to 32
//                        programs) into a per-row mask, per-block counts per program and the per-program totals; over a
//                        keyword store's rows (the hybrid query's keyword leg) the mask alone;
//   filter_scan_kernel   exclusive scan of each program's block counts, offset by the programs before it;
//   filter_write_kernel  each program's matching rows in ascending row order (and optionally their ids) into one buffer:
//                        the rows the host path stages after its sort and unique.
// mask_match_kernel turns bit 0 of the mask into the masked inverse norms the tensor-core scan takes.
// The host side is here too, one copy for the vector shard and the keyword store: program checks, attribute columns
// (AttrColumns) and program uploads (filter_upload), so the two legs of a filtered hybrid query cannot disagree.
#include <math.h>
#include <string.h>

#include "../../include/aurora_b200.h"
#include "internal.h"

namespace aur {
namespace {

constexpr int kFiltThreads = 256;
constexpr int kFiltWarps = kFiltThreads / 32;
constexpr unsigned kFull = 0xFFFFFFFFu;

__device__ __forceinline__ bool leaf_true(const FiltParams& p, const FiltToken& t, int64_t row) {
  const int32_t idx = __ldg(p.cols[t.col] + row) + 1;
  if (idx < 0 || idx >= t.bm_len) return false;
  const int64_t bit = static_cast<int64_t>(t.bm_off) + idx;
  return (__ldg(p.bitmap + (bit >> 5)) >> (bit & 31)) & 1u;
}

// Match bits of one row: the stack of a postfix program fits one word (<= kFiltMaxLeaves leaves, so <= 32 deep).
__device__ __forceinline__ uint32_t row_match(const FiltParams& p, int64_t row) {
  uint32_t m = 0u;
  for (int q = 0; q < p.n_programs; ++q) {
    uint32_t st = 0u;
    const int t1 = __ldg(p.prog_off + q + 1);
    for (int t = __ldg(p.prog_off + q); t < t1; ++t) {
      const FiltToken tk = p.tok[t];
      if (tk.kind == kFiltLeaf) {
        st = (st << 1) | static_cast<uint32_t>(leaf_true(p, tk, row));
      } else {
        const uint32_t a = st & 1u, b = (st >> 1) & 1u;
        st = ((st >> 2) << 1) | (tk.kind == kFiltAnd ? (a & b) : (a | b));
      }
    }
    m |= (st & 1u) << q;
  }
  return m;
}

// kMaskOnly: a keyword store's rows (liveness from p.live), the mask alone -- its consumer is a kernel, so nothing is
// counted for the host.  Otherwise a vector shard's rows (liveness from p.inv_norm), mask and counts.
template <bool kMaskOnly>
__global__ void __launch_bounds__(kFiltThreads) filter_count_kernel(FiltParams p, uint32_t* __restrict__ mask,
                                                                    uint32_t* __restrict__ block_counts,
                                                                    uint32_t* __restrict__ totals, int n_blocks) {
  if constexpr (kMaskOnly) {
    const int64_t base = static_cast<int64_t>(blockIdx.x) * kFiltBlockRows;
    for (int it = 0; it < kFiltBlockRows / kFiltThreads; ++it) {
      const int64_t row = base + it * kFiltThreads + threadIdx.x;
      if (row < p.n_rows) mask[row] = __ldg(p.live + row) ? row_match(p, row) : 0u;
    }
    return;
  }
  __shared__ uint32_t s_cnt[32];
  if (threadIdx.x < 32) s_cnt[threadIdx.x] = 0u;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  uint32_t mine = 0u;   // lane q: this warp's matches of program q
  const int64_t base = static_cast<int64_t>(blockIdx.x) * kFiltBlockRows;
  for (int it = 0; it < kFiltBlockRows / kFiltThreads; ++it) {
    const int64_t row = base + it * kFiltThreads + threadIdx.x;
    uint32_t m = 0u;
    if (row < p.n_rows) {
      const float inv = __ldg(p.inv_norm + row);
      if (inv == inv) m = row_match(p, row);   // NaN = tombstone
      mask[row] = m;
    }
    for (int q = 0; q < p.n_programs; ++q) {
      const uint32_t c = __popc(__ballot_sync(kFull, (m >> q) & 1u));
      if (lane == q) mine += c;
    }
  }
  if (lane < p.n_programs && mine) atomicAdd(&s_cnt[lane], mine);
  __syncthreads();
  if (threadIdx.x < p.n_programs) {
    block_counts[static_cast<size_t>(threadIdx.x) * n_blocks + blockIdx.x] = s_cnt[threadIdx.x];
    if (s_cnt[threadIdx.x]) atomicAdd(totals + threadIdx.x, s_cnt[threadIdx.x]);
  }
}

// One CTA per program: its block counts become exclusive offsets into the output, past the programs before it.
__global__ void __launch_bounds__(1024) filter_scan_kernel(uint32_t* __restrict__ block_counts, const uint32_t* __restrict__ totals,
                                                           int n_blocks) {
  __shared__ uint32_t s_warp[32];
  __shared__ uint32_t s_carry;
  const int q = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    uint32_t b = 0u;
    for (int j = 0; j < q; ++j) b += totals[j];
    s_carry = b;
  }
  __syncthreads();
  uint32_t* c = block_counts + static_cast<size_t>(q) * n_blocks;
  for (int i0 = 0; i0 < n_blocks; i0 += blockDim.x) {
    const int i = i0 + threadIdx.x;
    const uint32_t v = i < n_blocks ? c[i] : 0u;
    uint32_t x = v;   // inclusive warp scan
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(kFull, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    if (warp == 0) {
      uint32_t w = lane < static_cast<int>(blockDim.x >> 5) ? s_warp[lane] : 0u;
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(kFull, w, o);
        if (lane >= o) w += y;
      }
      s_warp[lane] = w;   // inclusive over warps
    }
    __syncthreads();
    const uint32_t before = (warp ? s_warp[warp - 1] : 0u) + x - v;
    if (i < n_blocks) c[i] = s_carry + before;
    __syncthreads();
    if (threadIdx.x == 0) s_carry += s_warp[(blockDim.x >> 5) - 1];
    __syncthreads();
  }
}

// Same rows per CTA as the count kernel; inside a CTA the rows go out in row order: by pass, then warp, then lane.
__global__ void __launch_bounds__(kFiltThreads) filter_write_kernel(const uint32_t* __restrict__ mask, const uint32_t* __restrict__ offsets,
                                                                    int n_blocks, int n_programs, int64_t n_rows,
                                                                    const int64_t* __restrict__ ids, int32_t* __restrict__ rows_out,
                                                                    int64_t* __restrict__ ids_out) {
  __shared__ uint32_t s_base[32];
  __shared__ uint32_t s_wcnt[kFiltWarps][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x < n_programs) s_base[threadIdx.x] = offsets[static_cast<size_t>(threadIdx.x) * n_blocks + blockIdx.x];
  const int64_t base = static_cast<int64_t>(blockIdx.x) * kFiltBlockRows;
  const uint32_t lt = (1u << lane) - 1u;
  for (int it = 0; it < kFiltBlockRows / kFiltThreads; ++it) {
    const int64_t row = base + it * kFiltThreads + threadIdx.x;
    const uint32_t m = row < n_rows ? mask[row] : 0u;
    for (int q = 0; q < n_programs; ++q) {
      const uint32_t bal = __ballot_sync(kFull, (m >> q) & 1u);
      if (lane == 0) s_wcnt[warp][q] = __popc(bal);
    }
    __syncthreads();
    for (int q = 0; q < n_programs; ++q) {
      const uint32_t bal = __ballot_sync(kFull, (m >> q) & 1u);
      if ((m >> q) & 1u) {
        uint32_t pos = s_base[q] + __popc(bal & lt);
        for (int w = 0; w < warp; ++w) pos += s_wcnt[w][q];
        rows_out[pos] = static_cast<int32_t>(row);
        if (ids_out) ids_out[pos] = ids[row];
      }
    }
    __syncthreads();
    if (threadIdx.x < n_programs) {
      uint32_t add = 0u;
      for (int w = 0; w < kFiltWarps; ++w) add += s_wcnt[w][threadIdx.x];
      s_base[threadIdx.x] += add;
    }
    __syncthreads();
  }
}

// Dense case: out[row] = row matches program 0 ? inv[row] : NaN (tombstones never match, so they stay NaN).
__global__ void mask_match_kernel(const float* __restrict__ inv, const uint32_t* __restrict__ mask, int64_t n, float* __restrict__ out) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  out[i] = (mask[i] & 1u) ? inv[i] : __uint_as_float(0x7FC00000u);
}

// Attribute codes by row (aur_set_attrs): pairs[2 i] = row, pairs[2 i + 1] = code.
__global__ void scatter_codes_kernel(const int32_t* __restrict__ pairs, int64_t n, int32_t* __restrict__ col) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) col[pairs[2 * i]] = pairs[2 * i + 1];
}

__global__ void gather_i32_kernel(const int32_t* __restrict__ src, const int32_t* __restrict__ map, int64_t n, int32_t* __restrict__ out) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) out[i] = src[map[i]];
}

unsigned blocks_of(int64_t n, int per) { return static_cast<unsigned>((n + per - 1) / per); }

}  // namespace

int filter_blocks(int64_t n_rows) { return static_cast<int>((n_rows + kFiltBlockRows - 1) / kFiltBlockRows); }

cudaError_t launch_filter_count(const FiltParams& p, uint32_t* mask, uint32_t* block_counts, uint32_t* totals, cudaStream_t s) {
  cudaError_t e = cudaMemsetAsync(totals, 0, 32 * sizeof(uint32_t), s);
  if (e != cudaSuccess || p.n_rows <= 0) return e;
  const int nb = filter_blocks(p.n_rows);
  filter_count_kernel<false><<<nb, kFiltThreads, 0, s>>>(p, mask, block_counts, totals, nb);
  return cudaGetLastError();
}

cudaError_t launch_filter_mask(const FiltParams& p, uint32_t* mask, cudaStream_t s) {
  if (p.n_rows <= 0) return cudaSuccess;
  const int nb = filter_blocks(p.n_rows);
  filter_count_kernel<true><<<nb, kFiltThreads, 0, s>>>(p, mask, nullptr, nullptr, nb);
  return cudaGetLastError();
}

cudaError_t launch_filter_write(const uint32_t* mask, uint32_t* block_counts, const uint32_t* totals, int n_programs, int64_t n_rows,
                                const int64_t* ids, int32_t* rows_out, int64_t* ids_out, cudaStream_t s) {
  if (n_rows <= 0) return cudaSuccess;
  const int nb = filter_blocks(n_rows);
  filter_scan_kernel<<<n_programs, 1024, 0, s>>>(block_counts, totals, nb);
  filter_write_kernel<<<nb, kFiltThreads, 0, s>>>(mask, block_counts, nb, n_programs, n_rows, ids, rows_out, ids_out);
  return cudaGetLastError();
}

cudaError_t launch_mask_match(const float* inv, const uint32_t* mask, int64_t n, float* out, cudaStream_t s) {
  if (n <= 0) return cudaSuccess;
  mask_match_kernel<<<blocks_of(n, 256), 256, 0, s>>>(inv, mask, n, out);
  return cudaGetLastError();
}

// ---------------------------------------------------------------- host side: programs, attribute columns, uploads
int filter_check_programs(const FiltProgs& fp) {
  if (!fp.prog || !fp.prog_off) return report_error(AUR_ERR_INVALID, "null program");
  if (fp.n_programs < 1 || fp.n_programs > kFiltCallPrograms) return report_error(AUR_ERR_INVALID, "1 <= n_programs <= %d", kFiltCallPrograms);
  if (fp.bitmap_words < 0 || (fp.bitmap_words > 0 && !fp.bitmap)) return report_error(AUR_ERR_INVALID, "bitmap / bitmap_words");
  if (fp.prog_off[0] != 0) return report_error(AUR_ERR_INVALID, "program offsets must start at 0");
  for (int32_t q = 0; q < fp.n_programs; ++q) {
    if (fp.prog_off[q + 1] < fp.prog_off[q]) return report_error(AUR_ERR_INVALID, "program offsets decrease at program %d", q);
    int depth = 0, leaves = 0;
    for (int32_t t = fp.prog_off[q]; t < fp.prog_off[q + 1]; ++t) {
      const int32_t* tk = fp.prog + 4 * static_cast<int64_t>(t);
      if (tk[0] == kFiltLeaf) {
        if (++leaves > kFiltMaxLeaves) return report_error(AUR_ERR_INVALID, "program %d has more than %d leaves", q, kFiltMaxLeaves);
        if (tk[1] < 0 || tk[1] >= kFiltCols) return report_error(AUR_ERR_INVALID, "program %d: column %d out of range", q, tk[1]);
        if (tk[2] < 0 || tk[3] < 0 || static_cast<int64_t>(tk[2]) + tk[3] > fp.bitmap_words * 32)
          return report_error(AUR_ERR_INVALID, "program %d: bitmap slice [%d, +%d) outside the bitmap", q, tk[2], tk[3]);
        ++depth;
      } else if (tk[0] == kFiltAnd || tk[0] == kFiltOr) {
        if (depth < 2) return report_error(AUR_ERR_INVALID, "program %d: operator without two operands", q);
        --depth;
      } else {
        return report_error(AUR_ERR_INVALID, "program %d: unknown token kind %d", q, tk[0]);
      }
    }
    if (depth != 1) return report_error(AUR_ERR_INVALID, "program %d leaves %d values, not one", q, depth);
  }
  return AUR_OK;
}

int filter_check_queries(const FiltProgs& fp, int32_t nq, int64_t max_list_rows) {
  if (!fp.q_program) return report_error(AUR_ERR_INVALID, "q_program is required");
  for (int32_t q = 0; q < nq; ++q)
    if (fp.q_program[q] < 0 || fp.q_program[q] >= fp.n_programs)
      return report_error(AUR_ERR_INVALID, "q_program[%d] = %d is not a program", q, fp.q_program[q]);
  if (max_list_rows < 0) return report_error(AUR_ERR_INVALID, "max_list_rows < 0");
  return AUR_OK;
}

int AttrColumns::write(int32_t col, const std::vector<int32_t>& pairs, int64_t rows, cudaStream_t s) {
  if (col < 2 || col >= kFiltCols) return report_error(AUR_ERR_INVALID, "attribute columns are 2 .. %d", kFiltCols - 1);
  const cudaError_t e = [&]() -> cudaError_t {
    if (!d_attr[col - 2].p) {   // (writes are serialised: only this call stores a column)
      int dev = 0;
      AUR_CU_RET(cudaGetDevice(&dev));
      VmmBuf<int32_t> a;
      AUR_CU_RET(a.open(dev, 1, static_cast<size_t>(rows)));
      AUR_CU_RET(cudaMemsetAsync(a.p, 0xFF, static_cast<size_t>(rows) * 4, s));
      AUR_CU_RET(cudaStreamSynchronize(s));
      std::lock_guard<std::mutex> lk(mu);
      d_attr[col - 2] = std::move(a);
    }
    if (pairs.empty()) return cudaSuccess;
    AUR_CU_RET(stage.reserve(pairs.size()));
    AUR_CU_RET(cudaMemcpyAsync(stage.p, pairs.data(), pairs.size() * 4, cudaMemcpyHostToDevice, s));
    const int64_t n = static_cast<int64_t>(pairs.size() / 2);
    scatter_codes_kernel<<<blocks_of(n, 256), 256, 0, s>>>(stage.p, n, d_attr[col - 2].p);
    AUR_CU_RET(cudaGetLastError());
    return cudaStreamSynchronize(s);
  }();
  if (e == cudaSuccess) return AUR_OK;
  return report_error(e == cudaErrorMemoryAllocation ? AUR_ERR_NOMEM : AUR_ERR_CUDA, "attribute column: %s", cudaGetErrorString(e));
}

bool AttrColumns::any() { return std::any_of(std::begin(d_attr), std::end(d_attr), [](const VmmBuf<int32_t>& a) { return a.p != nullptr; }); }

cudaError_t AttrColumns::grow(int64_t old_rows, int64_t rows, cudaStream_t s) {
  size_t before[kFiltAttrCols] = {};
  for (int i = 0; i < kFiltAttrCols; ++i) before[i] = d_attr[i].r.mapped();
  const cudaError_t e = [&]() -> cudaError_t {
    for (VmmBuf<int32_t>& a : d_attr) {
      if (!a.p || rows <= old_rows) continue;
      AUR_CU_RET(a.grow(static_cast<size_t>(rows)));
      AUR_CU_RET(cudaMemsetAsync(a.p + old_rows, 0xFF, static_cast<size_t>(rows - old_rows) * 4, s));
    }
    return cudaStreamSynchronize(s);
  }();
  if (e != cudaSuccess) {
    cudaStreamSynchronize(s);   // a tail memset may still be pending: nothing is unmapped under it
    cudaGetLastError();
    for (int i = 0; i < kFiltAttrCols; ++i) d_attr[i].shrink_to_bytes(before[i]);
  }
  return e;
}

cudaError_t AttrColumns::gather(const int32_t* map, int64_t m, int64_t dst0, int32_t* bounce, cudaStream_t s) {
  for (const VmmBuf<int32_t>& a : d_attr) {
    if (!a.p || m <= 0) continue;
    gather_i32_kernel<<<blocks_of(m, 256), 256, 0, s>>>(a.p, map, m, bounce);
    AUR_CU_RET(cudaGetLastError());
    AUR_CU_RET(cudaMemcpyAsync(a.p + dst0, bounce, static_cast<size_t>(m) * 4, cudaMemcpyDeviceToDevice, s));
  }
  return cudaSuccess;
}

cudaError_t AttrColumns::clear(int64_t r0, int64_t r1, cudaStream_t s) {
  for (const VmmBuf<int32_t>& a : d_attr)
    if (a.p && r1 > r0) AUR_CU_RET(cudaMemsetAsync(a.p + r0, 0xFF, static_cast<size_t>(r1 - r0) * 4, s));
  return cudaSuccess;
}

int AttrColumns::check(const FiltProgs& fp, const char* holder) {
  std::lock_guard<std::mutex> lk(mu);
  for (int32_t t = 0; t < fp.prog_off[fp.n_programs]; ++t) {
    const int32_t* tk = fp.prog + 4 * static_cast<int64_t>(t);
    if (tk[0] == kFiltLeaf && tk[1] >= 2 && !d_attr[tk[1] - 2].p)
      return report_error(AUR_ERR_INVALID, "column %d was never set on the %s", tk[1], holder);
  }
  return AUR_OK;
}

void AttrColumns::fill(FiltParams* p) {
  std::lock_guard<std::mutex> lk(mu);
  for (int i = 0; i < kFiltAttrCols; ++i) p->cols[2 + i] = d_attr[i].p;
}

cudaError_t filter_upload(const FiltProgs& fp, const int32_t* user, const int32_t* org, AttrColumns& attrs,
                          DevBuf<int32_t>& stage, cudaStream_t s, FiltParams* p) {
  const size_t n_tok = static_cast<size_t>(fp.prog_off[fp.n_programs]), n_off = static_cast<size_t>(fp.n_programs) + 1;
  std::vector<int32_t> st(n_tok * 4 + n_off + static_cast<size_t>(fp.bitmap_words));
  if (n_tok) memcpy(st.data(), fp.prog, n_tok * 16);
  memcpy(st.data() + n_tok * 4, fp.prog_off, n_off * 4);
  if (fp.bitmap_words) memcpy(st.data() + n_tok * 4 + n_off, fp.bitmap, static_cast<size_t>(fp.bitmap_words) * 4);
  AUR_CU_RET(stage.reserve(st.size()));
  AUR_CU_RET(cudaMemcpyAsync(stage.p, st.data(), st.size() * 4, cudaMemcpyHostToDevice, s));
  *p = FiltParams{};
  p->cols[0] = user; p->cols[1] = org;
  attrs.fill(p);
  p->tok = reinterpret_cast<const FiltToken*>(stage.p);
  p->prog_off = stage.p + n_tok * 4;   // token indices stay absolute: a pass starts at its first offset
  p->bitmap = reinterpret_cast<const uint32_t*>(p->prog_off + n_off);
  p->n_programs = fp.n_programs;
  return cudaSuccess;
}

}  // namespace aur
