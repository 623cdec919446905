// Host-side k-way merge of per-shard top-k lists for the single-owner multi-GPU deployment (engine.MultiIndex): every
// shard answers from its own GPU through aur_search, the owner process folds the <= 64 short, already sorted lists of a
// query here.  Order = the device merge's (csrc/kernels_simt.cu merge_topk_kernel): score descending, then id
// ascending; empty slots (id < 0) last.  Replaces the coordinator-side merge inside Weaviate for a multi-shard class
// (external to /root/reference; call site weaviate_client.py:252-259).  The same merge on fp64 scores folds the
// keyword stores' lists of aur_kw_search_multi (csrc/keyword.cu), whose scores are exact fp64 BM25.
#include <stddef.h>
#include <stdint.h>

#include <limits>

#include "../../include/aurora_b200.h"

namespace {

template <typename Score>
int merge_topk_host(const Score* scores, const int64_t* ids, int32_t n_lists, int32_t nq, int32_t k_in, int32_t k_out,
                    Score* out_scores, int64_t* out_ids) {
  if (!scores || !ids || !out_scores || !out_ids || n_lists < 1 || n_lists > 64 || nq < 0 || k_in < 1 || k_out < 1)
    return AUR_ERR_INVALID;
  const size_t plane = static_cast<size_t>(nq) * k_in;
  for (int32_t q = 0; q < nq; ++q) {
    int32_t head[64] = {0};
    for (int32_t o = 0; o < k_out; ++o) {
      int best = -1;
      Score bs = 0;
      int64_t bi = 0;
      for (int32_t l = 0; l < n_lists; ++l) {
        if (head[l] >= k_in) continue;
        const size_t at = l * plane + static_cast<size_t>(q) * k_in + head[l];
        const int64_t id = ids[at];
        if (id < 0) { head[l] = k_in; continue; }          // a list's padding starts here: it is exhausted
        const Score s = scores[at];
        if (best < 0 || s > bs || (s == bs && id < bi)) { best = l; bs = s; bi = id; }
      }
      if (best < 0) {
        out_scores[static_cast<size_t>(q) * k_out + o] = -std::numeric_limits<Score>::infinity();
        out_ids[static_cast<size_t>(q) * k_out + o] = -1;
      } else {
        out_scores[static_cast<size_t>(q) * k_out + o] = bs;
        out_ids[static_cast<size_t>(q) * k_out + o] = bi;
        ++head[best];
      }
    }
  }
  return AUR_OK;
}

}  // namespace

extern "C" int aur_merge_topk_host(const float* scores, const int64_t* ids, int32_t n_lists, int32_t nq, int32_t k_in,
                                   int32_t k_out, float* out_scores, int64_t* out_ids) {
  return merge_topk_host<float>(scores, ids, n_lists, nq, k_in, k_out, out_scores, out_ids);
}

extern "C" int aur_merge_topk_host_f64(const double* scores, const int64_t* ids, int32_t n_lists, int32_t nq, int32_t k_in,
                                       int32_t k_out, double* out_scores, int64_t* out_ids) {
  return merge_topk_host<double>(scores, ids, n_lists, nq, k_in, k_out, out_scores, out_ids);
}
