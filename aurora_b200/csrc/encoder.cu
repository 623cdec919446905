// Host runtime of the text encoder behind the C ABI (include/aurora_b200.h, "text encoder").
// Owns the bf16 parameters and one activation workspace in HBM:
//   x, y   [max_tokens_pad, H]    residual stream / pre-LayerNorm sum
//   qkv    [max_tokens_pad, 3H]   packed projections (attention reads Q, K, V tiles from it by TMA)
//   ctx    [max_tokens_pad, H]    attention output
//   inter  [max_tokens_pad, I]    FFN activation
// and the TMA descriptors over them (activations as GEMM A operands, weights as B operands).
// A forward is 2 + 7*L + 1 kernel launches on one stream; no CPU compute path exists.  aur_encoder_replicate copies a
// loaded encoder's parameters to a fresh encoder on any device; aur_encode_append_texts_multi runs one encoder per shard
// of a multi-GPU corpus, each on its own host thread, the text vectors going straight into its shard.  A text longer than
// the position table arrives as several windows (sequences); one more launch, window_fold_kernel, turns a batch's window
// vectors into text vectors, with the running sum of a text still open at the batch's end kept in a carry row:
//   fold   [max_seqs + 2, H] fp32  text vectors of the batch, then two carry rows (a batch may read one and write the other)
// (6.3 MB at bge-base dims and the default 2048 sequences).  Batches without such a text launch no fold.
#include <algorithm>
#include <functional>
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/aurora_b200.h"
#include "internal.h"

using namespace aur;

namespace {

struct Layer {
  DevBuf<__nv_bfloat16> wqkv, wo, wi, wo2;
  DevBuf<float> bqkv, bo, bi, bo2;
  DevBuf<float> ln1_g, ln1_b, ln2_g, ln2_b;
  CUtensorMap tm_wqkv, tm_wo, tm_wi, tm_wo2;
};

int round_up(int v, int m) { return (v + m - 1) / m * m; }

}  // namespace

struct aur_encoder {
  std::mutex mu;
  aur_encoder_config cfg{};
  int rows_pad = 0;            // workspace rows (max_tokens rounded up to 128)
  int bn = 256;                // GEMM N tile: 256 when every N divides, else 128
  int cta_group = 2;           // CTAs per GEMM tile (2: 256-row tiles, the weight tile split over the pair)
  int dh = 64;                 // real head dim (64, or 32 zero-padded to 64 inside the qkv / ctx layout)
  int hp = 0;                  // heads * 64: width of each of q, k, v in the qkv buffer and of ctx
  int sm_count = 0;
  Stream stream;
  Event ev[4];
  DevBuf<__nv_bfloat16> word, pos, type;
  DevBuf<float> emb_g, emb_b;
  std::vector<Layer> layers;
  std::vector<std::string> missing;   // parameter names not loaded yet
  DevBuf<__nv_bfloat16> x, y, qkv, ctx, inter;
  CUtensorMap tm_x, tm_ctx, tm_inter, tm_qkv;       // loads: box {64, 128}
  DevBuf<int32_t> d_tok, d_pos, d_cu;
  DevBuf<AttnItem> d_items;
  int max_items = 0;
  DevBuf<float> d_pool_f32;
  DevBuf<__nv_bfloat16> d_pool_bf16;
  DevBuf<float> d_fold_f32;                           // [max_seqs + 2, H]: window_fold_kernel's text vectors + 2 carry rows
  DevBuf<FoldItem> d_fold;                            // [max_seqs]
  HostBuf<FoldItem> h_fold;
  DevBuf<float> d_stage;                              // fp32 staging for parameter upload
  HostBuf<int32_t> h_tok, h_pos;
  HostBuf<AttnItem> h_items;
  aur_encoder_stats stats{};
  int64_t last_tokens = 0;
};

namespace {

int make_tmap(CUtensorMap* tm, const void* base, int cols, int rows, int box_rows) {
  const int r = encode_tmap_2d_bf16(tm, base, static_cast<uint64_t>(cols), static_cast<uint64_t>(rows),
                                    static_cast<uint64_t>(cols) * 2, 64, static_cast<uint32_t>(box_rows));
  if (r != 0) return report_error(AUR_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d) for [%d x %d] box %d", r, rows, cols, box_rows);
  return AUR_OK;
}

template <typename T>
int dev_alloc(DevBuf<T>& b, size_t n) {
  AUR_TRY(b.reserve(n));
  AUR_TRY(cudaMemset(b.p, 0, n * sizeof(T)));
  return AUR_OK;
}

// Every parameter buffer of e (its owner) with its element count (the head-dim-32 layouts padded as stored), in one fixed order:
// aur_encoder_open allocates them, aur_encoder_replicate copies them buffer for buffer.
template <typename F>
void for_each_param(aur_encoder* e, F&& f) {
  const aur_encoder_config& c = e->cfg;
  const size_t H = c.hidden, I = c.inter, HP = e->hp;
  f(e->word, static_cast<size_t>(c.vocab) * H); f(e->pos, static_cast<size_t>(c.max_pos) * H);
  f(e->type, static_cast<size_t>(c.type_vocab) * H); f(e->emb_g, H); f(e->emb_b, H);
  for (Layer& l : e->layers) {
    f(l.wqkv, 3 * HP * H); f(l.wo, H * HP); f(l.wi, I * H); f(l.wo2, H * I);
    f(l.bqkv, 3 * HP); f(l.bo, H); f(l.bi, I); f(l.bo2, H);
    f(l.ln1_g, H); f(l.ln1_b, H); f(l.ln2_g, H); f(l.ln2_b, H);
  }
}

// pad: 0 none; 1 rows are [3][heads][dh] -> [3][heads][64] (wqkv / bqkv); 2 columns are [heads][dh] -> [heads][64] (wo)
struct ParamSlot { void* dst; int64_t count; bool bf16; int pad; };

// Resolve a parameter name to its device buffer.
bool find_param(aur_encoder* e, const std::string& name, ParamSlot* out) {
  const aur_encoder_config& c = e->cfg;
  const int64_t H = c.hidden, I = c.inter;
  if (name == "word_emb") { *out = {e->word.p, static_cast<int64_t>(c.vocab) * H, true, 0}; return true; }
  if (name == "pos_emb") { *out = {e->pos.p, static_cast<int64_t>(c.max_pos) * H, true, 0}; return true; }
  if (name == "type_emb") { *out = {e->type.p, static_cast<int64_t>(c.type_vocab) * H, true, 0}; return true; }
  if (name == "emb_ln_g") { *out = {e->emb_g.p, H, false, 0}; return true; }
  if (name == "emb_ln_b") { *out = {e->emb_b.p, H, false, 0}; return true; }
  int l = -1; char leaf[32] = {0};
  if (sscanf(name.c_str(), "l%d.%31s", &l, leaf) != 2 || l < 0 || l >= c.layers) return false;
  Layer& L = e->layers[l];
  const std::string f = leaf;
  const int padded = e->dh != 64;
  if (f == "wqkv") { *out = {L.wqkv.p, 3 * H * H, true, padded ? 1 : 0}; return true; }
  if (f == "wo") { *out = {L.wo.p, H * H, true, padded ? 2 : 0}; return true; }
  if (f == "wi") { *out = {L.wi.p, I * H, true, 0}; return true; }
  if (f == "wo2") { *out = {L.wo2.p, H * I, true, 0}; return true; }
  if (f == "bqkv") { *out = {L.bqkv.p, 3 * H, false, padded ? 1 : 0}; return true; }
  if (f == "bo") { *out = {L.bo.p, H, false, 0}; return true; }
  if (f == "bi") { *out = {L.bi.p, I, false, 0}; return true; }
  if (f == "bo2") { *out = {L.bo2.p, H, false, 0}; return true; }
  if (f == "ln1_g") { *out = {L.ln1_g.p, H, false, 0}; return true; }
  if (f == "ln1_b") { *out = {L.ln1_b.p, H, false, 0}; return true; }
  if (f == "ln2_g") { *out = {L.ln2_g.p, H, false, 0}; return true; }
  if (f == "ln2_b") { *out = {L.ln2_b.p, H, false, 0}; return true; }
  return false;
}

int gemm(aur_encoder* e, const CUtensorMap* tm_a, const CUtensorMap* tm_w, __nv_bfloat16* out, int m_rows, int n,
         int k, int epi, const float* bias, const __nv_bfloat16* resid, int ldr) {
  GemmParams p{};
  p.bias = bias; p.resid = resid; p.ldr = ldr; p.out = out; p.ldo = n;
  const int tile_m = 128 * e->cta_group;
  p.m_tiles = (m_rows + tile_m - 1) / tile_m; p.n_tiles = n / e->bn; p.k_blocks = k / 64;
  AUR_TRY(gemm_tc_launch(e->cta_group, e->bn, epi, e->sm_count, tm_a, tm_w, p, e->stream));
  return AUR_OK;
}

// The whole forward for tokens already staged in h_tok / h_pos / h_items.
int forward_locked(aur_encoder* e, const int32_t* cu_host, int n_seq, int n_items) {
  const aur_encoder_config& c = e->cfg;
  const int T = cu_host[n_seq], H = c.hidden, I = c.inter;
  const int t_pad = round_up(T, 256);
  cudaStream_t s = e->stream;
  AUR_TRY(cudaMemcpyAsync(e->d_tok.p, e->h_tok.p, sizeof(int32_t) * T, cudaMemcpyHostToDevice, s));
  AUR_TRY(cudaMemcpyAsync(e->d_pos.p, e->h_pos.p, sizeof(int32_t) * T, cudaMemcpyHostToDevice, s));
  AUR_TRY(cudaMemcpyAsync(e->d_cu.p, cu_host, sizeof(int32_t) * (n_seq + 1), cudaMemcpyHostToDevice, s));
  AUR_TRY(cudaMemcpyAsync(e->d_items.p, e->h_items.p, sizeof(AttnItem) * n_items, cudaMemcpyHostToDevice, s));
  AUR_TRY(cudaEventRecord(e->ev[0], s));
  int launches = 0;
  AUR_TRY(launch_embed_ln(e->d_tok.p, e->d_pos.p, T, t_pad, e->word.p, e->pos.p, e->type.p, e->emb_g.p, e->emb_b.p, c.ln_eps, H, e->x.p, s));
  ++launches;
  AttnParams ap{};
  const int HP = e->hp;
  ap.items = e->d_items.p; ap.n_items = n_items; ap.heads = c.heads; ap.hidden = HP; ap.ctx = e->ctx.p; ap.ld_ctx = HP;
  ap.scale_log2e = 1.4426950408889634f / sqrtf(static_cast<float>(e->dh));
  for (int l = 0; l < c.layers; ++l) {
    Layer& L = e->layers[l];
    int rc;
    if ((rc = gemm(e, &e->tm_x, &L.tm_wqkv, e->qkv.p, T, 3 * HP, H, kEpiBias, L.bqkv.p, nullptr, 0))) return rc;
    AUR_TRY(attn_tc_launch(&e->tm_qkv, ap, s));
    if ((rc = gemm(e, &e->tm_ctx, &L.tm_wo, e->y.p, T, H, HP, kEpiBiasResid, L.bo.p, e->x.p, H))) return rc;
    AUR_TRY(launch_layernorm(e->y.p, L.ln1_g.p, L.ln1_b.p, c.ln_eps, T, H, e->x.p, s));
    if ((rc = gemm(e, &e->tm_x, &L.tm_wi, e->inter.p, T, I, H, kEpiBiasGelu, L.bi.p, nullptr, 0))) return rc;
    if ((rc = gemm(e, &e->tm_inter, &L.tm_wo2, e->y.p, T, H, I, kEpiBiasResid, L.bo2.p, e->x.p, H))) return rc;
    AUR_TRY(launch_layernorm(e->y.p, L.ln2_g.p, L.ln2_b.p, c.ln_eps, T, H, e->x.p, s));
    launches += 7;
  }
  AUR_TRY(launch_pool(e->x.p, e->d_cu.p, n_seq, H, c.pool, c.normalize, e->d_pool_f32.p, e->d_pool_bf16.p, s));
  ++launches;
  AUR_TRY(cudaEventRecord(e->ev[1], s));
  e->stats.tokens = T; e->stats.seqs = n_seq; e->stats.launches = launches;
  double af = 0.0;
  for (int i = 0; i < n_seq; ++i) { const double len = cu_host[i + 1] - cu_host[i]; af += 4.0 * len * len * H; }
  e->stats.attn_flops = af * c.layers;
  e->stats.gemm_flops = 2.0 * T * (3.0 * H * H + 1.0 * H * H + 2.0 * H * I) * c.layers;   // algorithmic (unpadded heads)
  e->last_tokens = T;
  return AUR_OK;
}

int check_loaded(aur_encoder* e) {
  std::lock_guard<std::mutex> g(e->mu);
  if (!e->missing.empty())
    return report_error(AUR_ERR_INVALID, "encoder parameters not loaded: %s (+%zu more)", e->missing[0].c_str(), e->missing.size() - 1);
  return AUR_OK;
}

// aur_encode's and aur_encode_append's own checks, before any device work: the parameters loaded, and the sequences one
// batch of the workspace (at most max_seqs sequences of at most max_tokens tokens in all).
int check_one_batch(aur_encoder* e, const int32_t* tokens, const int32_t* cu, int32_t n_seq) {
  const aur_encoder_config& c = e->cfg;
  int rc = check_loaded(e);
  if (rc != AUR_OK) return rc;
  if (!tokens || !cu || n_seq <= 0) return report_error(AUR_ERR_INVALID, "tokens / cu_seqlens / n_seq");
  if (n_seq > c.max_seqs) return report_error(AUR_ERR_NOMEM, "n_seq %d > max_seqs %d", n_seq, c.max_seqs);
  if (cu[0] != 0) return report_error(AUR_ERR_INVALID, "cu_seqlens[0] must be 0");
  if (cu[n_seq] > c.max_tokens) return report_error(AUR_ERR_NOMEM, "%d tokens > max_tokens %d", cu[n_seq], c.max_tokens);
  return AUR_OK;
}

bool same_config(const aur_encoder_config& a, const aur_encoder_config& b) {   // everything but the device
  return a.hidden == b.hidden && a.layers == b.layers && a.heads == b.heads && a.inter == b.inter && a.vocab == b.vocab &&
         a.max_pos == b.max_pos && a.type_vocab == b.type_vocab && a.pool == b.pool && a.normalize == b.normalize &&
         a.max_tokens == b.max_tokens && a.max_seqs == b.max_seqs && memcmp(&a.ln_eps, &b.ln_eps, sizeof(float)) == 0 &&
         a.reserved == b.reserved;
}

// The caller's packed windows: text j is sequences lo(j) .. hi(j) - 1 (one sequence per text without cu_texts).
struct Texts {
  const int32_t* tokens;
  const int32_t* cu;
  const int32_t* cu_texts;
  int32_t lo(int32_t j) const { return cu_texts ? cu_texts[j] : j; }
  int32_t hi(int32_t j) const { return cu_texts ? cu_texts[j + 1] : j + 1; }
};

// Checks of packed windows against the configuration c, before any device work: every window 1 .. max_pos long and
// within one call's token budget, every token id in the vocabulary, cu_texts well formed and ending at n_seq.
int check_texts(const aur_encoder_config& c, const Texts& in, int32_t n_seq, int32_t n_texts, int tok_budget) {
  if (in.cu[0] != 0) return report_error(AUR_ERR_INVALID, "cu_seqlens[0] must be 0");
  for (int32_t i = 0; i < n_seq; ++i) {
    const int len = in.cu[i + 1] - in.cu[i];
    if (len < 1 || len > c.max_pos) return report_error(AUR_ERR_INVALID, "sequence %d has length %d (1..%d)", i, len, c.max_pos);
    if (len > tok_budget) return report_error(AUR_ERR_NOMEM, "sequence %d has %d tokens > %d per call", i, len, tok_budget);
    for (int t = 0; t < len; ++t) {
      const int32_t id = in.tokens[in.cu[i] + t];
      if (id < 0 || id >= c.vocab) return report_error(AUR_ERR_INVALID, "token id %d out of range at sequence %d", id, i);
    }
  }
  if (in.cu_texts) {
    if (in.cu_texts[0] != 0) return report_error(AUR_ERR_INVALID, "cu_texts[0] must be 0");
    for (int32_t j = 0; j < n_texts; ++j)
      if (in.cu_texts[j + 1] <= in.cu_texts[j]) return report_error(AUR_ERR_INVALID, "text %d has no window (cu_texts must rise)", j);
    if (in.cu_texts[n_texts] != n_seq)
      return report_error(AUR_ERR_INVALID, "cu_texts[n_texts] = %d, n_seq = %d", in.cu_texts[n_texts], n_seq);
  } else if (n_texts != n_seq) {
    return report_error(AUR_ERR_INVALID, "%d texts of one window each, %d sequences", n_texts, n_seq);
  }
  return AUR_OK;
}

// Receives one batch's finished texts q[0 .. n): their bf16 rows are e->d_pool_bf16.p [0, n), their fp32 rows f32 [0, n);
// called on e's stream, under e's lock, before the batch's synchronise.
using TextSink = std::function<int(aur_encoder* e, const int32_t* q, int n, const float* f32)>;

// Texts q[0 .. nq) (already checked) through e, in order, in greedy batches of at most tok_budget tokens and seq_budget
// windows; a text's windows may span batches.  A batch with a text of several windows (or one carried in or left open)
// adds window_fold_kernel after the forward; the running sum of a text left open stays in e's carry row, and e stays
// locked until that text is finished, so no other caller of e can overwrite it.
int run_texts(aur_encoder* e, const Texts& in, const int32_t* q, int32_t nq, int tok_budget, int seq_budget, const TextSink& sink) {
  const int H = e->cfg.hidden;
  std::unique_lock<std::mutex> lk(e->mu, std::defer_lock);
  std::vector<int32_t> cu_b, wins;
  int32_t p = 0, w = nq > 0 ? in.lo(q[0]) : 0;   // next window: w, of text q[p]
  int slot = 0;                                    // the carry row an open text's sum is read from next
  while (p < nq) {
    const int32_t p0 = p;
    const bool carry_in = w != in.lo(q[p]);
    wins.clear();
    int64_t toks = 0;
    while (p < nq && static_cast<int>(wins.size()) < seq_budget && toks + (in.cu[w + 1] - in.cu[w]) <= tok_budget) {
      toks += in.cu[w + 1] - in.cu[w];
      wins.push_back(w);
      if (++w == in.hi(q[p]) && ++p < nq) w = in.lo(q[p]);
    }
    const int m = static_cast<int>(wins.size());
    const bool open = p < nq && w != in.lo(q[p]);
    const int n_closed = p - p0, n_fold = n_closed + (open ? 1 : 0);
    if (!lk.owns_lock()) lk.lock();
    AUR_TRY(cudaSetDevice(e->cfg.device));
    cu_b.assign(static_cast<size_t>(m) + 1, 0);
    int n_items = 0;
    for (int i = 0; i < m; ++i) {
      const int32_t len = in.cu[wins[i] + 1] - in.cu[wins[i]], at = cu_b[i];
      memcpy(e->h_tok.p + at, in.tokens + in.cu[wins[i]], sizeof(int32_t) * len);
      for (int t = 0; t < len; ++t) e->h_pos.p[at + t] = t;
      for (int q0 = 0; q0 < len; q0 += 128) e->h_items.p[n_items++] = AttnItem{at, len, q0, 0};
      cu_b[i + 1] = at + len;
    }
    bool fold = false;
    for (int k = 0, row = 0; k < n_fold; ++k) {
      const int32_t j = q[p0 + k], first = k == 0 ? wins[0] : in.lo(j), end = k == n_closed ? w : in.hi(j);
      e->h_fold.p[k] = FoldItem{row, row + (end - first), in.hi(j) - in.lo(j),
                              (k == 0 && carry_in ? kFoldCarryIn : 0) | (k == n_closed ? kFoldOpen : 0)};
      row += end - first;
      fold |= in.hi(j) - in.lo(j) > 1;
    }
    int rc = AUR_OK;
    if (fold) AUR_TRY(cudaMemcpyAsync(e->d_fold.p, e->h_fold.p, sizeof(FoldItem) * n_fold, cudaMemcpyHostToDevice, e->stream));
    rc = forward_locked(e, cu_b.data(), m, n_items);
    if (rc == AUR_OK && fold) {
      float* carry = e->d_fold_f32.p + static_cast<size_t>(e->cfg.max_seqs) * H;
      const cudaError_t ce = launch_window_fold(e->d_pool_f32.p, e->d_fold.p, n_fold, H, e->cfg.normalize, carry + slot * H,
                                                carry + (1 - slot) * H, e->d_fold_f32.p, e->d_pool_bf16.p, e->stream);
      if (open) slot = 1 - slot;
      if (ce != cudaSuccess) rc = report_error(AUR_ERR_CUDA, "window_fold_kernel: %s", cudaGetErrorString(ce));
      ++e->stats.launches;
    }
    if (rc == AUR_OK && n_closed > 0) rc = sink(e, q + p0, n_closed, fold ? e->d_fold_f32.p : e->d_pool_f32.p);
    // the pinned staging is reused by the next batch: the stream must be past its copies, whatever happened above
    const cudaError_t ce = cudaStreamSynchronize(e->stream);
    if (rc != AUR_OK) return rc;
    if (ce != cudaSuccess) return report_error(AUR_ERR_CUDA, "encode: %s", cudaGetErrorString(ce));
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e->ev[0], e->ev[1]);
    e->stats.total_ms = ms;
    if (!open) lk.unlock();
  }
  return AUR_OK;
}

// aur_encode_texts after its argument checks, and aur_encode with in.cu_texts = NULL (one window per text): every text
// through e's whole workspace.  out_f32 / out_bf16 are written only on success.  One output of windows that fit one
// batch (every aur_encode call that asks for one) is copied straight into the caller's buffer, behind the forward on
// e's stream, which a failed forward never gets past.  Several batches, or both outputs (the first copy could land
// before the second fails), are staged on the host and copied out once everything has succeeded.
int encode_texts(aur_encoder* e, const Texts& in, int32_t n_seq, int32_t n_texts, float* out_f32, uint16_t* out_bf16) {
  int rc = check_texts(e->cfg, in, n_seq, n_texts, e->cfg.max_tokens);
  if (rc != AUR_OK) return rc;
  const size_t H = e->cfg.hidden;
  const bool one_batch = n_seq <= e->cfg.max_seqs && in.cu[n_seq] <= e->cfg.max_tokens;
  const bool direct = one_batch && !(out_f32 && out_bf16);
  std::vector<float> f32(out_f32 && !direct ? static_cast<size_t>(n_texts) * H : 0);
  std::vector<uint16_t> bf16(out_bf16 && !direct ? static_cast<size_t>(n_texts) * H : 0);
  float* const to_f32 = direct || !out_f32 ? out_f32 : f32.data();
  uint16_t* const to_bf16 = direct || !out_bf16 ? out_bf16 : bf16.data();
  std::vector<int32_t> q(static_cast<size_t>(n_texts));
  for (int32_t j = 0; j < n_texts; ++j) q[j] = j;
  rc = run_texts(e, in, q.data(), n_texts, e->cfg.max_tokens, e->cfg.max_seqs,
                 [&](aur_encoder* enc, const int32_t* qs, int n, const float* rows) -> int {
                   const size_t at = static_cast<size_t>(qs[0]) * H, len = static_cast<size_t>(n) * H;
                   if (to_f32) AUR_TRY(cudaMemcpyAsync(to_f32 + at, rows, len * sizeof(float), cudaMemcpyDeviceToHost, enc->stream));
                   if (to_bf16) AUR_TRY(cudaMemcpyAsync(to_bf16 + at, enc->d_pool_bf16.p, len * 2, cudaMemcpyDeviceToHost, enc->stream));
                   return AUR_OK;
                 });
  if (rc != AUR_OK) return rc;
  if (!f32.empty()) memcpy(out_f32, f32.data(), f32.size() * sizeof(float));
  if (!bf16.empty()) memcpy(out_bf16, bf16.data(), bf16.size() * 2);
  return AUR_OK;
}

// aur_encode_pair_cosines after aur_encode_texts' own checks, with n_texts > 0: every text through e's whole workspace
// as encode_texts runs it, each batch's fp32 text rows copied device to device into this call's vecs [n_texts, hidden]
// (per call: run_texts drops e's lock between batches, so nothing of e's may hold them across batches).  The sink of the
// batch that finishes the last text uploads the pairs, launches cosine_gather_kernel and copies the cosines (and the
// vectors) back, all on e's stream before that batch's synchronise.  Outputs are staged and written only on success.
int pair_cosines(aur_encoder* e, const Texts& in, int32_t n_seq, int32_t n_texts, const int32_t* pair_a,
                 const int32_t* pair_b, int64_t n_pairs, int32_t clamp, double* cos_out, float* vec_out) {
  int rc = check_texts(e->cfg, in, n_seq, n_texts, e->cfg.max_tokens);
  if (rc != AUR_OK) return rc;
  for (int64_t p = 0; p < n_pairs; ++p)
    if (pair_a[p] < 0 || pair_a[p] >= n_texts || pair_b[p] < 0 || pair_b[p] >= n_texts)
      return report_error(AUR_ERR_INVALID, "pair %lld is (%d, %d): indices must be in 0 .. %d", static_cast<long long>(p),
                          pair_a[p], pair_b[p], n_texts - 1);
  if (n_pairs == 0 && !vec_out) return AUR_OK;
  const size_t H = e->cfg.hidden, np = static_cast<size_t>(n_pairs);
  AUR_TRY(cudaSetDevice(e->cfg.device));
  DevBuf<float> d_vec;
  DevBuf<int32_t> d_pairs;   // pair_a, then pair_b
  DevBuf<double> d_cos;
  AUR_TRY(d_vec.reserve(static_cast<size_t>(n_texts) * H));
  AUR_TRY(d_pairs.reserve(2 * np));
  AUR_TRY(d_cos.reserve(np));
  std::vector<double> cos_h(np);
  std::vector<float> vec_h(vec_out ? static_cast<size_t>(n_texts) * H : 0);
  std::vector<int32_t> q(static_cast<size_t>(n_texts));
  for (int32_t j = 0; j < n_texts; ++j) q[j] = j;
  rc = run_texts(e, in, q.data(), n_texts, e->cfg.max_tokens, e->cfg.max_seqs,
                 [&](aur_encoder* enc, const int32_t* qs, int n, const float* rows) -> int {
                   cudaStream_t s = enc->stream;
                   AUR_TRY(cudaMemcpyAsync(d_vec.p + static_cast<size_t>(qs[0]) * H, rows, static_cast<size_t>(n) * H * sizeof(float),
                                           cudaMemcpyDeviceToDevice, s));
                   if (qs[n - 1] != n_texts - 1) return AUR_OK;   // texts finish in order: the last one is the call's end
                   if (np > 0) {
                     AUR_TRY(cudaMemcpyAsync(d_pairs.p, pair_a, np * sizeof(int32_t), cudaMemcpyHostToDevice, s));
                     AUR_TRY(cudaMemcpyAsync(d_pairs.p + np, pair_b, np * sizeof(int32_t), cudaMemcpyHostToDevice, s));
                     AUR_TRY(launch_cosine_gather(d_vec.p, d_pairs.p, d_pairs.p + np, n_pairs, static_cast<int>(H), clamp, d_cos.p, s));
                     ++enc->stats.launches;
                     AUR_TRY(cudaMemcpyAsync(cos_h.data(), d_cos.p, np * sizeof(double), cudaMemcpyDeviceToHost, s));
                   }
                   if (vec_out) AUR_TRY(cudaMemcpyAsync(vec_h.data(), d_vec.p, vec_h.size() * sizeof(float), cudaMemcpyDeviceToHost, s));
                   return AUR_OK;
                 });
  if (rc != AUR_OK) return rc;
  if (np > 0) memcpy(cos_out, cos_h.data(), np * sizeof(double));
  if (vec_out) memcpy(vec_out, vec_h.data(), vec_h.size() * sizeof(float));
  return AUR_OK;
}

// aur_encode_append_texts_multi, aur_encode_append_multi with in.cu_texts = NULL (one window per text), and
// aur_encode_append, which is that with n = 1 after its one-batch checks.
int append_texts_multi(aur_encoder* const* encs, aur_index* const* shards, int32_t n, const Texts& in, int32_t n_seq,
                       int32_t n_texts, const int64_t* ids, const int32_t* user_codes, const int32_t* org_codes,
                       int32_t max_tokens_per_call, int32_t max_seqs_per_call) {
  constexpr int kMaxShards = 64;
  if (!encs || !shards) return report_error(AUR_ERR_INVALID, "null argument");
  if (n < 1 || n > kMaxShards) return report_error(AUR_ERR_INVALID, "n must be in 1 .. %d", kMaxShards);
  for (int32_t s = 0; s < n; ++s)
    if (!shards[s] || !encs[s]) return report_error(AUR_ERR_INVALID, "shard or encoder %d is NULL", s);
  std::vector<aur_index*> order(shards, shards + n);
  std::sort(order.begin(), order.end(), std::less<aur_index*>());
  if (std::adjacent_find(order.begin(), order.end()) != order.end()) return report_error(AUR_ERR_INVALID, "a shard is listed twice");
  const aur_encoder_config& c = encs[0]->cfg;   // fixed at open
  for (int32_t s = 0; s < n; ++s) {
    aur_encoder* e = encs[s];
    if (!same_config(e->cfg, c)) return report_error(AUR_ERR_INVALID, "encoder %d has another configuration than encoder 0", s);
    {
      std::lock_guard<std::mutex> g(e->mu);
      if (!e->missing.empty())
        return report_error(AUR_ERR_INVALID, "encoder %d parameters not loaded: %s (+%zu more)", s, e->missing[0].c_str(),
                            e->missing.size() - 1);
    }
    if (e->cfg.device != index_device(shards[s]))
      return report_error(AUR_ERR_INVALID, "encoder %d is on device %d, its shard on device %d", s, e->cfg.device, index_device(shards[s]));
  }
  std::vector<aur_stats> st(static_cast<size_t>(n));
  for (int32_t s = 0; s < n; ++s) {
    int rc = aur_get_stats(shards[s], &st[s]);
    if (rc != AUR_OK) return rc;
    if (st[s].dim != c.hidden || st[s].dtype == AUR_F32)   // (an int8 shard quantizes the bf16 rows as it adds them)
      return report_error(AUR_ERR_INVALID, "shard %d is %d-d dtype %d; the encoder produces %d-d bf16", s, st[s].dim, st[s].dtype, c.hidden);
  }
  if (max_tokens_per_call < 0 || max_tokens_per_call > c.max_tokens || max_seqs_per_call < 0 || max_seqs_per_call > c.max_seqs)
    return report_error(AUR_ERR_INVALID, "per-call limits must be 0 .. the workspace (%d tokens, %d sequences)", c.max_tokens, c.max_seqs);
  const int tok_budget = max_tokens_per_call ? max_tokens_per_call : c.max_tokens;
  const int seq_budget = max_seqs_per_call ? max_seqs_per_call : c.max_seqs;
  if (n_seq < 0 || n_texts < 0) return report_error(AUR_ERR_INVALID, "n_seq / n_texts < 0");
  if (n_seq == 0 && n_texts == 0) return AUR_OK;
  if (!in.tokens || !in.cu || !ids) return report_error(AUR_ERR_INVALID, "tokens, cu_seqlens and ids are required");
  int rc = check_texts(c, in, n_seq, n_texts, tok_budget);
  if (rc != AUR_OK) return rc;
  std::vector<std::vector<int32_t>> share(static_cast<size_t>(n));
  for (int32_t j = 0; j < n_texts; ++j) {
    if (ids[j] < 0) return report_error(AUR_ERR_INVALID, "ids must be >= 0");
    share[static_cast<size_t>(ids[j] % n)].push_back(j);
  }
  for (int32_t s = 0; s < n; ++s)
    if (st[s].rows + static_cast<int64_t>(share[s].size()) > st[s].capacity)
      return report_error(AUR_ERR_NOMEM, "shard %d full: %lld + %zu > capacity %lld (aur_compact reclaims tombstones)", s,
                          static_cast<long long>(st[s].rows), share[s].size(), static_cast<long long>(st[s].capacity));
  // each shard's share, in input order, in greedy workspace batches; the shards run on their own host threads
  std::vector<int> rcs(static_cast<size_t>(n), AUR_OK);
  std::vector<std::string> errs(static_cast<size_t>(n));
  auto run = [&](int32_t s) {
    std::vector<int64_t> id_b;
    std::vector<int32_t> u_b, o_b;
    const int r = run_texts(encs[s], in, share[s].data(), static_cast<int32_t>(share[s].size()), tok_budget, seq_budget,
                            [&](aur_encoder* e, const int32_t* q, int m, const float*) -> int {
                              id_b.resize(static_cast<size_t>(m));
                              if (user_codes) u_b.resize(static_cast<size_t>(m));
                              if (org_codes) o_b.resize(static_cast<size_t>(m));
                              for (int i = 0; i < m; ++i) {
                                id_b[i] = ids[q[i]];
                                if (user_codes) u_b[i] = user_codes[q[i]];
                                if (org_codes) o_b[i] = org_codes[q[i]];
                              }
                              // the rows stay in HBM: the shard copies them device-to-device on the encoder's stream
                              return aur_add_dev(shards[s], e->d_pool_bf16.p, id_b.data(), user_codes ? u_b.data() : nullptr,
                                                 org_codes ? o_b.data() : nullptr, m, e->stream);
                            });
    if (r != AUR_OK) {
      rcs[s] = r;
      const char* msg = aur_last_error();
      errs[s] = msg ? msg : "";
    }
  };
  std::vector<std::thread> th;
  for (int32_t s = 1; s < n; ++s)
    if (!share[s].empty()) th.emplace_back(run, s);
  run(0);
  for (std::thread& t : th) t.join();
  for (int32_t s = 0; s < n; ++s)
    if (rcs[s] != AUR_OK) return report_error(rcs[s], "shard %d: %s", s, errs[s].c_str());
  return AUR_OK;
}

}  // namespace

extern "C" {

int aur_encoder_open(const aur_encoder_config* cfg, aur_encoder** out) {
  if (!cfg || !out) return report_error(AUR_ERR_INVALID, "null argument");
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return report_error(AUR_ERR_NO_DEVICE, "no CUDA device: aurora_b200 has no CPU path");
  if (cfg->device < 0 || cfg->device >= ndev) return report_error(AUR_ERR_INVALID, "device %d of %d", cfg->device, ndev);
  const int H = cfg->hidden, I = cfg->inter;
  if (H <= 0 || cfg->heads <= 0 || H % cfg->heads || (H / cfg->heads != 64 && H / cfg->heads != 32))
    return report_error(AUR_ERR_UNSUPPORTED, "head dim must be 64 or 32 (hidden %d, heads %d)", H, cfg->heads);
  if (H % 128 || I % 128 || H > 1024) return report_error(AUR_ERR_UNSUPPORTED, "hidden / inter must be multiples of 128, hidden <= 1024");
  if (cfg->max_pos < 1 || cfg->max_pos > 512) return report_error(AUR_ERR_UNSUPPORTED, "max_pos must be 1..512");
  if (cfg->layers < 1 || cfg->vocab < 1 || cfg->type_vocab < 1 || cfg->max_tokens < 1 || cfg->max_seqs < 1)
    return report_error(AUR_ERR_INVALID, "layers / vocab / type_vocab / max_tokens / max_seqs must be positive");
  AUR_TRY(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  AUR_TRY(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9) return report_error(AUR_ERR_UNSUPPORTED, "sm_%d%d device: this library is built for sm_90a only", prop.major, prop.minor);
  std::unique_ptr<aur_encoder> e(new aur_encoder());
  e->cfg = *cfg;
  e->sm_count = prop.multiProcessorCount;
  e->rows_pad = round_up(cfg->max_tokens, 256) + 512;   // + one full key window past the last sequence
  e->cta_group = cfg->reserved == 1 ? 1 : 2;            // reserved = 1 selects the single-CTA GEMM (bring-up)
  e->dh = H / cfg->heads;
  e->hp = cfg->heads * 64;     // head dim 32 is zero-padded to 64: q.k and P.V are unchanged by zero dims
  e->bn = (H % 256 == 0 && I % 256 == 0 && e->hp % 256 == 0) ? 256 : 128;
  e->layers.resize(cfg->layers);
  int rc = AUR_OK;
  auto A = [&](auto& b, size_t n) { if (rc == AUR_OK) rc = dev_alloc(b, n); };
  for_each_param(e.get(), A);
  const size_t R = e->rows_pad;
  A(e->x, R * H); A(e->y, R * H); A(e->qkv, R * 3 * e->hp); A(e->ctx, R * e->hp); A(e->inter, R * I);
  A(e->d_tok, cfg->max_tokens); A(e->d_pos, cfg->max_tokens); A(e->d_cu, cfg->max_seqs + 1);
  e->max_items = cfg->max_seqs * 4;
  A(e->d_items, e->max_items);
  A(e->d_pool_f32, static_cast<size_t>(cfg->max_seqs) * H); A(e->d_pool_bf16, static_cast<size_t>(cfg->max_seqs) * H);
  A(e->d_fold_f32, static_cast<size_t>(cfg->max_seqs + 2) * H); A(e->d_fold, cfg->max_seqs);
  if (rc != AUR_OK) return rc;
  if (e->h_tok.reserve(cfg->max_tokens, cudaHostAllocDefault) != cudaSuccess ||
      e->h_pos.reserve(cfg->max_tokens, cudaHostAllocDefault) != cudaSuccess ||
      e->h_items.reserve(e->max_items, cudaHostAllocDefault) != cudaSuccess ||
      e->h_fold.reserve(cfg->max_seqs, cudaHostAllocDefault) != cudaSuccess)
    return report_error(AUR_ERR_NOMEM, "pinned staging allocation failed");
  if (e->stream.create(cudaStreamNonBlocking) != cudaSuccess) return report_error(AUR_ERR_CUDA, "cudaStreamCreate failed");
  for (Event& ev : e->ev)
    if (ev.create() != cudaSuccess) return report_error(AUR_ERR_CUDA, "cudaEventCreate failed");
  // tensor maps: activations are A operands (box 128 rows), weights B operands (box bn rows)
  const int Ri = static_cast<int>(R);
  const int HP = e->hp;
  if ((rc = make_tmap(&e->tm_x, e->x.p, H, Ri, 128)) || (rc = make_tmap(&e->tm_ctx, e->ctx.p, HP, Ri, 128)) ||
      (rc = make_tmap(&e->tm_inter, e->inter.p, I, Ri, 128)) || (rc = make_tmap(&e->tm_qkv, e->qkv.p, 3 * HP, Ri, 128)))
    return rc;
  for (Layer& l : e->layers) {
    if ((rc = make_tmap(&l.tm_wqkv, l.wqkv.p, H, 3 * HP, e->bn / e->cta_group)) ||
        (rc = make_tmap(&l.tm_wo, l.wo.p, HP, H, e->bn / e->cta_group)) ||
        (rc = make_tmap(&l.tm_wi, l.wi.p, H, I, e->bn / e->cta_group)) ||
        (rc = make_tmap(&l.tm_wo2, l.wo2.p, I, H, e->bn / e->cta_group)))
      return rc;
  }
  e->missing = {"word_emb", "pos_emb", "type_emb", "emb_ln_g", "emb_ln_b"};
  for (int l = 0; l < cfg->layers; ++l)
    for (const char* leaf : {"wqkv", "bqkv", "wo", "bo", "ln1_g", "ln1_b", "wi", "bi", "wo2", "bo2", "ln2_g", "ln2_b"})
      e->missing.push_back("l" + std::to_string(l) + "." + leaf);
  *out = e.release();
  return AUR_OK;
}

int aur_encoder_close(aur_encoder* e) {
  if (!e) return AUR_OK;
  { std::lock_guard<std::mutex> g(e->mu); cudaSetDevice(e->cfg.device); cudaStreamSynchronize(e->stream); }
  delete e;
  return AUR_OK;
}

int aur_encoder_load(aur_encoder* e, const char* name, const float* data, int64_t count) {
  if (!e || !name || !data) return report_error(AUR_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> g(e->mu);
  AUR_TRY(cudaSetDevice(e->cfg.device));
  ParamSlot slot{};
  if (!find_param(e, name, &slot)) return report_error(AUR_ERR_INVALID, "unknown parameter '%s'", name);
  if (slot.count != count) return report_error(AUR_ERR_INVALID, "parameter '%s' has %lld elements, expected %lld", name,
                                               static_cast<long long>(count), static_cast<long long>(slot.count));
  std::vector<float> padded;
  int64_t n_up = count;
  if (slot.pad) {   // head dim 32: spread each head's 32 rows / columns over a 64-wide slot, zeros between
    const int64_t H = e->cfg.hidden, HP = e->hp, nh = e->cfg.heads, dh = e->dh;
    if (slot.pad == 1) {
      const int64_t inner = slot.bf16 ? H : 1;          // wqkv rows have H columns; bqkv is a vector
      padded.assign(static_cast<size_t>(3 * HP * inner), 0.f);
      for (int64_t part = 0; part < 3; ++part)
        for (int64_t h = 0; h < nh; ++h)
          for (int64_t d = 0; d < dh; ++d)
            memcpy(&padded[((part * nh + h) * 64 + d) * inner], &data[((part * nh + h) * dh + d) * inner], sizeof(float) * inner);
    } else {
      padded.assign(static_cast<size_t>(H * HP), 0.f);
      for (int64_t r = 0; r < H; ++r)
        for (int64_t h = 0; h < nh; ++h)
          memcpy(&padded[r * HP + h * 64], &data[r * H + h * dh], sizeof(float) * dh);
    }
    data = padded.data();
    n_up = static_cast<int64_t>(padded.size());
  }
  if (slot.bf16) {
    AUR_TRY(e->d_stage.reserve(static_cast<size_t>(n_up)));
    AUR_TRY(cudaMemcpyAsync(e->d_stage.p, data, sizeof(float) * n_up, cudaMemcpyHostToDevice, e->stream));
    AUR_TRY(launch_f32_to_bf16(e->d_stage.p, static_cast<__nv_bfloat16*>(slot.dst), n_up, e->stream));
  } else {
    AUR_TRY(cudaMemcpyAsync(slot.dst, data, sizeof(float) * n_up, cudaMemcpyHostToDevice, e->stream));
  }
  AUR_TRY(cudaStreamSynchronize(e->stream));
  for (size_t i = 0; i < e->missing.size(); ++i)
    if (e->missing[i] == name) { e->missing.erase(e->missing.begin() + i); break; }
  return AUR_OK;
}

int aur_encode(aur_encoder* e, const int32_t* tokens, const int32_t* cu, int32_t n_seq, float* out_f32, uint16_t* out_bf16) {
  if (!e) return report_error(AUR_ERR_INVALID, "null encoder");
  const int rc = check_one_batch(e, tokens, cu, n_seq);
  if (rc != AUR_OK) return rc;
  return encode_texts(e, Texts{tokens, cu, nullptr}, n_seq, n_seq, out_f32, out_bf16);
}

int aur_encode_append(aur_encoder* e, aur_index* ix, const int32_t* tokens, const int32_t* cu, int32_t n_seq,
                      const int64_t* ids, const int32_t* user_codes, const int32_t* org_codes) {
  if (!e || !ix || !ids) return report_error(AUR_ERR_INVALID, "null argument");
  const int rc = check_one_batch(e, tokens, cu, n_seq);
  if (rc != AUR_OK) return rc;
  return append_texts_multi(&e, &ix, 1, Texts{tokens, cu, nullptr}, n_seq, n_seq, ids, user_codes, org_codes, 0, 0);
}

int aur_encoder_replicate(aur_encoder* src, int32_t device, aur_encoder** out) {
  if (!src || !out) return report_error(AUR_ERR_INVALID, "null argument");
  *out = nullptr;
  std::lock_guard<std::mutex> g(src->mu);   // no upload or close of src while its bits are read
  if (!src->missing.empty())
    return report_error(AUR_ERR_INVALID, "encoder parameters not loaded: %s (+%zu more)", src->missing[0].c_str(), src->missing.size() - 1);
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev)
    return report_error(AUR_ERR_INVALID, "device %d of %d", device, ndev);
  aur_encoder_config cfg = src->cfg;
  cfg.device = device;
  aur_encoder* r = nullptr;
  int rc = aur_encoder_open(&cfg, &r);
  if (rc != AUR_OK) return rc;
  std::vector<const void*> from;
  std::vector<size_t> bytes;
  std::vector<void*> to;
  for_each_param(src, [&](auto& b, size_t n) { from.push_back(b.p); bytes.push_back(n * sizeof(*b.p)); });
  for_each_param(r, [&](auto& b, size_t) { to.push_back(b.p); });
  const cudaError_t ce = [&]() -> cudaError_t {
    for (size_t i = 0; i < to.size(); ++i)   // staged by the driver when the devices are not peers
      AUR_CU_RET(cudaMemcpyPeerAsync(to[i], device, from[i], src->cfg.device, bytes[i], r->stream));
    return cudaStreamSynchronize(r->stream);
  }();
  if (ce != cudaSuccess) {
    aur_encoder_close(r);
    return report_error(AUR_ERR_CUDA, "encoder replica on device %d: %s", device, cudaGetErrorString(ce));
  }
  r->missing.clear();
  *out = r;
  return AUR_OK;
}

int aur_encode_texts(aur_encoder* e, const int32_t* tokens, const int32_t* cu, int32_t n_seq, const int32_t* cu_texts,
                     int32_t n_texts, float* out_f32, uint16_t* out_bf16) {
  if (!e) return report_error(AUR_ERR_INVALID, "null encoder");
  const int rc = check_loaded(e);
  if (rc != AUR_OK) return rc;
  if (n_seq < 0 || n_texts < 0) return report_error(AUR_ERR_INVALID, "n_seq / n_texts < 0");
  if (n_texts == 0 && n_seq == 0) return AUR_OK;
  if (!tokens || !cu || !cu_texts) return report_error(AUR_ERR_INVALID, "tokens, cu_seqlens and cu_texts are required");
  return encode_texts(e, Texts{tokens, cu, cu_texts}, n_seq, n_texts, out_f32, out_bf16);
}

int aur_encode_pair_cosines(aur_encoder* e, const int32_t* tokens, const int32_t* cu, int32_t n_seq, const int32_t* cu_texts,
                            int32_t n_texts, const int32_t* pair_a, const int32_t* pair_b, int64_t n_pairs, int32_t clamp,
                            double* cos_out, float* vec_out) {
  if (!e) return report_error(AUR_ERR_INVALID, "null encoder");
  const int rc = check_loaded(e);
  if (rc != AUR_OK) return rc;
  if (n_seq < 0 || n_texts < 0) return report_error(AUR_ERR_INVALID, "n_seq / n_texts < 0");
  if (n_pairs < 0) return report_error(AUR_ERR_INVALID, "n_pairs < 0");
  if (n_pairs > 0 && (!pair_a || !pair_b || !cos_out)) return report_error(AUR_ERR_INVALID, "pair_a, pair_b and cos_out are required");
  if (clamp != 0 && clamp != 1) return report_error(AUR_ERR_INVALID, "clamp must be 0 or 1");
  if (n_texts == 0 && n_seq == 0) {
    if (n_pairs > 0) return report_error(AUR_ERR_INVALID, "%lld pairs over no texts", static_cast<long long>(n_pairs));
    return AUR_OK;
  }
  if (!tokens || !cu || !cu_texts) return report_error(AUR_ERR_INVALID, "tokens, cu_seqlens and cu_texts are required");
  return pair_cosines(e, Texts{tokens, cu, cu_texts}, n_seq, n_texts, pair_a, pair_b, n_pairs, clamp, cos_out, vec_out);
}

int aur_encode_append_texts_multi(aur_encoder* const* encs, aur_index* const* shards, int32_t n, const int32_t* tokens,
                                  const int32_t* cu, int32_t n_seq, const int32_t* cu_texts, int32_t n_texts,
                                  const int64_t* ids, const int32_t* user_codes, const int32_t* org_codes,
                                  int32_t max_tokens_per_call, int32_t max_seqs_per_call) {
  if (!cu_texts && n_texts > 0) return report_error(AUR_ERR_INVALID, "cu_texts is required");
  return append_texts_multi(encs, shards, n, Texts{tokens, cu, cu_texts}, n_seq, n_texts, ids, user_codes, org_codes,
                            max_tokens_per_call, max_seqs_per_call);
}

int aur_encode_append_multi(aur_encoder* const* encs, aur_index* const* shards, int32_t n, const int32_t* tokens,
                            const int32_t* cu, int32_t n_seq, const int64_t* ids, const int32_t* user_codes,
                            const int32_t* org_codes, int32_t max_tokens_per_call, int32_t max_seqs_per_call) {
  return append_texts_multi(encs, shards, n, Texts{tokens, cu, nullptr}, n_seq, n_seq, ids, user_codes, org_codes,
                            max_tokens_per_call, max_seqs_per_call);
}

int aur_encoder_get_stats(aur_encoder* e, aur_encoder_stats* out) {
  if (!e || !out) return report_error(AUR_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> g(e->mu);
  *out = e->stats;
  return AUR_OK;
}

int aur_debug_encoder_hidden(aur_encoder* e, uint16_t* out, int64_t count) {
  if (!e || !out) return report_error(AUR_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> g(e->mu);
  AUR_TRY(cudaSetDevice(e->cfg.device));
  if (count != e->last_tokens * e->cfg.hidden) return report_error(AUR_ERR_INVALID, "count must be tokens * hidden of the last call");
  AUR_TRY(cudaStreamSynchronize(e->stream));
  AUR_TRY(cudaMemcpy(out, e->x.p, count * 2, cudaMemcpyDeviceToHost));
  return AUR_OK;
}

int aur_debug_gemm(int32_t device, const uint16_t* a, const uint16_t* w, const float* bias, const uint16_t* resid,
                   int32_t m, int32_t n, int32_t k, int32_t epi, int32_t cta_group, uint16_t* out, float* ms_out) {
  if (!a || !w || !bias || !out || m <= 0) return report_error(AUR_ERR_INVALID, "null argument");
  if (n % 128 || k % 64 || epi < 0 || epi > 2 || (epi == kEpiBiasResid && !resid) || (cta_group != 1 && cta_group != 2))
    return report_error(AUR_ERR_UNSUPPORTED, "n %% 128, k %% 64, epi 0..2, cta_group 1..2");
  AUR_TRY(cudaSetDevice(device));
  cudaDeviceProp prop;
  AUR_TRY(cudaGetDeviceProperties(&prop, device));
  const int m_pad = round_up(m, 128 * cta_group), bn = n % 256 == 0 ? 256 : 128;
  DevBuf<__nv_bfloat16> da, dw, dr, dout; DevBuf<float> db;   // freed on return (cudaFree waits for the device)
  int rc = AUR_OK;
  auto A = [&](auto& b, size_t cnt) { if (rc == AUR_OK) rc = dev_alloc(b, cnt); };
  A(da, static_cast<size_t>(m_pad) * k); A(dw, static_cast<size_t>(n) * k); A(dr, static_cast<size_t>(m_pad) * n);
  A(dout, static_cast<size_t>(m_pad) * n); A(db, n);
  if (rc) return rc;
  cudaMemcpy(da.p, a, static_cast<size_t>(m) * k * 2, cudaMemcpyHostToDevice);
  cudaMemcpy(dw.p, w, static_cast<size_t>(n) * k * 2, cudaMemcpyHostToDevice);
  cudaMemcpy(db.p, bias, sizeof(float) * n, cudaMemcpyHostToDevice);
  if (resid) cudaMemcpy(dr.p, resid, static_cast<size_t>(m) * n * 2, cudaMemcpyHostToDevice);
  CUtensorMap tm_a, tm_w;
  if ((rc = make_tmap(&tm_a, da.p, k, m_pad, 128)) || (rc = make_tmap(&tm_w, dw.p, k, n, bn / cta_group))) return rc;
  GemmParams p{};
  p.bias = db.p; p.resid = dr.p; p.ldr = n; p.out = dout.p; p.ldo = n;
  p.m_tiles = m_pad / (128 * cta_group); p.n_tiles = n / bn; p.k_blocks = k / 64;
  Event e0, e1;
  e0.create(); e1.create();
  cudaError_t ce = cudaSuccess;
  for (int rep = 0; rep < 3 && ce == cudaSuccess; ++rep) {   // last repetition is the timed one
    cudaEventRecord(e0, nullptr);
    ce = gemm_tc_launch(cta_group, bn, epi, prop.multiProcessorCount, &tm_a, &tm_w, p, nullptr);
    cudaEventRecord(e1, nullptr);
  }
  if (ce == cudaSuccess) ce = cudaDeviceSynchronize();
  float ms = 0.f;
  if (ce == cudaSuccess) cudaEventElapsedTime(&ms, e0, e1);
  if (ce != cudaSuccess) return report_error(AUR_ERR_CUDA, "gemm: %s", cudaGetErrorString(ce));
  ce = cudaMemcpy(out, dout.p, static_cast<size_t>(m) * n * 2, cudaMemcpyDeviceToHost);
  if (ce != cudaSuccess) return report_error(AUR_ERR_CUDA, "gemm d2h: %s", cudaGetErrorString(ce));
  if (ms_out) *ms_out = ms;
  return AUR_OK;
}

int aur_debug_attention(int32_t device, const uint16_t* qkv, const int32_t* cu, int32_t n_seq, int32_t heads,
                        int32_t hidden, uint16_t* ctx, float* ms_out) {
  if (!qkv || !cu || !ctx || n_seq <= 0) return report_error(AUR_ERR_INVALID, "null argument");
  if (heads <= 0 || hidden != heads * 64) return report_error(AUR_ERR_UNSUPPORTED, "head dim must be 64");
  AUR_TRY(cudaSetDevice(device));
  cudaDeviceProp prop;
  AUR_TRY(cudaGetDeviceProperties(&prop, device));
  const int T = cu[n_seq], rows = round_up(T, 128) + 512;
  std::vector<AttnItem> items;
  for (int i = 0; i < n_seq; ++i) {
    const int len = cu[i + 1] - cu[i];
    if (len < 1 || len > 512) return report_error(AUR_ERR_INVALID, "sequence length %d", len);
    for (int q0 = 0; q0 < len; q0 += 128) items.push_back(AttnItem{cu[i], len, q0, 0});
  }
  DevBuf<__nv_bfloat16> dq, dc; DevBuf<AttnItem> di;   // freed on return (cudaFree waits for the device)
  int rc = AUR_OK;
  auto A = [&](auto& b, size_t cnt) { if (rc == AUR_OK) rc = dev_alloc(b, cnt); };
  A(dq, static_cast<size_t>(rows) * 3 * hidden); A(dc, static_cast<size_t>(rows) * hidden); A(di, items.size());
  if (rc) return rc;
  cudaMemcpy(dq.p, qkv, static_cast<size_t>(T) * 3 * hidden * 2, cudaMemcpyHostToDevice);
  cudaMemcpy(di.p, items.data(), sizeof(AttnItem) * items.size(), cudaMemcpyHostToDevice);
  CUtensorMap tm;
  if ((rc = make_tmap(&tm, dq.p, 3 * hidden, rows, 128))) return rc;
  AttnParams ap{};
  ap.items = di.p; ap.n_items = static_cast<int>(items.size()); ap.heads = heads; ap.hidden = hidden; ap.ctx = dc.p; ap.ld_ctx = hidden;
  ap.scale_log2e = 1.4426950408889634f / 8.0f;
  Event e0, e1;
  e0.create(); e1.create();
  cudaError_t ce = cudaSuccess;
  for (int rep = 0; rep < 3 && ce == cudaSuccess; ++rep) {
    cudaEventRecord(e0, nullptr);
    ce = attn_tc_launch(&tm, ap, nullptr);
    cudaEventRecord(e1, nullptr);
  }
  if (ce == cudaSuccess) ce = cudaDeviceSynchronize();
  float ms = 0.f;
  if (ce == cudaSuccess) cudaEventElapsedTime(&ms, e0, e1);
  if (ce != cudaSuccess) return report_error(AUR_ERR_CUDA, "attention: %s", cudaGetErrorString(ce));
  ce = cudaMemcpy(ctx, dc.p, static_cast<size_t>(T) * hidden * 2, cudaMemcpyDeviceToHost);
  if (ce != cudaSuccess) return report_error(AUR_ERR_CUDA, "attention d2h: %s", cudaGetErrorString(ce));
  if (ms_out) *ms_out = ms;
  return AUR_OK;
}

}  // extern "C"
