// Host runtime of the text encoder behind the C ABI (include/aurora_b200.h, "text encoder").
// Owns the bf16 parameters and one activation workspace in HBM:
//   x, y   [max_tokens_pad, H]    residual stream / pre-LayerNorm sum
//   qkv    [max_tokens_pad, 3H]   packed projections (attention reads Q, K, V tiles from it by TMA)
//   ctx    [max_tokens_pad, H]    attention output
//   inter  [max_tokens_pad, I]    FFN activation
// and the TMA descriptors over them (activations as GEMM A operands, weights as B operands).
// A forward is 2 + 7*L + 1 kernel launches on one stream; no CPU compute path exists.
#include <algorithm>
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>
#include <string>
#include <vector>

#include "../../include/aurora_b200.h"
#include "internal.h"

using namespace aur;

#define ENC_TRY(expr)                                                                                  \
  do {                                                                                                 \
    cudaError_t e_ = (expr);                                                                           \
    if (e_ != cudaSuccess)                                                                             \
      return report_error(AUR_ERR_CUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); \
  } while (0)

namespace {

struct Layer {
  __nv_bfloat16 *wqkv = nullptr, *wo = nullptr, *wi = nullptr, *wo2 = nullptr;
  float *bqkv = nullptr, *bo = nullptr, *bi = nullptr, *bo2 = nullptr;
  float *ln1_g = nullptr, *ln1_b = nullptr, *ln2_g = nullptr, *ln2_b = nullptr;
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
  cudaStream_t stream = nullptr;
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  __nv_bfloat16 *word = nullptr, *pos = nullptr, *type = nullptr;
  float *emb_g = nullptr, *emb_b = nullptr;
  std::vector<Layer> layers;
  std::vector<std::string> missing;   // parameter names not loaded yet
  __nv_bfloat16 *x = nullptr, *y = nullptr, *qkv = nullptr, *ctx = nullptr, *inter = nullptr;
  CUtensorMap tm_x, tm_ctx, tm_inter, tm_qkv;       // loads: box {64, 128}
  int32_t *d_tok = nullptr, *d_pos = nullptr, *d_cu = nullptr;
  AttnItem* d_items = nullptr;
  int max_items = 0;
  float* d_pool_f32 = nullptr;
  __nv_bfloat16* d_pool_bf16 = nullptr;
  float* d_stage = nullptr; size_t stage_elems = 0;   // fp32 staging for parameter upload
  int32_t *h_tok = nullptr, *h_pos = nullptr;          // pinned
  AttnItem* h_items = nullptr;
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
int dev_alloc(T** p, size_t n) {
  ENC_TRY(cudaMalloc(reinterpret_cast<void**>(p), n * sizeof(T)));
  ENC_TRY(cudaMemset(*p, 0, n * sizeof(T)));
  return AUR_OK;
}

void free_all(aur_encoder* e) {
  cudaSetDevice(e->cfg.device);
  auto f = [](auto*& p) { if (p) cudaFree(p); p = nullptr; };
  f(e->word); f(e->pos); f(e->type); f(e->emb_g); f(e->emb_b);
  for (Layer& l : e->layers) {
    f(l.wqkv); f(l.wo); f(l.wi); f(l.wo2); f(l.bqkv); f(l.bo); f(l.bi); f(l.bo2);
    f(l.ln1_g); f(l.ln1_b); f(l.ln2_g); f(l.ln2_b);
  }
  f(e->x); f(e->y); f(e->qkv); f(e->ctx); f(e->inter);
  f(e->d_tok); f(e->d_pos); f(e->d_cu); f(e->d_items); f(e->d_pool_f32); f(e->d_pool_bf16); f(e->d_stage);
  if (e->h_tok) cudaFreeHost(e->h_tok);
  if (e->h_pos) cudaFreeHost(e->h_pos);
  if (e->h_items) cudaFreeHost(e->h_items);
  for (auto& ev : e->ev) if (ev) cudaEventDestroy(ev);
  if (e->stream) cudaStreamDestroy(e->stream);
}

// pad: 0 none; 1 rows are [3][heads][dh] -> [3][heads][64] (wqkv / bqkv); 2 columns are [heads][dh] -> [heads][64] (wo)
struct ParamSlot { void* dst; int64_t count; bool bf16; int pad; };

// Resolve a parameter name to its device buffer.
bool find_param(aur_encoder* e, const std::string& name, ParamSlot* out) {
  const aur_encoder_config& c = e->cfg;
  const int64_t H = c.hidden, I = c.inter;
  if (name == "word_emb") { *out = {e->word, static_cast<int64_t>(c.vocab) * H, true, 0}; return true; }
  if (name == "pos_emb") { *out = {e->pos, static_cast<int64_t>(c.max_pos) * H, true, 0}; return true; }
  if (name == "type_emb") { *out = {e->type, static_cast<int64_t>(c.type_vocab) * H, true, 0}; return true; }
  if (name == "emb_ln_g") { *out = {e->emb_g, H, false, 0}; return true; }
  if (name == "emb_ln_b") { *out = {e->emb_b, H, false, 0}; return true; }
  int l = -1; char leaf[32] = {0};
  if (sscanf(name.c_str(), "l%d.%31s", &l, leaf) != 2 || l < 0 || l >= c.layers) return false;
  Layer& L = e->layers[l];
  const std::string f = leaf;
  const int padded = e->dh != 64;
  if (f == "wqkv") { *out = {L.wqkv, 3 * H * H, true, padded ? 1 : 0}; return true; }
  if (f == "wo") { *out = {L.wo, H * H, true, padded ? 2 : 0}; return true; }
  if (f == "wi") { *out = {L.wi, I * H, true, 0}; return true; }
  if (f == "wo2") { *out = {L.wo2, H * I, true, 0}; return true; }
  if (f == "bqkv") { *out = {L.bqkv, 3 * H, false, padded ? 1 : 0}; return true; }
  if (f == "bo") { *out = {L.bo, H, false, 0}; return true; }
  if (f == "bi") { *out = {L.bi, I, false, 0}; return true; }
  if (f == "bo2") { *out = {L.bo2, H, false, 0}; return true; }
  if (f == "ln1_g") { *out = {L.ln1_g, H, false, 0}; return true; }
  if (f == "ln1_b") { *out = {L.ln1_b, H, false, 0}; return true; }
  if (f == "ln2_g") { *out = {L.ln2_g, H, false, 0}; return true; }
  if (f == "ln2_b") { *out = {L.ln2_b, H, false, 0}; return true; }
  return false;
}

int gemm(aur_encoder* e, const CUtensorMap* tm_a, const CUtensorMap* tm_w, __nv_bfloat16* out, int m_rows, int n,
         int k, int epi, const float* bias, const __nv_bfloat16* resid, int ldr) {
  GemmParams p{};
  p.bias = bias; p.resid = resid; p.ldr = ldr; p.out = out; p.ldo = n;
  const int tile_m = 128 * e->cta_group;
  p.m_tiles = (m_rows + tile_m - 1) / tile_m; p.n_tiles = n / e->bn; p.k_blocks = k / 64;
  ENC_TRY(gemm_tc_launch(e->cta_group, e->bn, epi, e->sm_count, tm_a, tm_w, p, e->stream));
  return AUR_OK;
}

// The whole forward for tokens already staged in h_tok / h_pos / h_items.
int forward_locked(aur_encoder* e, const int32_t* cu_host, int n_seq, int n_items) {
  const aur_encoder_config& c = e->cfg;
  const int T = cu_host[n_seq], H = c.hidden, I = c.inter;
  const int t_pad = round_up(T, 256);
  cudaStream_t s = e->stream;
  ENC_TRY(cudaMemcpyAsync(e->d_tok, e->h_tok, sizeof(int32_t) * T, cudaMemcpyHostToDevice, s));
  ENC_TRY(cudaMemcpyAsync(e->d_pos, e->h_pos, sizeof(int32_t) * T, cudaMemcpyHostToDevice, s));
  ENC_TRY(cudaMemcpyAsync(e->d_cu, cu_host, sizeof(int32_t) * (n_seq + 1), cudaMemcpyHostToDevice, s));
  ENC_TRY(cudaMemcpyAsync(e->d_items, e->h_items, sizeof(AttnItem) * n_items, cudaMemcpyHostToDevice, s));
  ENC_TRY(cudaEventRecord(e->ev[0], s));
  int launches = 0;
  ENC_TRY(launch_embed_ln(e->d_tok, e->d_pos, T, t_pad, e->word, e->pos, e->type, e->emb_g, e->emb_b, c.ln_eps, H, e->x, s));
  ++launches;
  AttnParams ap{};
  const int HP = e->hp;
  ap.items = e->d_items; ap.n_items = n_items; ap.heads = c.heads; ap.hidden = HP; ap.ctx = e->ctx; ap.ld_ctx = HP;
  ap.scale_log2e = 1.4426950408889634f / sqrtf(static_cast<float>(e->dh));
  for (int l = 0; l < c.layers; ++l) {
    Layer& L = e->layers[l];
    int rc;
    if ((rc = gemm(e, &e->tm_x, &L.tm_wqkv, e->qkv, T, 3 * HP, H, kEpiBias, L.bqkv, nullptr, 0))) return rc;
    ENC_TRY(attn_tc_launch(&e->tm_qkv, ap, s));
    if ((rc = gemm(e, &e->tm_ctx, &L.tm_wo, e->y, T, H, HP, kEpiBiasResid, L.bo, e->x, H))) return rc;
    ENC_TRY(launch_layernorm(e->y, L.ln1_g, L.ln1_b, c.ln_eps, T, H, e->x, s));
    if ((rc = gemm(e, &e->tm_x, &L.tm_wi, e->inter, T, I, H, kEpiBiasGelu, L.bi, nullptr, 0))) return rc;
    if ((rc = gemm(e, &e->tm_inter, &L.tm_wo2, e->y, T, H, I, kEpiBiasResid, L.bo2, e->x, H))) return rc;
    ENC_TRY(launch_layernorm(e->y, L.ln2_g, L.ln2_b, c.ln_eps, T, H, e->x, s));
    launches += 7;
  }
  ENC_TRY(launch_pool(e->x, e->d_cu, n_seq, H, c.pool, c.normalize, e->d_pool_f32, e->d_pool_bf16, s));
  ++launches;
  ENC_TRY(cudaEventRecord(e->ev[1], s));
  e->stats.tokens = T; e->stats.seqs = n_seq; e->stats.launches = launches;
  double af = 0.0;
  for (int i = 0; i < n_seq; ++i) { const double len = cu_host[i + 1] - cu_host[i]; af += 4.0 * len * len * H; }
  e->stats.attn_flops = af * c.layers;
  e->stats.gemm_flops = 2.0 * T * (3.0 * H * H + 1.0 * H * H + 2.0 * H * I) * c.layers;   // algorithmic (unpadded heads)
  e->last_tokens = T;
  return AUR_OK;
}

int stage_inputs(aur_encoder* e, const int32_t* tokens, const int32_t* cu, int n_seq, int* n_items_out) {
  const aur_encoder_config& c = e->cfg;
  if (!e->missing.empty())
    return report_error(AUR_ERR_INVALID, "encoder parameters not loaded: %s (+%zu more)", e->missing[0].c_str(), e->missing.size() - 1);
  if (!tokens || !cu || n_seq <= 0) return report_error(AUR_ERR_INVALID, "tokens / cu_seqlens / n_seq");
  if (n_seq > c.max_seqs) return report_error(AUR_ERR_NOMEM, "n_seq %d > max_seqs %d", n_seq, c.max_seqs);
  if (cu[0] != 0) return report_error(AUR_ERR_INVALID, "cu_seqlens[0] must be 0");
  const int64_t T = cu[n_seq];
  if (T > c.max_tokens) return report_error(AUR_ERR_NOMEM, "%lld tokens > max_tokens %d", static_cast<long long>(T), c.max_tokens);
  int n_items = 0;
  for (int i = 0; i < n_seq; ++i) {
    const int len = cu[i + 1] - cu[i];
    if (len < 1 || len > c.max_pos) return report_error(AUR_ERR_INVALID, "sequence %d has length %d (1..%d)", i, len, c.max_pos);
    for (int t = 0; t < len; ++t) {
      const int32_t id = tokens[cu[i] + t];
      if (id < 0 || id >= c.vocab) return report_error(AUR_ERR_INVALID, "token id %d out of range at sequence %d", id, i);
      e->h_tok[cu[i] + t] = id; e->h_pos[cu[i] + t] = t;
    }
    for (int q0 = 0; q0 < len; q0 += 128) e->h_items[n_items++] = AttnItem{cu[i], len, q0, 0};
  }
  *n_items_out = n_items;
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
  ENC_TRY(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  ENC_TRY(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9) return report_error(AUR_ERR_UNSUPPORTED, "sm_%d%d device: this library is built for sm_90a only", prop.major, prop.minor);
  aur_encoder* e = new aur_encoder();
  e->cfg = *cfg;
  e->sm_count = prop.multiProcessorCount;
  e->rows_pad = round_up(cfg->max_tokens, 256) + 512;   // + one full key window past the last sequence
  e->cta_group = cfg->reserved == 1 ? 1 : 2;            // reserved = 1 selects the single-CTA GEMM (bring-up)
  e->dh = H / cfg->heads;
  e->hp = cfg->heads * 64;     // head dim 32 is zero-padded to 64: q.k and P.V are unchanged by zero dims
  e->bn = (H % 256 == 0 && I % 256 == 0 && e->hp % 256 == 0) ? 256 : 128;
  e->layers.resize(cfg->layers);
  int rc = AUR_OK;
  auto A = [&](auto** p, size_t n) { if (rc == AUR_OK) rc = dev_alloc(p, n); };
  A(&e->word, static_cast<size_t>(cfg->vocab) * H); A(&e->pos, static_cast<size_t>(cfg->max_pos) * H);
  A(&e->type, static_cast<size_t>(cfg->type_vocab) * H); A(&e->emb_g, H); A(&e->emb_b, H);
  for (Layer& l : e->layers) {
    A(&l.wqkv, static_cast<size_t>(3) * e->hp * H); A(&l.wo, static_cast<size_t>(H) * e->hp);
    A(&l.wi, static_cast<size_t>(I) * H); A(&l.wo2, static_cast<size_t>(H) * I);
    A(&l.bqkv, 3 * e->hp); A(&l.bo, H); A(&l.bi, I); A(&l.bo2, H);
    A(&l.ln1_g, H); A(&l.ln1_b, H); A(&l.ln2_g, H); A(&l.ln2_b, H);
  }
  const size_t R = e->rows_pad;
  A(&e->x, R * H); A(&e->y, R * H); A(&e->qkv, R * 3 * e->hp); A(&e->ctx, R * e->hp); A(&e->inter, R * I);
  A(&e->d_tok, cfg->max_tokens); A(&e->d_pos, cfg->max_tokens); A(&e->d_cu, cfg->max_seqs + 1);
  e->max_items = cfg->max_seqs * 4;
  A(&e->d_items, e->max_items);
  A(&e->d_pool_f32, static_cast<size_t>(cfg->max_seqs) * H); A(&e->d_pool_bf16, static_cast<size_t>(cfg->max_seqs) * H);
  auto fail_open = [&](int code) { free_all(e); delete e; return code; };
  if (rc != AUR_OK) return fail_open(rc);
  if (cudaMallocHost(reinterpret_cast<void**>(&e->h_tok), sizeof(int32_t) * cfg->max_tokens) != cudaSuccess ||
      cudaMallocHost(reinterpret_cast<void**>(&e->h_pos), sizeof(int32_t) * cfg->max_tokens) != cudaSuccess ||
      cudaMallocHost(reinterpret_cast<void**>(&e->h_items), sizeof(AttnItem) * e->max_items) != cudaSuccess)
    return fail_open(report_error(AUR_ERR_NOMEM, "pinned staging allocation failed"));
  if (cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking) != cudaSuccess)
    return fail_open(report_error(AUR_ERR_CUDA, "cudaStreamCreate failed"));
  for (auto& ev : e->ev)
    if (cudaEventCreate(&ev) != cudaSuccess) return fail_open(report_error(AUR_ERR_CUDA, "cudaEventCreate failed"));
  // tensor maps: activations are A operands (box 128 rows), weights B operands (box bn rows)
  const int Ri = static_cast<int>(R);
  const int HP = e->hp;
  if ((rc = make_tmap(&e->tm_x, e->x, H, Ri, 128)) || (rc = make_tmap(&e->tm_ctx, e->ctx, HP, Ri, 128)) ||
      (rc = make_tmap(&e->tm_inter, e->inter, I, Ri, 128)) || (rc = make_tmap(&e->tm_qkv, e->qkv, 3 * HP, Ri, 128)))
    return fail_open(rc);
  for (Layer& l : e->layers) {
    if ((rc = make_tmap(&l.tm_wqkv, l.wqkv, H, 3 * HP, e->bn / e->cta_group)) ||
        (rc = make_tmap(&l.tm_wo, l.wo, HP, H, e->bn / e->cta_group)) ||
        (rc = make_tmap(&l.tm_wi, l.wi, H, I, e->bn / e->cta_group)) ||
        (rc = make_tmap(&l.tm_wo2, l.wo2, I, H, e->bn / e->cta_group)))
      return fail_open(rc);
  }
  e->missing = {"word_emb", "pos_emb", "type_emb", "emb_ln_g", "emb_ln_b"};
  for (int l = 0; l < cfg->layers; ++l)
    for (const char* leaf : {"wqkv", "bqkv", "wo", "bo", "ln1_g", "ln1_b", "wi", "bi", "wo2", "bo2", "ln2_g", "ln2_b"})
      e->missing.push_back("l" + std::to_string(l) + "." + leaf);
  *out = e;
  return AUR_OK;
}

int aur_encoder_close(aur_encoder* e) {
  if (!e) return AUR_OK;
  { std::lock_guard<std::mutex> g(e->mu); cudaSetDevice(e->cfg.device); cudaStreamSynchronize(e->stream); free_all(e); }
  delete e;
  return AUR_OK;
}

int aur_encoder_load(aur_encoder* e, const char* name, const float* data, int64_t count) {
  if (!e || !name || !data) return report_error(AUR_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> g(e->mu);
  ENC_TRY(cudaSetDevice(e->cfg.device));
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
    if (e->stage_elems < static_cast<size_t>(n_up)) {
      if (e->d_stage) cudaFree(e->d_stage);
      e->d_stage = nullptr; e->stage_elems = 0;
      ENC_TRY(cudaMalloc(reinterpret_cast<void**>(&e->d_stage), sizeof(float) * n_up));
      e->stage_elems = n_up;
    }
    ENC_TRY(cudaMemcpyAsync(e->d_stage, data, sizeof(float) * n_up, cudaMemcpyHostToDevice, e->stream));
    ENC_TRY(launch_f32_to_bf16(e->d_stage, static_cast<__nv_bfloat16*>(slot.dst), n_up, e->stream));
  } else {
    ENC_TRY(cudaMemcpyAsync(slot.dst, data, sizeof(float) * n_up, cudaMemcpyHostToDevice, e->stream));
  }
  ENC_TRY(cudaStreamSynchronize(e->stream));
  for (size_t i = 0; i < e->missing.size(); ++i)
    if (e->missing[i] == name) { e->missing.erase(e->missing.begin() + i); break; }
  return AUR_OK;
}

int aur_encode(aur_encoder* e, const int32_t* tokens, const int32_t* cu, int32_t n_seq, float* out_f32, uint16_t* out_bf16) {
  if (!e) return report_error(AUR_ERR_INVALID, "null encoder");
  std::lock_guard<std::mutex> g(e->mu);
  ENC_TRY(cudaSetDevice(e->cfg.device));
  int n_items = 0, rc;
  if ((rc = stage_inputs(e, tokens, cu, n_seq, &n_items))) return rc;
  if ((rc = forward_locked(e, cu, n_seq, n_items))) return rc;
  const size_t n = static_cast<size_t>(n_seq) * e->cfg.hidden;
  // outputs are written only on success: copy into the caller's buffers after the forward is known good
  ENC_TRY(cudaStreamSynchronize(e->stream));
  if (out_f32) ENC_TRY(cudaMemcpy(out_f32, e->d_pool_f32, n * sizeof(float), cudaMemcpyDeviceToHost));
  if (out_bf16) ENC_TRY(cudaMemcpy(out_bf16, e->d_pool_bf16, n * 2, cudaMemcpyDeviceToHost));
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e->ev[0], e->ev[1]);
  e->stats.total_ms = ms;
  return AUR_OK;
}

int aur_encode_append(aur_encoder* e, aur_index* ix, const int32_t* tokens, const int32_t* cu, int32_t n_seq,
                      const int64_t* ids, const int32_t* user_codes, const int32_t* org_codes) {
  if (!e || !ix || !ids) return report_error(AUR_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> g(e->mu);
  ENC_TRY(cudaSetDevice(e->cfg.device));
  aur_stats st{};
  int rc;
  if ((rc = aur_get_stats(ix, &st))) return rc;
  if (st.dim != e->cfg.hidden || st.dtype != AUR_BF16)
    return report_error(AUR_ERR_INVALID, "index is %d-d dtype %d; the encoder produces %d-d bf16", st.dim, st.dtype, e->cfg.hidden);
  int n_items = 0;
  if ((rc = stage_inputs(e, tokens, cu, n_seq, &n_items))) return rc;
  if ((rc = forward_locked(e, cu, n_seq, n_items))) return rc;
  // the pooled rows stay in HBM: the shard copies them device-to-device on the encoder's stream
  if ((rc = aur_add_dev(ix, e->d_pool_bf16, ids, user_codes, org_codes, n_seq, e->stream))) return rc;
  ENC_TRY(cudaStreamSynchronize(e->stream));
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e->ev[0], e->ev[1]);
  e->stats.total_ms = ms;
  return AUR_OK;
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
  ENC_TRY(cudaSetDevice(e->cfg.device));
  if (count != e->last_tokens * e->cfg.hidden) return report_error(AUR_ERR_INVALID, "count must be tokens * hidden of the last call");
  ENC_TRY(cudaStreamSynchronize(e->stream));
  ENC_TRY(cudaMemcpy(out, e->x, count * 2, cudaMemcpyDeviceToHost));
  return AUR_OK;
}

int aur_debug_gemm(int32_t device, const uint16_t* a, const uint16_t* w, const float* bias, const uint16_t* resid,
                   int32_t m, int32_t n, int32_t k, int32_t epi, int32_t cta_group, uint16_t* out, float* ms_out) {
  if (!a || !w || !bias || !out || m <= 0) return report_error(AUR_ERR_INVALID, "null argument");
  if (n % 128 || k % 64 || epi < 0 || epi > 2 || (epi == kEpiBiasResid && !resid) || (cta_group != 1 && cta_group != 2))
    return report_error(AUR_ERR_UNSUPPORTED, "n %% 128, k %% 64, epi 0..2, cta_group 1..2");
  ENC_TRY(cudaSetDevice(device));
  cudaDeviceProp prop;
  ENC_TRY(cudaGetDeviceProperties(&prop, device));
  const int m_pad = round_up(m, 128 * cta_group), bn = n % 256 == 0 ? 256 : 128;
  __nv_bfloat16 *da = nullptr, *dw = nullptr, *dr = nullptr, *dout = nullptr; float* db = nullptr;
  int rc = AUR_OK;
  auto A = [&](auto** p, size_t cnt) { if (rc == AUR_OK) rc = dev_alloc(p, cnt); };
  A(&da, static_cast<size_t>(m_pad) * k); A(&dw, static_cast<size_t>(n) * k); A(&dr, static_cast<size_t>(m_pad) * n);
  A(&dout, static_cast<size_t>(m_pad) * n); A(&db, n);
  auto cleanup = [&](int code) { cudaDeviceSynchronize(); cudaFree(da); cudaFree(dw); cudaFree(dr); cudaFree(dout); cudaFree(db); return code; };
  if (rc) return cleanup(rc);
  cudaMemcpy(da, a, static_cast<size_t>(m) * k * 2, cudaMemcpyHostToDevice);
  cudaMemcpy(dw, w, static_cast<size_t>(n) * k * 2, cudaMemcpyHostToDevice);
  cudaMemcpy(db, bias, sizeof(float) * n, cudaMemcpyHostToDevice);
  if (resid) cudaMemcpy(dr, resid, static_cast<size_t>(m) * n * 2, cudaMemcpyHostToDevice);
  CUtensorMap tm_a, tm_w;
  if ((rc = make_tmap(&tm_a, da, k, m_pad, 128)) || (rc = make_tmap(&tm_w, dw, k, n, bn / cta_group)))
    return cleanup(rc);
  GemmParams p{};
  p.bias = db; p.resid = dr; p.ldr = n; p.out = dout; p.ldo = n;
  p.m_tiles = m_pad / (128 * cta_group); p.n_tiles = n / bn; p.k_blocks = k / 64;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaError_t ce = cudaSuccess;
  for (int rep = 0; rep < 3 && ce == cudaSuccess; ++rep) {   // last repetition is the timed one
    cudaEventRecord(e0, nullptr);
    ce = gemm_tc_launch(cta_group, bn, epi, prop.multiProcessorCount, &tm_a, &tm_w, p, nullptr);
    cudaEventRecord(e1, nullptr);
  }
  if (ce == cudaSuccess) ce = cudaDeviceSynchronize();
  float ms = 0.f;
  if (ce == cudaSuccess) cudaEventElapsedTime(&ms, e0, e1);
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  if (ce != cudaSuccess) return cleanup(report_error(AUR_ERR_CUDA, "gemm: %s", cudaGetErrorString(ce)));
  ce = cudaMemcpy(out, dout, static_cast<size_t>(m) * n * 2, cudaMemcpyDeviceToHost);
  if (ce != cudaSuccess) return cleanup(report_error(AUR_ERR_CUDA, "gemm d2h: %s", cudaGetErrorString(ce)));
  if (ms_out) *ms_out = ms;
  return cleanup(AUR_OK);
}

int aur_debug_attention(int32_t device, const uint16_t* qkv, const int32_t* cu, int32_t n_seq, int32_t heads,
                        int32_t hidden, uint16_t* ctx, float* ms_out) {
  if (!qkv || !cu || !ctx || n_seq <= 0) return report_error(AUR_ERR_INVALID, "null argument");
  if (heads <= 0 || hidden != heads * 64) return report_error(AUR_ERR_UNSUPPORTED, "head dim must be 64");
  ENC_TRY(cudaSetDevice(device));
  cudaDeviceProp prop;
  ENC_TRY(cudaGetDeviceProperties(&prop, device));
  const int T = cu[n_seq], rows = round_up(T, 128) + 512;
  std::vector<AttnItem> items;
  for (int i = 0; i < n_seq; ++i) {
    const int len = cu[i + 1] - cu[i];
    if (len < 1 || len > 512) return report_error(AUR_ERR_INVALID, "sequence length %d", len);
    for (int q0 = 0; q0 < len; q0 += 128) items.push_back(AttnItem{cu[i], len, q0, 0});
  }
  __nv_bfloat16 *dq = nullptr, *dc = nullptr; AttnItem* di = nullptr;
  int rc = AUR_OK;
  auto A = [&](auto** p, size_t cnt) { if (rc == AUR_OK) rc = dev_alloc(p, cnt); };
  A(&dq, static_cast<size_t>(rows) * 3 * hidden); A(&dc, static_cast<size_t>(rows) * hidden); A(&di, items.size());
  auto cleanup = [&](int code) { cudaDeviceSynchronize(); cudaFree(dq); cudaFree(dc); cudaFree(di); return code; };
  if (rc) return cleanup(rc);
  cudaMemcpy(dq, qkv, static_cast<size_t>(T) * 3 * hidden * 2, cudaMemcpyHostToDevice);
  cudaMemcpy(di, items.data(), sizeof(AttnItem) * items.size(), cudaMemcpyHostToDevice);
  CUtensorMap tm;
  if ((rc = make_tmap(&tm, dq, 3 * hidden, rows, 128))) return cleanup(rc);
  AttnParams ap{};
  ap.items = di; ap.n_items = static_cast<int>(items.size()); ap.heads = heads; ap.hidden = hidden; ap.ctx = dc; ap.ld_ctx = hidden;
  ap.scale_log2e = 1.4426950408889634f / 8.0f;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaError_t ce = cudaSuccess;
  for (int rep = 0; rep < 3 && ce == cudaSuccess; ++rep) {
    cudaEventRecord(e0, nullptr);
    ce = attn_tc_launch(&tm, ap, nullptr);
    cudaEventRecord(e1, nullptr);
  }
  if (ce == cudaSuccess) ce = cudaDeviceSynchronize();
  float ms = 0.f;
  if (ce == cudaSuccess) cudaEventElapsedTime(&ms, e0, e1);
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  if (ce != cudaSuccess) return cleanup(report_error(AUR_ERR_CUDA, "attention: %s", cudaGetErrorString(ce)));
  ce = cudaMemcpy(ctx, dc, static_cast<size_t>(T) * hidden * 2, cudaMemcpyDeviceToHost);
  if (ce != cudaSuccess) return cleanup(report_error(AUR_ERR_CUDA, "attention d2h: %s", cudaGetErrorString(ce)));
  if (ms_out) *ms_out = ms;
  return cleanup(AUR_OK);
}

}  // extern "C"
