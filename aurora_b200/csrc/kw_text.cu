// Keyword analysis on the device (aur_kw_vocab_*, aur_kw_add_text; DESIGN.md section 10, "Text analysis"): UTF-8 text
// in, (term id, tf) rows in one or more keyword stores out, with the vocabulary (word -> term id) held in HBM.
//
// The definition is bm25.build_csr: words are re.findall(r"[0-9a-z]+", text.lower()), on bytes:
//   ASCII letters and digits are word characters (upper case lowered); E2 84 AA (U+212A KELVIN SIGN) is "k" inside
//   the word; C4 B0 (U+0130) is "i" followed by a break (Python lowers it to "i" + U+0307); every other byte breaks.
// A word the vocabulary lacks gets the next free id in order of first occurrence in the batch (document order, then
// position), which is build_csr's Counter order, so ids and rows equal build_csr's for the same texts in the same order.
//
// One slice of documents runs on the vocabulary's device and stream:
//   classify bytes -> scans -> normalised word bytes (the words back to back) and each word's start and document
//   -> FNV-1a hash per word -> lookup in the vocabulary's open-addressing table (hash -> id; equality on the bytes)
//   -> words not found meet in a batch table (CAS on the first occupant, bytes compared within a hash, atomicMin of the
//      first occurrence) -> the first occurrences are ranked by a scan and get ids V + rank -> one read-back of the new
//      word count and bytes, table (1/2 load) and pool growth, insertion (distinct absent words: one CAS per slot)
//   -> radix sort of (document, term id), run lengths as tf -> rows, read back as term ids + per-document counts for
//      the stores' host bookkeeping, and copied (peer copy across devices) behind each store's published prefix.
#include <cuda_runtime.h>
#include <string.h>

#include <cub/cub.cuh>

#include <algorithm>
#include <memory>
#include <mutex>
#include <vector>

#include "../../include/aurora_b200.h"
#include "internal.h"

using namespace aur;

namespace {

constexpr int64_t kMaxWords = int64_t(1) << 28;       // the store's term id range
constexpr int64_t kSliceBytes = int64_t(64) << 20;    // text bytes one slice takes (a larger document is a slice alone)
constexpr int64_t kMaxDocBytes = 0x7FFFFFFFll;        // byte positions of a slice are int32
constexpr int kMaxStores = 64;
constexpr int kT = 256;

unsigned blocks(int64_t n) { return static_cast<unsigned>(std::max<int64_t>(1, (n + kT - 1) / kT)); }

// ------------------------------------------------------------------------------------------------------- kernels
enum : int { kBreak = 0, kWord = 1, kSkip = 2 };

// Class of byte p of a document spanning [ds, de); *ch = the word character it contributes (kWord).
__device__ __forceinline__ int classify(const uint8_t* t, int64_t p, int64_t ds, int64_t de, uint8_t* ch) {
  const uint8_t c = t[p];
  if ((c >= '0' && c <= '9') || (c >= 'a' && c <= 'z')) { *ch = c; return kWord; }
  if (c >= 'A' && c <= 'Z') { *ch = static_cast<uint8_t>(c + 32); return kWord; }
  if (c == 0xE2 && p + 2 < de && t[p + 1] == 0x84 && t[p + 2] == 0xAA) { *ch = 'k'; return kWord; }
  if (c == 0x84 && p >= ds + 1 && p + 1 < de && t[p - 1] == 0xE2 && t[p + 1] == 0xAA) return kSkip;
  if (c == 0xAA && p >= ds + 2 && t[p - 2] == 0xE2 && t[p - 1] == 0x84) return kSkip;
  if (c == 0xC4 && p + 1 < de && t[p + 1] == 0xB0) { *ch = 'i'; return kWord; }
  return kBreak;
}

// Document of byte p: the last d with off[d] <= p (off [n + 1], non-decreasing, p < off[n]).
__device__ __forceinline__ int32_t doc_of(const int64_t* off, int32_t n, int64_t p) {
  int32_t lo = 0, hi = n;   // off[lo] <= p < off[hi]
  while (hi - lo > 1) {
    const int32_t mid = (lo + hi) >> 1;
    if (off[mid] <= p) lo = mid; else hi = mid;
  }
  return lo;
}

// is_w[p] = byte p contributes a word character, is_s[p] = it starts a word.
__global__ void tx_classify(const uint8_t* t, int64_t nb, const int64_t* off, int32_t n, int32_t* is_w, int32_t* is_s) {
  const int64_t p = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= nb) return;
  const int32_t d = doc_of(off, n, p);
  const int64_t ds = off[d], de = off[d + 1];
  uint8_t ch = 0;
  const int k = classify(t, p, ds, de, &ch);
  int start = 0;
  if (k == kWord) {
    int64_t q = p - 1;
    int kq = kBreak;
    while (q >= ds && (kq = classify(t, q, ds, de, &ch)) == kSkip) --q;   // at most the two tail bytes of a KELVIN SIGN
    start = q < ds || kq != kWord;
  }
  is_w[p] = k == kWord;
  is_s[p] = start;
}

// Scatter: norm[cpos[p]] = the character of byte p; word w = widx[p] starts at cpos[p] in document d.
__global__ void tx_compact(const uint8_t* t, int64_t nb, const int64_t* off, int32_t n, const int32_t* is_w, const int32_t* is_s,
                           const int32_t* cpos, const int32_t* widx, uint8_t* norm, int32_t* wstart, int32_t* wdoc) {
  const int64_t p = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= nb || !is_w[p]) return;
  const int32_t d = doc_of(off, n, p);
  uint8_t ch = 0;
  classify(t, p, off[d], off[d + 1], &ch);
  norm[cpos[p]] = ch;
  if (is_s[p]) { wstart[widx[p]] = cpos[p]; wdoc[widx[p]] = d; }
}

__device__ __forceinline__ uint64_t fnv1a(const uint8_t* s, int64_t len) {
  uint64_t h = 1469598103934665603ull;
  for (int64_t i = 0; i < len; ++i) h = (h ^ s[i]) * 1099511628211ull;
  return h;
}
__device__ __forceinline__ uint64_t slot_of(uint64_t h, uint64_t mask) { return (h * 0x9E3779B97F4A7C15ull >> 17) & mask; }
__device__ __forceinline__ bool same_bytes(const uint8_t* a, const uint8_t* b, int64_t len) {
  for (int64_t i = 0; i < len; ++i) if (a[i] != b[i]) return false;
  return true;
}

// The vocabulary in HBM: table [cap] (hash, id; id -1 = empty), words' bytes pool[woff[id] .. woff[id + 1]).
struct VocabDev { uint64_t* hkey; int32_t* hid; uint64_t mask; const uint8_t* pool; const int64_t* woff; };
// One slice's words: word w is norm[wstart[w] .. wstart[w + 1]) (wstart[nw] = normalised bytes).
struct Words { const uint8_t* norm; const int32_t* wstart; int32_t nw; };

__global__ void tx_hash(Words w, uint64_t hmask, uint64_t* wh) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= w.nw) return;
  wh[i] = fnv1a(w.norm + w.wstart[i], w.wstart[i + 1] - w.wstart[i]) & hmask;
}

// found[w] = the vocabulary's id of word w, -1 when absent.
__global__ void tx_lookup(Words w, const uint64_t* wh, VocabDev v, int32_t* found) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= w.nw) return;
  const uint64_t h = wh[i];
  const uint8_t* s = w.norm + w.wstart[i];
  const int64_t len = w.wstart[i + 1] - w.wstart[i];
  int32_t out = -1;
  for (uint64_t slot = slot_of(h, v.mask);; slot = (slot + 1) & v.mask) {
    const int32_t id = v.hid[slot];
    if (id < 0) break;
    if (v.hkey[slot] == h && v.woff[id + 1] - v.woff[id] == len && same_bytes(v.pool + v.woff[id], s, len)) { out = id; break; }
  }
  found[i] = out;
}

// Words not found meet in the batch table [mask + 1]: occ = the word that claimed the slot (-1 empty), first = the
// least word index with the same bytes.  bslot[w] = word w's slot.  Words of one hash probe the same run, so two
// words with equal hashes but different bytes take different slots.
__global__ void tx_group(Words w, const uint64_t* wh, const int32_t* found, int32_t* occ, int32_t* first, uint64_t mask,
                         int32_t* bslot) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= w.nw) return;
  if (found[i] >= 0) { bslot[i] = -1; return; }
  const uint64_t h = wh[i];
  const uint8_t* s = w.norm + w.wstart[i];
  const int32_t len = w.wstart[i + 1] - w.wstart[i];
  for (uint64_t slot = slot_of(h, mask);; slot = (slot + 1) & mask) {
    const int32_t cur = atomicCAS(occ + slot, -1, static_cast<int32_t>(i));
    if (cur < 0 || (wh[cur] == h && w.wstart[cur + 1] - w.wstart[cur] == len && same_bytes(w.norm + w.wstart[cur], s, len))) {
      atomicMin(first + slot, static_cast<int32_t>(i));
      bslot[i] = static_cast<int32_t>(slot);
      return;
    }
  }
}

// is_first[w] = word w is the first occurrence of a new word; nlen[w] = its length then (0 otherwise).
__global__ void tx_mark(Words w, const int32_t* bslot, const int32_t* first, int32_t* is_first, int32_t* nlen) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= w.nw) return;
  const bool f = bslot[i] >= 0 && first[bslot[i]] == i;
  is_first[i] = f;
  nlen[i] = f ? w.wstart[i + 1] - w.wstart[i] : 0;
}

// totals[0] = new words, totals[1] = their bytes (inclusive ends of the two exclusive scans).
__global__ void tx_totals(const int32_t* is_first, const int32_t* rank, const int32_t* nlen, const int32_t* noff, int32_t nw,
                          int64_t* totals) {
  totals[0] = nw ? static_cast<int64_t>(rank[nw - 1]) + is_first[nw - 1] : 0;
  totals[1] = nw ? static_cast<int64_t>(noff[nw - 1]) + nlen[nw - 1] : 0;
}

// New word w (first occurrence): id V + rank[w], bytes appended to the pool, one CAS into the table (the new words are
// distinct and absent, so a slot that is taken holds another word).
__global__ void tx_insert(Words w, const uint64_t* wh, const int32_t* is_first, const int32_t* rank, const int32_t* noff,
                          int64_t V, int64_t pool_used, uint64_t* hkey, int32_t* hid, uint64_t mask, uint8_t* pool, int64_t* woff) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= w.nw || !is_first[i]) return;
  const int32_t id = static_cast<int32_t>(V + rank[i]);
  const int32_t len = w.wstart[i + 1] - w.wstart[i];
  const int64_t at = pool_used + noff[i];
  for (int32_t j = 0; j < len; ++j) pool[at + j] = w.norm[w.wstart[i] + j];
  woff[id + 1] = at + len;
  for (uint64_t slot = slot_of(wh[i], mask);; slot = (slot + 1) & mask)
    if (atomicCAS(hid + slot, -1, id) < 0) { hkey[slot] = wh[i]; return; }
}

// Rehash the old table into the new one (the new one all empty).
__global__ void tx_rehash(const uint64_t* okey, const int32_t* oid, int64_t ocap, uint64_t* hkey, int32_t* hid, uint64_t mask) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= ocap || oid[i] < 0) return;
  for (uint64_t slot = slot_of(okey[i], mask);; slot = (slot + 1) & mask)
    if (atomicCAS(hid + slot, -1, oid[i]) < 0) { hkey[slot] = okey[i]; return; }
}

// key[w] = (document << 28) | term id of word w.
__global__ void tx_keys(const int32_t* wdoc, const int32_t* found, const int32_t* bslot, const int32_t* first,
                        const int32_t* rank, int64_t V, int32_t nw, uint64_t* key) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= nw) return;
  const int64_t id = found[i] >= 0 ? found[i] : V + rank[first[bslot[i]]];
  key[i] = (static_cast<uint64_t>(wdoc[i]) << 28) | static_cast<uint64_t>(id);
}

// Run r of the sorted keys -> posting (term id, tf); its document gains a posting and tf tokens.
__global__ void tx_postings(const uint64_t* ukey, const int32_t* cnt, const int32_t* n_runs, uint2* post, int32_t* tid,
                            int32_t* dcnt, int32_t* dlen) {
  const int64_t r = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r >= *n_runs) return;
  const uint32_t id = static_cast<uint32_t>(ukey[r] & ((1u << 28) - 1));
  const int32_t d = static_cast<int32_t>(ukey[r] >> 28);
  post[r] = make_uint2(id, static_cast<uint32_t>(cnt[r]));
  tid[r] = static_cast<int32_t>(id);
  atomicAdd(dcnt + d, 1);
  atomicAdd(dlen + d, cnt[r]);
}

// Postings of the documents map[0 .. m) (source offsets src_off) to dst at dst_off; one warp per document.
__global__ void tx_gather(const uint2* post, const int64_t* src_off, const int32_t* map, const int64_t* dst_off, int64_t m, uint2* dst) {
  const int64_t w = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (w >= m) return;
  const int64_t o0 = src_off[map[w]], o1 = src_off[map[w] + 1], d = dst_off[w];
  for (int64_t i = threadIdx.x & 31; i < o1 - o0; i += 32) dst[d + i] = post[o0 + i];
}

}  // namespace

struct aur_kw_vocab {
  std::mutex mu;                   // one text add (or read) at a time
  int device = 0;
  Stream stream;
  int hash_bits = 64;
  int64_t words = 0, bytes = 0;    // V and the pool bytes in use
  DevBuf<uint64_t> hkey; DevBuf<int32_t> hid;                         // table (power of two entries)
  DevBuf<uint8_t> pool;
  DevBuf<int64_t> woff;                                                // [words + 1]
  // one slice's scratch (grow-only)
  HostBuf<uint8_t> h_stage;                                            // page-locked text staging
  DevBuf<uint8_t> text, norm, cub_tmp;
  DevBuf<int64_t> doff, totals, goff_src, goff_dst;
  DevBuf<int32_t> is_w, is_s, cpos, widx, wstart, wdoc, found, bslot, occ, first, is_first, rank, nlen, noff;
  DevBuf<int32_t> cnt, n_runs, tid, dcnt, dlen, gmap;
  DevBuf<uint64_t> wh, key, key_sorted, ukey;
  DevBuf<uint2> post, spost;
};

namespace {

int ensure_table(aur_kw_vocab* v, int64_t need_words) {
  const int64_t tcap = static_cast<int64_t>(v->hkey.n);
  if (tcap && 2 * need_words <= tcap) return AUR_OK;
  int64_t cap = std::max<int64_t>(tcap, 1024);
  while (2 * need_words > cap) cap *= 2;
  DevBuf<uint64_t> hk; DevBuf<int32_t> hi;
  const cudaError_t e = [&]() -> cudaError_t {
    AUR_CU_RET(hk.reserve(static_cast<size_t>(cap)));
    AUR_CU_RET(hi.reserve(static_cast<size_t>(cap)));
    AUR_CU_RET(cudaMemsetAsync(hi.p, 0xFF, static_cast<size_t>(cap) * 4, v->stream));
    if (tcap) {
      tx_rehash<<<blocks(tcap), kT, 0, v->stream>>>(v->hkey.p, v->hid.p, tcap, hk.p, hi.p, static_cast<uint64_t>(cap - 1));
      AUR_CU_RET(cudaGetLastError());
    }
    return cudaStreamSynchronize(v->stream);
  }();
  if (e != cudaSuccess)
    return report_error(e == cudaErrorMemoryAllocation ? AUR_ERR_NOMEM : AUR_ERR_CUDA, "vocabulary table: %s", cudaGetErrorString(e));
  v->hkey = std::move(hk); v->hid = std::move(hi);
  return AUR_OK;
}

// Analysed rows of one slice of documents, on the vocabulary's device: post [total] (term id, tf) in document order,
// and on the host each document's posting count, length and every posting's term id.
struct SliceRows {
  int64_t total = 0;
  std::vector<int32_t> dcnt, dlen, tid;
  std::vector<int64_t> off;   // [n + 1]
  int32_t max_term = -1;
};

// Analyse documents [0, n) of the slice whose text is text[0 .. nb) with offsets off[0 .. n] (from 0) into the
// vocabulary and v->post.  The 2^28 word limit is checked before the vocabulary changes.
int analyse(aur_kw_vocab* v, const char* text, const int64_t* off, int32_t n, SliceRows* out) {
  cudaStream_t s = v->stream;
  const int64_t nb = off[n];
  if (v->h_stage.n < static_cast<size_t>(nb))
    AUR_TRY(v->h_stage.reserve(static_cast<size_t>(std::max<int64_t>(nb, 1 << 20)), cudaHostAllocDefault));
  // 1. text in (the staging buffer is reused only after this slice's work has completed)
  if (nb) memcpy(v->h_stage.p, text, static_cast<size_t>(nb));
  const size_t B = static_cast<size_t>(std::max<int64_t>(nb, 1));
  AUR_TRY(v->text.reserve(B)); AUR_TRY(v->doff.reserve(static_cast<size_t>(n) + 1));
  AUR_TRY(v->is_w.reserve(B)); AUR_TRY(v->is_s.reserve(B)); AUR_TRY(v->cpos.reserve(B)); AUR_TRY(v->widx.reserve(B));
  AUR_TRY(v->totals.reserve(2));
  if (nb) AUR_TRY(cudaMemcpyAsync(v->text.p, v->h_stage.p, static_cast<size_t>(nb), cudaMemcpyHostToDevice, s));
  AUR_TRY(cudaMemcpyAsync(v->doff.p, off, (static_cast<size_t>(n) + 1) * 8, cudaMemcpyHostToDevice, s));
  // 2. classify, scans: normalised bytes and word starts
  int32_t nw = 0, nl = 0;
  if (nb) {
    tx_classify<<<blocks(nb), kT, 0, s>>>(v->text.p, nb, v->doff.p, n, v->is_w.p, v->is_s.p);
    AUR_TRY(cudaGetLastError());
    size_t tb = 0, tb2 = 0;
    AUR_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tb, v->is_w.p, v->cpos.p, static_cast<int>(nb), s));
    AUR_TRY(v->cub_tmp.reserve(std::max<size_t>(tb, 1)));
    AUR_TRY(cub::DeviceScan::ExclusiveSum(v->cub_tmp.p, tb, v->is_w.p, v->cpos.p, static_cast<int>(nb), s));
    AUR_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tb2, v->is_s.p, v->widx.p, static_cast<int>(nb), s));
    AUR_TRY(v->cub_tmp.reserve(std::max<size_t>(tb2, 1)));
    AUR_TRY(cub::DeviceScan::ExclusiveSum(v->cub_tmp.p, tb2, v->is_s.p, v->widx.p, static_cast<int>(nb), s));
    int32_t tail[4];
    AUR_TRY(cudaMemcpyAsync(tail, v->cpos.p + nb - 1, 4, cudaMemcpyDeviceToHost, s));
    AUR_TRY(cudaMemcpyAsync(tail + 1, v->is_w.p + nb - 1, 4, cudaMemcpyDeviceToHost, s));
    AUR_TRY(cudaMemcpyAsync(tail + 2, v->widx.p + nb - 1, 4, cudaMemcpyDeviceToHost, s));
    AUR_TRY(cudaMemcpyAsync(tail + 3, v->is_s.p + nb - 1, 4, cudaMemcpyDeviceToHost, s));
    AUR_TRY(cudaStreamSynchronize(s));
    nl = tail[0] + tail[1];
    nw = tail[2] + tail[3];
  }
  out->dcnt.assign(static_cast<size_t>(n), 0);
  out->dlen.assign(static_cast<size_t>(n), 0);
  out->off.assign(static_cast<size_t>(n) + 1, 0);
  out->tid.clear();
  out->total = 0;
  out->max_term = -1;
  if (nw == 0) return AUR_OK;
  const size_t W = static_cast<size_t>(nw);
  AUR_TRY(v->norm.reserve(static_cast<size_t>(nl))); AUR_TRY(v->wstart.reserve(W + 1)); AUR_TRY(v->wdoc.reserve(W));
  tx_compact<<<blocks(nb), kT, 0, s>>>(v->text.p, nb, v->doff.p, n, v->is_w.p, v->is_s.p, v->cpos.p, v->widx.p, v->norm.p,
                                      v->wstart.p, v->wdoc.p);
  AUR_TRY(cudaGetLastError());
  AUR_TRY(cudaMemcpyAsync(v->wstart.p + nw, &nl, 4, cudaMemcpyHostToDevice, s));
  const Words w{v->norm.p, v->wstart.p, nw};
  // 3. hash, 4. lookup
  AUR_TRY(v->wh.reserve(W)); AUR_TRY(v->found.reserve(W)); AUR_TRY(v->bslot.reserve(W));
  const uint64_t hmask = v->hash_bits >= 64 ? ~0ull : ((1ull << v->hash_bits) - 1);
  tx_hash<<<blocks(nw), kT, 0, s>>>(w, hmask, v->wh.p);
  tx_lookup<<<blocks(nw), kT, 0, s>>>(w, v->wh.p, VocabDev{v->hkey.p, v->hid.p, static_cast<uint64_t>(v->hkey.n - 1), v->pool.p, v->woff.p},
                                      v->found.p);
  AUR_TRY(cudaGetLastError());
  // 5. new words: group, rank by first occurrence
  int64_t bcap = 1024;
  while (bcap < 2 * static_cast<int64_t>(nw)) bcap *= 2;
  AUR_TRY(v->occ.reserve(static_cast<size_t>(bcap))); AUR_TRY(v->first.reserve(static_cast<size_t>(bcap)));
  AUR_TRY(v->is_first.reserve(W)); AUR_TRY(v->rank.reserve(W)); AUR_TRY(v->nlen.reserve(W)); AUR_TRY(v->noff.reserve(W));
  AUR_TRY(cudaMemsetAsync(v->occ.p, 0xFF, static_cast<size_t>(bcap) * 4, s));
  AUR_TRY(cudaMemsetAsync(v->first.p, 0x7F, static_cast<size_t>(bcap) * 4, s));
  tx_group<<<blocks(nw), kT, 0, s>>>(w, v->wh.p, v->found.p, v->occ.p, v->first.p, static_cast<uint64_t>(bcap - 1), v->bslot.p);
  tx_mark<<<blocks(nw), kT, 0, s>>>(w, v->bslot.p, v->first.p, v->is_first.p, v->nlen.p);
  AUR_TRY(cudaGetLastError());
  {
    size_t tb = 0;
    AUR_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tb, v->is_first.p, v->rank.p, nw, s));
    AUR_TRY(v->cub_tmp.reserve(std::max<size_t>(tb, 1)));
    AUR_TRY(cub::DeviceScan::ExclusiveSum(v->cub_tmp.p, tb, v->is_first.p, v->rank.p, nw, s));
    AUR_TRY(cub::DeviceScan::ExclusiveSum(v->cub_tmp.p, tb, v->nlen.p, v->noff.p, nw, s));
  }
  tx_totals<<<1, 1, 0, s>>>(v->is_first.p, v->rank.p, v->nlen.p, v->noff.p, nw, v->totals.p);
  int64_t tot[2];
  AUR_TRY(cudaMemcpyAsync(tot, v->totals.p, 16, cudaMemcpyDeviceToHost, s));
  AUR_TRY(cudaStreamSynchronize(s));
  const int64_t n_new = tot[0], new_bytes = tot[1], V = v->words;
  if (V + n_new > kMaxWords)
    return report_error(AUR_ERR_INVALID, "the vocabulary would hold %lld words (at most 2^28)", (long long)(V + n_new));
  // Everything the rest of the slice allocates is reserved before the vocabulary changes, and the new words are
  // committed (V, bytes) as soon as their insertion is enqueued: a failure after that point leaves them fully in the
  // vocabulary (ids V .. V + n_new - 1, as the table and pool hold them), never in the table without being counted.
  AUR_TRY(v->key.reserve(W)); AUR_TRY(v->key_sorted.reserve(W)); AUR_TRY(v->ukey.reserve(W)); AUR_TRY(v->cnt.reserve(W));
  AUR_TRY(v->n_runs.reserve(1)); AUR_TRY(v->post.reserve(W)); AUR_TRY(v->tid.reserve(W));
  AUR_TRY(v->dcnt.reserve(static_cast<size_t>(n))); AUR_TRY(v->dlen.reserve(static_cast<size_t>(n)));
  int end_bit = 28;
  while (end_bit < 64 && (int64_t(1) << (end_bit - 28)) < n) ++end_bit;
  size_t tb_sort = 0, tb_rle = 0;
  AUR_TRY(cub::DeviceRadixSort::SortKeys(nullptr, tb_sort, v->key.p, v->key_sorted.p, nw, 0, end_bit, s));
  AUR_TRY(cub::DeviceRunLengthEncode::Encode(nullptr, tb_rle, v->key_sorted.p, v->ukey.p, v->cnt.p, v->n_runs.p, nw, s));
  AUR_TRY(v->cub_tmp.reserve(std::max<size_t>(std::max(tb_sort, tb_rle), 1)));
  // growth, then insertion
  const int rc = ensure_table(v, V + n_new);
  if (rc != AUR_OK) return rc;
  const cudaError_t e = [&]() -> cudaError_t {
    AUR_CU_RET(v->pool.grow_keep(static_cast<size_t>(v->bytes + new_bytes), static_cast<size_t>(v->bytes), s));
    return v->woff.grow_keep(static_cast<size_t>(V + n_new + 1), static_cast<size_t>(V + 1), s);
  }();
  if (e != cudaSuccess)
    return report_error(e == cudaErrorMemoryAllocation ? AUR_ERR_NOMEM : AUR_ERR_CUDA, "vocabulary growth: %s", cudaGetErrorString(e));
  if (n_new) {
    tx_insert<<<blocks(nw), kT, 0, s>>>(w, v->wh.p, v->is_first.p, v->rank.p, v->noff.p, V, v->bytes, v->hkey.p, v->hid.p,
                                        static_cast<uint64_t>(v->hkey.n - 1), v->pool.p, v->woff.p);
    AUR_TRY(cudaGetLastError());
    v->words = V + n_new;
    v->bytes += new_bytes;
  }
  // 6. rows: sort (document, term id), run lengths as tf
  tx_keys<<<blocks(nw), kT, 0, s>>>(v->wdoc.p, v->found.p, v->bslot.p, v->first.p, v->rank.p, V, nw, v->key.p);
  AUR_TRY(cudaGetLastError());
  AUR_TRY(cub::DeviceRadixSort::SortKeys(v->cub_tmp.p, tb_sort, v->key.p, v->key_sorted.p, nw, 0, end_bit, s));
  AUR_TRY(cub::DeviceRunLengthEncode::Encode(v->cub_tmp.p, tb_rle, v->key_sorted.p, v->ukey.p, v->cnt.p, v->n_runs.p, nw, s));
  AUR_TRY(cudaMemsetAsync(v->dcnt.p, 0, static_cast<size_t>(n) * 4, s));
  AUR_TRY(cudaMemsetAsync(v->dlen.p, 0, static_cast<size_t>(n) * 4, s));
  tx_postings<<<blocks(nw), kT, 0, s>>>(v->ukey.p, v->cnt.p, v->n_runs.p, v->post.p, v->tid.p, v->dcnt.p, v->dlen.p);
  AUR_TRY(cudaGetLastError());
  // the host's share: per document (postings, length), then every posting's term id
  AUR_TRY(cudaMemcpyAsync(out->dcnt.data(), v->dcnt.p, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToHost, s));
  AUR_TRY(cudaMemcpyAsync(out->dlen.data(), v->dlen.p, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToHost, s));
  AUR_TRY(cudaStreamSynchronize(s));
  for (int32_t i = 0; i < n; ++i) out->off[static_cast<size_t>(i) + 1] = out->off[static_cast<size_t>(i)] + out->dcnt[static_cast<size_t>(i)];
  out->total = out->off.back();
  out->tid.resize(static_cast<size_t>(out->total));
  if (out->total) {
    AUR_TRY(cudaMemcpyAsync(out->tid.data(), v->tid.p, static_cast<size_t>(out->total) * 4, cudaMemcpyDeviceToHost, s));
    AUR_TRY(cudaStreamSynchronize(s));
  }
  out->max_term = *std::max_element(out->tid.begin(), out->tid.end());   // nw > 0: at least one posting
  return AUR_OK;
}

// 7. Slice rows -> stores: documents of store s (ids mod n_stores) in batch order.  The postings of every store's
// documents are gathered store by store on the vocabulary's device, then each store copies its range in.
int publish(aur_kw_vocab* v, aur_kw* const* stores, int ns, const int64_t* ids, const int32_t* user, const int32_t* org,
            int32_t n, const SliceRows& r) {
  std::vector<std::vector<int32_t>> docs(static_cast<size_t>(ns));
  for (int32_t i = 0; i < n; ++i) docs[static_cast<size_t>(ids[i] % ns)].push_back(i);
  const uint2* src = v->post.p;
  std::vector<int64_t> sbase(static_cast<size_t>(ns) + 1, 0);   // store s's postings at src[sbase[s] ..)
  if (ns > 1 && r.total) {
    std::vector<int32_t> map;
    std::vector<int64_t> doff;
    int64_t at = 0;
    for (int s = 0; s < ns; ++s) {
      sbase[static_cast<size_t>(s)] = at;
      for (int32_t d : docs[static_cast<size_t>(s)]) {
        map.push_back(d);
        doff.push_back(at);
        at += r.dcnt[static_cast<size_t>(d)];
      }
    }
    sbase[static_cast<size_t>(ns)] = at;
    const int64_t m = static_cast<int64_t>(map.size());
    AUR_TRY(v->gmap.reserve(static_cast<size_t>(m))); AUR_TRY(v->goff_dst.reserve(static_cast<size_t>(m)));
    AUR_TRY(v->goff_src.reserve(static_cast<size_t>(n) + 1)); AUR_TRY(v->spost.reserve(static_cast<size_t>(r.total)));
    AUR_TRY(cudaMemcpyAsync(v->gmap.p, map.data(), static_cast<size_t>(m) * 4, cudaMemcpyHostToDevice, v->stream));
    AUR_TRY(cudaMemcpyAsync(v->goff_dst.p, doff.data(), static_cast<size_t>(m) * 8, cudaMemcpyHostToDevice, v->stream));
    AUR_TRY(cudaMemcpyAsync(v->goff_src.p, r.off.data(), (static_cast<size_t>(n) + 1) * 8, cudaMemcpyHostToDevice, v->stream));
    tx_gather<<<blocks(m * 32), kT, 0, v->stream>>>(v->post.p, v->goff_src.p, v->gmap.p, v->goff_dst.p, m, v->spost.p);
    AUR_TRY(cudaGetLastError());
    AUR_TRY(cudaStreamSynchronize(v->stream));
    src = v->spost.p;
  }
  int rc = AUR_OK;
  for (int s = 0; s < ns && rc == AUR_OK; ++s) {
    const std::vector<int32_t>& dl = docs[static_cast<size_t>(s)];
    if (dl.empty()) continue;
    const size_t m = dl.size();
    std::vector<int64_t> sid(m), soff(m + 1, 0);
    std::vector<int32_t> su(m), so(m), slen(m), stid;
    int32_t max_term = -1;
    for (size_t j = 0; j < m; ++j) {
      const int32_t d = dl[j];
      sid[j] = ids[d]; su[j] = user ? user[d] : 0; so[j] = org ? org[d] : -1;
      slen[j] = r.dlen[static_cast<size_t>(d)];
      soff[j + 1] = soff[j] + r.dcnt[static_cast<size_t>(d)];
      for (int64_t p = r.off[static_cast<size_t>(d)]; p < r.off[static_cast<size_t>(d) + 1]; ++p) {
        stid.push_back(r.tid[static_cast<size_t>(p)]);
        max_term = std::max(max_term, r.tid[static_cast<size_t>(p)]);
      }
    }
    const int64_t total = soff[m];
    const uint2* from = src + (ns > 1 ? sbase[static_cast<size_t>(s)] : 0);
    const int vdev = v->device, sdev = kw_device(stores[s]);
    const KwRows rows{sid.data(), su.data(), so.data(), soff.data(), stid.data(), slen.data(), static_cast<int64_t>(m), total,
                      max_term};
    rc = kw_append_rows(stores[s], rows, [&](uint2* dst, cudaStream_t st) -> cudaError_t {
      if (!total) return cudaSuccess;
      if (sdev == vdev) return cudaMemcpyAsync(dst, from, static_cast<size_t>(total) * 8, cudaMemcpyDeviceToDevice, st);
      return cudaMemcpyPeerAsync(dst, sdev, from, vdev, static_cast<size_t>(total) * 8, st);
    });
  }
  return rc;
}

}  // namespace

extern "C" {

int aur_kw_vocab_open(int32_t device, aur_kw_vocab** out) {
  if (!out) return report_error(AUR_ERR_INVALID, "null argument");
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess) { cudaGetLastError(); ndev = 0; }
  if (ndev == 0) return report_error(AUR_ERR_NO_DEVICE, "no CUDA device: aurora_b200 has no CPU fallback");
  if (device < 0 || device >= ndev) return report_error(AUR_ERR_INVALID, "device %d out of range", device);
  AUR_TRY(cudaSetDevice(device));
  cudaDeviceProp prop;
  AUR_TRY(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9) return report_error(AUR_ERR_UNSUPPORTED, "sm_%d%d device: this library is built for sm_90a only", prop.major, prop.minor);
  std::unique_ptr<aur_kw_vocab> v(new aur_kw_vocab());
  v->device = device;
  const cudaError_t e = [&]() -> cudaError_t {
    AUR_CU_RET(v->stream.create(cudaStreamNonBlocking));
    AUR_CU_RET(v->woff.reserve(1024));
    AUR_CU_RET(cudaMemsetAsync(v->woff.p, 0, 8, v->stream));
    AUR_CU_RET(v->pool.reserve(1 << 16));
    return cudaStreamSynchronize(v->stream);
  }();
  if (e != cudaSuccess)
    return report_error(e == cudaErrorMemoryAllocation ? AUR_ERR_NOMEM : AUR_ERR_CUDA, "aur_kw_vocab_open: %s", cudaGetErrorString(e));
  const int rc = ensure_table(v.get(), 0);
  if (rc != AUR_OK) return rc;
  *out = v.release();
  return AUR_OK;
}

int aur_kw_vocab_close(aur_kw_vocab* v) {
  if (!v) return AUR_OK;
  cudaSetDevice(v->device);
  if (v->stream) cudaStreamSynchronize(v->stream);
  delete v;
  return AUR_OK;
}

int aur_kw_vocab_size(aur_kw_vocab* v, int64_t* words, int64_t* bytes) {
  if (!v) return report_error(AUR_ERR_INVALID, "null vocabulary");
  std::lock_guard<std::mutex> lk(v->mu);
  if (words) *words = v->words;
  if (bytes) *bytes = v->bytes;
  return AUR_OK;
}

int aur_kw_vocab_read(aur_kw_vocab* v, int64_t id0, int64_t n, char* bytes_out, int64_t bytes_cap, int64_t* offsets_out) {
  if (!v || !offsets_out) return report_error(AUR_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(v->mu);
  if (id0 < 0 || n < 0 || id0 + n > v->words)
    return report_error(AUR_ERR_INVALID, "words [%lld, %lld) outside the vocabulary's %lld", (long long)id0, (long long)(id0 + n),
                        (long long)v->words);
  std::vector<int64_t> wo(static_cast<size_t>(n) + 1);
  AUR_TRY(cudaSetDevice(v->device));
  AUR_TRY(cudaMemcpyAsync(wo.data(), v->woff.p + id0, wo.size() * 8, cudaMemcpyDeviceToHost, v->stream));
  AUR_TRY(cudaStreamSynchronize(v->stream));
  const int64_t nbytes = wo.back() - wo[0];
  if (bytes_out && bytes_cap < nbytes)
    return report_error(AUR_ERR_INVALID, "bytes_cap %lld < %lld bytes", (long long)bytes_cap, (long long)nbytes);
  if (bytes_out && nbytes) {
    AUR_TRY(cudaMemcpyAsync(bytes_out, v->pool.p + wo[0], static_cast<size_t>(nbytes), cudaMemcpyDeviceToHost, v->stream));
    AUR_TRY(cudaStreamSynchronize(v->stream));
  }
  for (int64_t i = 0; i <= n; ++i) offsets_out[i] = wo[static_cast<size_t>(i)] - wo[0];
  return AUR_OK;
}

int aur_kw_vocab_set_option(aur_kw_vocab* v, const char* name, int64_t value) {
  if (!v || !name) return report_error(AUR_ERR_INVALID, "null argument");
  if (strcmp(name, "hash_bits") == 0) {
    if (value < 1 || value > 64) return report_error(AUR_ERR_INVALID, "hash_bits must be in 1 .. 64");
    std::lock_guard<std::mutex> lk(v->mu);
    if (v->words) return report_error(AUR_ERR_INVALID, "hash_bits is set on an empty vocabulary only");
    v->hash_bits = static_cast<int>(value);
    return AUR_OK;
  }
  return report_error(AUR_ERR_INVALID, "unknown vocabulary option '%s'", name);
}

int aur_kw_add_text(aur_kw* const* stores, int32_t n_stores, aur_kw_vocab* v, const int64_t* ids, const int32_t* user_codes,
                    const int32_t* org_codes, const char* texts_utf8, const int64_t* text_offsets, int64_t n) {
  if (!stores || !v) return report_error(AUR_ERR_INVALID, "null argument");
  if (n_stores < 1 || n_stores > kMaxStores) return report_error(AUR_ERR_INVALID, "n_stores must be in 1 .. %d", kMaxStores);
  for (int32_t s = 0; s < n_stores; ++s) if (!stores[s]) return report_error(AUR_ERR_INVALID, "store %d is NULL", s);
  std::vector<aur_kw*> order(stores, stores + n_stores);
  std::sort(order.begin(), order.end(), std::less<aur_kw*>());
  if (std::adjacent_find(order.begin(), order.end()) != order.end()) return report_error(AUR_ERR_INVALID, "a store is listed twice");
  if (n < 0) return report_error(AUR_ERR_INVALID, "n < 0");
  if (n == 0) return AUR_OK;
  if (n > 0x7FFFFFFFll) return report_error(AUR_ERR_INVALID, "n > 2^31 - 1");
  if (!ids || !text_offsets) return report_error(AUR_ERR_INVALID, "ids and text_offsets are required");
  if (text_offsets[0] != 0) return report_error(AUR_ERR_INVALID, "text_offsets[0] must be 0");
  for (int64_t i = 0; i < n; ++i) {
    if (ids[i] < 0) return report_error(AUR_ERR_INVALID, "ids must be >= 0");
    if (text_offsets[i + 1] < text_offsets[i]) return report_error(AUR_ERR_INVALID, "text_offsets must be non-decreasing");
    if (text_offsets[i + 1] - text_offsets[i] > kMaxDocBytes) return report_error(AUR_ERR_INVALID, "a text is longer than 2^31 - 1 bytes");
  }
  if (text_offsets[n] > text_offsets[0] && !texts_utf8) return report_error(AUR_ERR_INVALID, "texts_utf8 is required");
  // writers: every store's mu_write in address order, then the vocabulary's mutex; each store's rw inside
  // kw_append_rows (searches hold only rw, so none waits on anything this call holds before rw)
  std::vector<std::unique_lock<std::mutex>> wl;
  for (aur_kw* kw : order) wl.emplace_back(kw_write_mutex(kw));
  std::vector<int64_t> per(static_cast<size_t>(n_stores), 0);
  for (int64_t i = 0; i < n; ++i) ++per[static_cast<size_t>(ids[i] % n_stores)];
  for (int32_t s = 0; s < n_stores; ++s) {
    const int rc = kw_check_room(stores[s], per[static_cast<size_t>(s)]);
    if (rc != AUR_OK) return rc;
  }
  std::lock_guard<std::mutex> vl(v->mu);
  AUR_TRY(cudaSetDevice(v->device));
  int rc = AUR_OK;
  SliceRows rows;
  std::vector<int64_t> soff;
  for (int64_t d0 = 0; d0 < n && rc == AUR_OK;) {   // slices of whole documents, at least one each
    int64_t d1 = d0 + 1;
    while (d1 < n && d1 - d0 < 0x7FFFFFFF && text_offsets[d1 + 1] - text_offsets[d0] <= kSliceBytes) ++d1;
    const int32_t m = static_cast<int32_t>(d1 - d0);
    soff.resize(static_cast<size_t>(m) + 1);
    for (int32_t i = 0; i <= m; ++i) soff[static_cast<size_t>(i)] = text_offsets[d0 + i] - text_offsets[d0];
    AUR_TRY(cudaSetDevice(v->device));
    rc = analyse(v, soff[m] ? texts_utf8 + text_offsets[d0] : nullptr, soff.data(), m, &rows);
    if (rc == AUR_OK)
      rc = publish(v, stores, n_stores, ids + d0, user_codes ? user_codes + d0 : nullptr, org_codes ? org_codes + d0 : nullptr,
                   m, rows);
    d0 = d1;
  }
  for (int32_t s = 0; s < n_stores; ++s) kw_after_append(stores[s], rc);
  return rc;
}

}  // extern "C"
