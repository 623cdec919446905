// WordPiece tokenisation for the uncased / cased BERT vocabularies (all-MiniLM-L6-v2, bge-*-en): text -> token
// ids, multi-threaded, behind the C ABI (aur_tokenizer_*, aur_tokenize, aur_encode_text_append).
//
// In the reference this runs inside the t2v-transformers sidecar: the application posts raw text
// (server/services/correlation/embedding_client.py:52-59) or lets Weaviate vectorise a property
// (server/routes/knowledge_base/weaviate_client.py:113-126, :252-259).  The algorithm is the published BERT
// one, with the exact semantics of the `tokenizers` BertNormalizer + BertPreTokenizer + WordPiece that
// transformers.BertTokenizer wraps (tests/test_tokenizer_native.py compares ids with it):
//   clean      drop U+0000, U+FFFD and Cc / Cf / Co (except TAB, LF, CR); White_Space -> ' '
//   cjk        every CJK ideograph becomes its own word
//   accents    NFD, drop Mn            (uncased vocabularies)
//   lower      per-character full lower-casing (no final-sigma rule -- like the Rust implementation)
//   split      on whitespace, then every punctuation character is its own word
//   wordpiece  greedy longest-match-first, "##" continuation pieces, > 100 characters or no match -> [UNK]
//   encode     [CLS] pieces [SEP], truncated to max_len ids
// Unicode properties come from tables generated out of Python's unicodedata (tools/gen_unicode_tables.py).
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/aurora_b200.h"
#include "internal.h"

namespace {
#include "unicode_tables.inc"

template <size_t N>
bool in_ranges(const uint32_t (&tab)[N][2], uint32_t cp) {
  size_t lo = 0, hi = N;
  while (lo < hi) {
    const size_t mid = (lo + hi) / 2;
    if (cp < tab[mid][0]) hi = mid; else if (cp > tab[mid][1]) lo = mid + 1; else return true;
  }
  return false;
}

inline bool is_cjk(uint32_t cp) {
  return (cp >= 0x4E00 && cp <= 0x9FFF) || (cp >= 0x3400 && cp <= 0x4DBF) || (cp >= 0x20000 && cp <= 0x2A6DF) ||
         (cp >= 0x2A700 && cp <= 0x2B73F) || (cp >= 0x2B740 && cp <= 0x2B81F) || (cp >= 0x2B820 && cp <= 0x2CEAF) ||
         (cp >= 0xF900 && cp <= 0xFAFF) || (cp >= 0x2F800 && cp <= 0x2FA1F);
}

template <size_t N>
const uint32_t* find_fold(const uint32_t (&index)[N][3], uint32_t cp) {
  size_t lo = 0, hi = N;
  while (lo < hi) {
    const size_t mid = (lo + hi) / 2;
    if (index[mid][0] < cp) lo = mid + 1; else hi = mid;
  }
  return (lo < N && index[lo][0] == cp) ? index[lo] : nullptr;
}

// NFD, drop Mn, lower-case: one code point of an uncased vocabulary's text, appended to out.
void fold_cp(uint32_t cp, std::vector<uint32_t>& out) {
  if (cp < 0x80) { out.push_back(cp >= 'A' && cp <= 'Z' ? cp + 32 : cp); return; }
  if (cp >= 0xAC00 && cp <= 0xD7A3) {   // Hangul syllable: algorithmic canonical decomposition (jamo are Lo: kept)
    const uint32_t s = cp - 0xAC00;
    out.push_back(0x1100 + s / 588);
    out.push_back(0x1161 + (s % 588) / 28);
    if (s % 28) out.push_back(0x11A7 + s % 28);
    return;
  }
  const uint32_t* e = find_fold(kFoldLowerIndex, cp);
  if (!e) { out.push_back(cp); return; }
  for (uint32_t i = 0; i < e[2]; ++i) out.push_back(kFoldLowerData[e[1] + i]);
}

// Lenient UTF-8 decoder: malformed bytes become U+FFFD (which clean-up then drops, like any replacement char).
inline uint32_t next_cp(const unsigned char* s, size_t n, size_t& i) {
  const unsigned char c = s[i];
  if (c < 0x80) { ++i; return c; }
  int len = (c >= 0xF0 && c <= 0xF4) ? 4 : (c >= 0xE0) ? 3 : (c >= 0xC2 && c < 0xE0) ? 2 : 0;
  if (len == 0 || i + len > n) { ++i; return 0xFFFD; }
  uint32_t cp = c & (0xFF >> (len + 1));
  for (int k = 1; k < len; ++k) {
    if ((s[i + k] & 0xC0) != 0x80) { ++i; return 0xFFFD; }
    cp = (cp << 6) | (s[i + k] & 0x3F);
  }
  i += len;
  if ((len == 3 && cp < 0x800) || (len == 4 && (cp < 0x10000 || cp > 0x10FFFF)) || (cp >= 0xD800 && cp <= 0xDFFF)) return 0xFFFD;
  return cp;
}

inline void append_utf8(std::string& s, uint32_t cp) {
  if (cp < 0x80) s.push_back(static_cast<char>(cp));
  else if (cp < 0x800) { s.push_back(static_cast<char>(0xC0 | (cp >> 6))); s.push_back(static_cast<char>(0x80 | (cp & 0x3F))); }
  else if (cp < 0x10000) {
    s.push_back(static_cast<char>(0xE0 | (cp >> 12))); s.push_back(static_cast<char>(0x80 | ((cp >> 6) & 0x3F)));
    s.push_back(static_cast<char>(0x80 | (cp & 0x3F)));
  } else {
    s.push_back(static_cast<char>(0xF0 | (cp >> 18))); s.push_back(static_cast<char>(0x80 | ((cp >> 12) & 0x3F)));
    s.push_back(static_cast<char>(0x80 | ((cp >> 6) & 0x3F))); s.push_back(static_cast<char>(0x80 | (cp & 0x3F)));
  }
}

struct AsciiClass {
  uint8_t cls[128];
  AsciiClass() {
    for (uint32_t c = 0; c < 128; ++c)
      cls[c] = in_ranges(kRemoved, c) ? 1 : in_ranges(kSpace, c) ? 2 : in_ranges(kPunct, c) ? 3 : 0;
  }
};
const AsciiClass kAscii;

}  // namespace

// Worker threads that live as long as the tokenizer: a batch of a few hundred chunks tokenises in well under a
// millisecond, less than it costs to create the threads for it.  One dispatch at a time (run() returns false when
// another caller holds the pool: that caller tokenises inline).
struct TokPool {
  std::vector<std::thread> threads;
  std::mutex m, run_m;
  std::condition_variable cv, done_cv;
  const std::function<void()>* job = nullptr;
  uint64_t gen = 0;
  int pending = 0;
  bool stop = false;
  void start(int n) {
    for (int i = 0; i < n; ++i)
      threads.emplace_back([this] {
        uint64_t seen = 0;
        for (;;) {
          const std::function<void()>* j;
          {
            std::unique_lock<std::mutex> lk(m);
            cv.wait(lk, [&] { return stop || gen != seen; });
            if (stop) return;
            seen = gen; j = job;
          }
          (*j)();
          {
            std::lock_guard<std::mutex> lk(m);
            if (--pending == 0) done_cv.notify_all();
          }
        }
      });
  }
  bool run(const std::function<void()>& work) {          // every worker (and the caller) runs `work` once
    std::unique_lock<std::mutex> rl(run_m, std::try_to_lock);
    if (!rl.owns_lock() || threads.empty()) return false;
    {
      std::lock_guard<std::mutex> lk(m);
      job = &work; pending = static_cast<int>(threads.size()); ++gen;
    }
    cv.notify_all();
    work();
    std::unique_lock<std::mutex> lk(m);
    done_cv.wait(lk, [&] { return pending == 0; });
    return true;
  }
  ~TokPool() {
    { std::lock_guard<std::mutex> lk(m); stop = true; }
    cv.notify_all();
    for (auto& t : threads) t.join();
  }
};

struct aur_tokenizer {
  TokPool pool;
  std::once_flag pool_once;
  std::unordered_map<std::string, int32_t> vocab;
  bool lower = true;
  int32_t unk = -1, cls = -1, sep = -1;
  int max_chars_per_word = 100;

  // One word (code points, already normalised) -> piece ids appended to out.
  void wordpiece(const uint32_t* w, size_t n, std::vector<int32_t>& out, std::string& buf, std::vector<uint32_t>& offs) const {
    if (static_cast<int>(n) > max_chars_per_word) { out.push_back(unk); return; }
    // UTF-8 of the whole word once, with the byte offset of every character
    buf.clear(); offs.clear();
    for (size_t i = 0; i < n; ++i) { offs.push_back(static_cast<uint32_t>(buf.size())); append_utf8(buf, w[i]); }
    offs.push_back(static_cast<uint32_t>(buf.size()));
    const size_t first = out.size();
    size_t start = 0;
    std::string piece;
    while (start < n) {
      size_t end = n;
      int32_t cur = -1;
      while (start < end) {
        piece.clear();
        if (start > 0) piece.append("##");
        piece.append(buf, offs[start], offs[end] - offs[start]);
        auto it = vocab.find(piece);
        if (it != vocab.end()) { cur = it->second; break; }
        --end;
      }
      if (cur < 0) { out.resize(first); out.push_back(unk); return; }   // one unknown piece makes the whole word [UNK]
      out.push_back(cur);
      start = end;
    }
  }

  // text -> [CLS] pieces [SEP], at most body_max pieces.
  void encode(const unsigned char* s, size_t n, size_t body_max, std::vector<int32_t>& out) const {
    out.clear();
    out.push_back(cls);
    std::vector<uint32_t> word, offs;
    std::string buf;
    auto flush = [&]() {
      if (!word.empty() && out.size() - 1 < body_max) wordpiece(word.data(), word.size(), out, buf, offs);
      word.clear();
    };
    std::vector<uint32_t> folded;
    size_t i = 0;
    while (i < n && out.size() - 1 < body_max) {
      if (s[i] < 0x80) {   // ASCII fast path: one table look-up per character (0 other, 1 removed, 2 space, 3 punctuation)
        const unsigned char c = s[i++];
        const uint8_t cls_ = kAscii.cls[c];
        if (cls_ == 0) word.push_back(lower && c >= 'A' && c <= 'Z' ? c + 32u : c);
        else if (cls_ == 2) flush();
        else if (cls_ == 3) { flush(); word.push_back(c); flush(); }
        continue;
      }
      const uint32_t cp = next_cp(s, n, i);
      if (in_ranges(kRemoved, cp)) continue;
      if (in_ranges(kSpace, cp)) { flush(); continue; }
      folded.clear();
      if (lower) fold_cp(cp, folded); else folded.push_back(cp);
      if (is_cjk(cp)) {   // isolated first, normalised second (compatibility ideographs fold to the unified ones)
        flush();
        for (uint32_t f : folded) word.push_back(f);
        flush();
        continue;
      }
      for (uint32_t f : folded) {
        if (in_ranges(kPunct, f)) { flush(); word.push_back(f); flush(); }
        else word.push_back(f);
      }
    }
    flush();
    if (out.size() - 1 > body_max) out.resize(body_max + 1);
    out.push_back(sep);
  }
};

// Every text through t->encode (at most body_max pieces each) into ids[i]: inline for n_threads == 1 or a handful of
// texts, otherwise on the tokenizer's resident workers (all host cores up to 64, started on first use); when another
// caller holds them, inline instead of waiting.
static void tokenize_all(aur_tokenizer* t, const char* texts_utf8, const int64_t* offsets, int32_t n_texts, size_t body_max,
                         std::vector<std::vector<int32_t>>& ids, int32_t n_threads) {
  std::atomic<int32_t> next{0};
  const std::function<void()> work = [&]() {
    for (;;) {
      const int32_t b = next.fetch_add(4);
      if (b >= n_texts) break;
      for (int32_t i = b; i < std::min(n_texts, b + 4); ++i)
        t->encode(reinterpret_cast<const unsigned char*>(texts_utf8) + offsets[i], static_cast<size_t>(offsets[i + 1] - offsets[i]), body_max, ids[i]);
    }
  };
  bool done = false;
  if (n_threads != 1 && n_texts > 4) {
    std::call_once(t->pool_once, [&] {
      const int hw = static_cast<int>(std::thread::hardware_concurrency());
      t->pool.start(std::max(1, std::min(hw > 0 ? hw : 8, 64) - 1));
    });
    done = t->pool.run(work);
  }
  if (!done) work();
}

extern "C" {

int aur_tokenizer_open_mem(const char* vocab_utf8, int64_t nbytes, int32_t lower_case, aur_tokenizer** out) {
  if (!vocab_utf8 || nbytes <= 0 || !out) return aur::report_error(AUR_ERR_INVALID, "null / empty vocabulary");
  *out = nullptr;
  aur_tokenizer* t = new aur_tokenizer();
  t->lower = lower_case != 0;
  // later duplicates overwrite earlier ones in a Python dict built from enumerate(lines): emulate by inserting in
  // reverse so that emplace (first wins) keeps the LAST line's id ... but ids must stay line numbers
  {
    std::vector<std::pair<size_t, size_t>> lines;
    size_t i = 0, n = static_cast<size_t>(nbytes);
    while (i < n) {
      size_t j = i;
      while (j < n && vocab_utf8[j] != '\n') ++j;
      size_t e = j;
      if (e > i && vocab_utf8[e - 1] == '\r') --e;
      lines.emplace_back(i, e - i);
      i = j + 1;
    }
    for (size_t k = lines.size(); k-- > 0;) t->vocab.emplace(std::string(vocab_utf8 + lines[k].first, lines[k].second), static_cast<int32_t>(k));
  }
  auto get = [&](const char* name) { auto it = t->vocab.find(name); return it == t->vocab.end() ? -1 : it->second; };
  t->unk = get("[UNK]"); t->cls = get("[CLS]"); t->sep = get("[SEP]");
  if (t->unk < 0 || t->cls < 0 || t->sep < 0) { delete t; return aur::report_error(AUR_ERR_INVALID, "vocabulary lacks [UNK] / [CLS] / [SEP]"); }
  *out = t;
  return AUR_OK;
}

int aur_tokenizer_open(const char* vocab_path, int32_t lower_case, aur_tokenizer** out) {
  if (!vocab_path || !out) return aur::report_error(AUR_ERR_INVALID, "null argument");
  FILE* f = fopen(vocab_path, "rb");
  if (!f) return aur::report_error(AUR_ERR_INVALID, "cannot open vocabulary file %s", vocab_path);
  std::string data;
  char chunk[65536];
  size_t got;
  while ((got = fread(chunk, 1, sizeof chunk, f)) > 0) data.append(chunk, got);
  fclose(f);
  return aur_tokenizer_open_mem(data.data(), static_cast<int64_t>(data.size()), lower_case, out);
}

int aur_tokenizer_close(aur_tokenizer* t) { delete t; return AUR_OK; }

int aur_tokenizer_info(aur_tokenizer* t, int32_t* vocab_size, int32_t* unk_id, int32_t* cls_id, int32_t* sep_id) {
  if (!t) return aur::report_error(AUR_ERR_INVALID, "null tokenizer");
  if (vocab_size) *vocab_size = static_cast<int32_t>(t->vocab.size());
  if (unk_id) *unk_id = t->unk;
  if (cls_id) *cls_id = t->cls;
  if (sep_id) *sep_id = t->sep;
  return AUR_OK;
}

int aur_tokenize(aur_tokenizer* t, const char* texts_utf8, const int64_t* offsets, int32_t n_texts, int32_t max_len,
                 int32_t* tokens_out, int64_t tokens_cap, int32_t* cu_seqlens_out, int32_t n_threads) {
  if (!t || !offsets || !cu_seqlens_out || n_texts < 0 || (n_texts > 0 && !texts_utf8 && offsets[n_texts] > 0))
    return aur::report_error(AUR_ERR_INVALID, "null argument");
  if (max_len < 2) return aur::report_error(AUR_ERR_INVALID, "max_len must be >= 2 ([CLS] and [SEP])");
  std::vector<std::vector<int32_t>> ids(static_cast<size_t>(n_texts));
  tokenize_all(t, texts_utf8, offsets, n_texts, static_cast<size_t>(max_len - 2), ids, n_threads);
  int64_t total = 0;
  cu_seqlens_out[0] = 0;
  for (int32_t i = 0; i < n_texts; ++i) {
    total += static_cast<int64_t>(ids[i].size());
    if (total > 0x7FFFFFFFll) return aur::report_error(AUR_ERR_INVALID, "more than 2^31 tokens in one call");
    cu_seqlens_out[i + 1] = static_cast<int32_t>(total);
  }
  if (!tokens_out && tokens_cap == 0) return AUR_OK;      // count mode: only the lengths (cu_seqlens_out) were asked for
  if (total > tokens_cap || (total > 0 && !tokens_out))
    return aur::report_error(AUR_ERR_NOMEM, "tokens_out holds %lld ids, %lld needed (n_texts * max_len always suffices)", (long long)tokens_cap, (long long)total);
  for (int32_t i = 0; i < n_texts; ++i)
    if (!ids[i].empty()) memcpy(tokens_out + cu_seqlens_out[i], ids[i].data(), ids[i].size() * 4);
  return AUR_OK;
}

int aur_tokenize_windows(aur_tokenizer* t, const char* texts_utf8, const int64_t* offsets, int32_t n_texts, int32_t max_len,
                         int32_t* tokens_out, int64_t tokens_cap, int32_t* cu_seqlens_out, int32_t seqs_cap,
                         int32_t* cu_texts_out, int64_t* totals_out, int32_t n_threads) {
  if (!t || !offsets || !cu_texts_out || n_texts < 0 || (n_texts > 0 && !texts_utf8 && offsets[n_texts] > 0))
    return aur::report_error(AUR_ERR_INVALID, "null argument");
  if (max_len < 3) return aur::report_error(AUR_ERR_INVALID, "max_len must be >= 3 ([CLS], one piece, [SEP])");
  if (tokens_cap < 0 || seqs_cap < 0) return aur::report_error(AUR_ERR_INVALID, "negative capacity");
  std::vector<std::vector<int32_t>> ids(static_cast<size_t>(n_texts));
  tokenize_all(t, texts_utf8, offsets, n_texts, SIZE_MAX, ids, n_threads);   // the whole text: [CLS] b [SEP]
  const int64_t step = max_len - 2;
  int64_t windows = 0, total = 0;
  cu_texts_out[0] = 0;
  for (int32_t i = 0; i < n_texts; ++i) {
    const int64_t body = static_cast<int64_t>(ids[i].size()) - 2;
    const int64_t w = body <= step ? 1 : (body + step - 1) / step;
    windows += w;
    total += body + 2 * w;
    if (windows > 0x7FFFFFFFll || total > 0x7FFFFFFFll) return aur::report_error(AUR_ERR_INVALID, "more than 2^31 windows or tokens in one call");
    cu_texts_out[i + 1] = static_cast<int32_t>(windows);
  }
  if (totals_out) { totals_out[0] = windows; totals_out[1] = total; }
  if (!tokens_out && tokens_cap == 0 && !cu_seqlens_out && seqs_cap == 0) return AUR_OK;   // count mode
  if (windows > seqs_cap || total > tokens_cap || !cu_seqlens_out || (total > 0 && !tokens_out))
    return aur::report_error(AUR_ERR_NOMEM, "%lld windows of %lld tokens, the buffers hold %d and %lld", (long long)windows,
                             (long long)total, seqs_cap, (long long)tokens_cap);
  int64_t at = 0, k = 0;
  cu_seqlens_out[0] = 0;
  for (int32_t i = 0; i < n_texts; ++i) {
    const std::vector<int32_t>& v = ids[i];
    const int64_t body = static_cast<int64_t>(v.size()) - 2;
    int64_t b = 0;
    do {   // [CLS] b[b0 : b0 + step] [SEP]; a text that fits is one window, aur_tokenize's output
      const int64_t len = std::min(step, body - b);
      tokens_out[at] = v.front();
      if (len > 0) memcpy(tokens_out + at + 1, v.data() + 1 + b, static_cast<size_t>(len) * 4);
      tokens_out[at + 1 + len] = v.back();
      at += len + 2;
      cu_seqlens_out[++k] = static_cast<int32_t>(at);
      b += step;
    } while (b < body);
  }
  return AUR_OK;
}

int aur_encode_text_append(aur_encoder* enc, aur_tokenizer* tok, aur_index* ix, const char* texts_utf8, const int64_t* offsets,
                           int32_t n_texts, int32_t max_len, int32_t max_tokens_per_call, int32_t max_seqs_per_call,
                           const int64_t* ids, const int32_t* user_codes, const int32_t* org_codes, int32_t n_threads) {
  if (!enc || !tok || !ix || !ids) return aur::report_error(AUR_ERR_INVALID, "null argument");
  if (n_texts <= 0) return AUR_OK;
  if (max_len < 2 || max_len > 512) return aur::report_error(AUR_ERR_INVALID, "max_len must be 2..512 (BERT position table)");
  if (max_tokens_per_call < max_len || max_seqs_per_call < 1) return aur::report_error(AUR_ERR_INVALID, "per-call limits smaller than one sequence");
  std::vector<int32_t> tokens(static_cast<size_t>(n_texts) * max_len);
  std::vector<int32_t> cu(static_cast<size_t>(n_texts) + 1);
  int rc = aur_tokenize(tok, texts_utf8, offsets, n_texts, max_len, tokens.data(), static_cast<int64_t>(tokens.size()), cu.data(), n_threads);
  if (rc != AUR_OK) return rc;
  return aur_encode_append_multi(&enc, &ix, 1, tokens.data(), cu.data(), n_texts, ids, user_codes, org_codes,
                                 max_tokens_per_call, max_seqs_per_call);
}

}  // extern "C"
