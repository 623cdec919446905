// Fused similarity + top-k for sm_90a: S = Q . C^T on wgmma tensor cores with the query
// block resident on the SM (shared memory, and for 128-row tiles its first k-blocks in the MMA warpgroup's registers),
// the corpus streamed once from HBM by TMA, and a per-query candidate list kept in shared memory by the epilogue warps.
//
// Replaces the dense leg of collection.query.hybrid(...) / near_text(...) that the
// reference sends to Weaviate (server/routes/knowledge_base/weaviate_client.py:252-259,
// server/routes/incident_feedback/weaviate_client.py:286-291).
//
// Tile width N = 64 or 128 corpus rows (kTileN, chosen per launch on the host, tc_auto_tile in capi.cu): 128 when its
// layout with the whole query block in shared memory keeps at least four 16 KB ring stages, else 64.  The wide tile runs
// wgmma m64n128k16: the query operand is fetched once per 128 corpus rows instead of once per 64, and the drain,
// score-buffer hand-off and threshold read happen once per 128 rows.  Its epilogue examines a tile 64 scores at a time
// with the 64-row code.  A wide launch then keeps its first kTcQRegs query k-blocks as wgmma's register A operand (kQReg,
// when dim / 64 has that many) and spends the 8 KB of shared memory each one leaves on the ring: at dim 768 / top-32
// seven 16 KB stages against the eight 8 KB ones of the 64-row kernel, in the same footprint as four.
//
// One CTA, persistent, 1 CTA / SM:
//   warps 1..2   epilogue  : thread r of the two warps owns query r (score-buffer row r): reads its N scores of a
//                            tile, scales them by the rows' inverse norms, keeps one max per 16 scores and
//                            compares it with the query's threshold; a four-score group that reaches it is
//                            parked in a per-thread FIFO in shared memory and examined later, out of line and
//                            rarely (drain_fifo); large k without room for the FIFO pushes at once (push_group4).
//   warp 0      threshold  : serves the certified global threshold of the queries assigned to this CTA (see
//                            "Threshold exchange").
//   warp 3      TMA producer: corpus tiles [N rows x 64 k] -> smem ring (SWIZZLE_128B)
//   warps 4..7  MMA        : wgmma m64nNk16, A = the CTA's 64 queries (K-major tiles in shared memory; k-blocks
//                            0 .. kQReg - 1 as register fragments loaded once from global memory), B =
//                            corpus tile from the ring; the [64 queries x N rows] fp32 accumulator lives in
//                            registers for the whole tile and is then stored to a padded score buffer that the
//                            epilogue warps read row-wise.  The MMA of the next tile runs while the epilogue
//                            works on the buffer it just released.
// Two-CTA clusters (AUR_KERNEL_TC2): the pair shares every corpus tile -- each CTA TMA-loads N / 2 of the N rows and
// multicasts them to both, so a tile crosses L2 -> SM once per pair; each CTA scores its own 64 queries.
// Single CTAs: when nq > 64 several CTAs take the same tiles for different query blocks (sharing through L2).
//
// Threshold exchange.  A CTA sees only a slice of the corpus, so its own k-th best is a loose
// filter.  Every epilogue thread therefore publishes its best (or 2nd best) score so far
// into a [query][CTA] table.  Query q is served by one CTA of its query block: its threshold
// warp reads the row of q every couple of microseconds, takes the R-th largest entry (R * m >= k +
// slack) and publishes it: at least k + slack rows with a score >= that value exist
// somewhere, so nothing below it can reach the final top-k.  Every epilogue thread reads its
// query's current threshold once per tile.  A query then admits only a handful of rows per
// CTA over a 1M-row scan.
//
// Bootstrap.  On its first tile a thread only publishes the tile's best score and waits for
// the first certified threshold (all CTAs do this at the same time, once), then
// examines the tile against it: no arbitrary rows ever enter a list.
//
// Candidate list.  Append-only, ksel slots per query.  If it fills up it is compacted:
// entries under the current threshold are dropped, and only if ksel live candidates remain
// does it fall back to replace-the-minimum.  At the end the survivors are appended to the
// query's compact row in global memory for the finalize kernel.
#include <cuda.h>
#include "internal.h"
#include "ptx.cuh"

// Bring-up timers compile to nothing unless the library is built with AUR_TC_PROFILE=1: every
// clock64() is a scheduling barrier inside the hot loops.
#ifdef AUR_TC_PROFILE
#define TCLK() clock64()
#else
#define TCLK() 0ll
#endif

namespace aur {
using namespace ptx;

namespace {

// warps: threshold, two epilogue, producer, then the MMA warpgroup at the next multiple of four: 8 warps, two per SM
// sub-partition, up to 255 registers a thread (no spills).
constexpr int kThrWarps = 1;
constexpr int kEpiWarps = 2;
constexpr int kProducerWarp = kThrWarps + kEpiWarps;
constexpr int kMmaWarp0 = (kProducerWarp + 1 + 3) / 4 * 4;   // first warp of the MMA warpgroup (warpgroup-aligned)
constexpr int kThreads = 32 * (kMmaWarp0 + 4);
constexpr uint32_t kSlot = kTcQRows * 8u;   // byte stride between list slots of one query
constexpr uint32_t kQTileBytes = kTcQRows * 128u;   // one 64-dim k-block of the query block
// one 64-dim k-block of a corpus tile (a ring stage); floats per score-buffer row (padding spreads the banks)
__host__ __device__ constexpr uint32_t stage_bytes(int tile_n) { return static_cast<uint32_t>(tile_n) * 128u; }
__host__ __device__ constexpr int sc_stride(int tile_n) { return tile_n + 4; }
__host__ __device__ constexpr uint32_t sc_bytes(int tile_n) { return kTcQRows * sc_stride(tile_n) * 4u; }

struct SmemLayout {
  uint32_t lcap, fifo_recs;
  uint32_t off_qs, off_sc, off_list, off_norm, off_mask, off_fifo, off_tau, off_bar, total;
};
// The 128-row layout fits a fourth 16 KB ring stage at dim 768 / ksel 40 only without what the 64-row one can afford:
// it reserves the tenant-scope masks for kMask launches alone and parks half as many groups per thread in the FIFO.
// qregs: leading query k-blocks the MMA warpgroup keeps in registers; only the others have a tile at off_qs.
__host__ __device__ inline SmemLayout make_layout(int num_stages, int ksel, int dim, int tile_n, bool mask, int qregs) {
  SmemLayout L;
  const bool wide = tile_n == kTcTileWide;
  L.lcap = static_cast<uint32_t>(ksel);
  uint32_t o = stage_bytes(tile_n) * num_stages;
  // the query block: [64 queries x 64] bf16 K-major SWIZZLE_128B tiles, one per k-block (the wgmma A operand)
  L.off_qs = o;     o += static_cast<uint32_t>(dim / kTcKBlock - qregs) * kQTileBytes;
  L.off_sc = o;     o += sc_bytes(tile_n);
  L.off_list = o;   o += L.lcap * kSlot;
  L.off_norm = o;   o += 2u * 2u * tile_n * 4u;
  L.off_mask = o;   if (mask || !wide) o += 2u * 2u * tile_n * 4u;   // per-row tenant-scope bit masks (kMask launches)
  // deferred-candidate FIFO: per thread kTcFifoRecs records of four adjacent scores (16 B) + a row tag
  L.fifo_recs = ksel <= kTcFifoMaxKsel ? (wide ? kTcFifoRecs / 2 : kTcFifoRecs) : 0u;
  L.off_fifo = o;   o += L.fifo_recs * kTcQRows * (16u + 4u);
  L.off_tau = o;    o += kTcQRows * 4u;   // certified thresholds of this CTA's queries, refreshed by the threshold warp
  L.off_bar = o;    o += (2u * kTcMaxStages + 2u + 2u + 1u) * 8u + 16u;
  L.total = o;
  return L;
}

// Per-thread (= per-query) selection state of the epilogue.
struct TopkState {
  uint64_t min_key;   // smallest key, valid when the list holds exactly ksel entries (nfill == ksel)
  float tau_local;    // its score, else -inf
  float tau;          // admission filter = max(tau_local, certified global threshold)
  float top[4];       // best four chunk maxima seen so far (distinct rows), descending: top[xm - 1] is published
  int minpos, nfill;
};

// The last key of a list in candidate order (key_before): the one to evict.
__device__ __forceinline__ void scan_min(uint32_t list_a, int n, const int64_t* ids, uint64_t& m, int& mp) {
  m = lds_u64(list_a); mp = 0;
#pragma unroll 8
  for (int t = 1; t < n; ++t) {
    const uint64_t v = lds_u64(list_a + t * kSlot);
    if (key_before(m, v, ids)) { m = v; mp = t; }
  }
}

// Drop what the threshold has made useless, then cut down to ksel entries.
__device__ __noinline__ TopkState compact_list(TopkState st, uint32_t list_a, int ksel, const int64_t* ids) {
  const uint32_t thr = f32_to_ord(st.tau);
  int w = 0;
  for (int t = 0; t < st.nfill; ++t) {
    const uint64_t k = lds_u64(list_a + t * kSlot);
    if (static_cast<uint32_t>(k >> 32) >= thr) { sts_u64(list_a + w * kSlot, k); ++w; }
  }
  st.nfill = w;
  while (st.nfill > ksel) {  // rare: this CTA owns more than ksel of the current global best
    uint64_t m; int mp;
    scan_min(list_a, st.nfill, ids, m, mp);
    --st.nfill;
    sts_u64(list_a + mp * kSlot, lds_u64(list_a + st.nfill * kSlot));
  }
  if (st.nfill == ksel) {
    scan_min(list_a, ksel, ids, st.min_key, st.minpos);
    st.tau_local = key_score(st.min_key);
    st.tau = fmaxf(st.tau, st.tau_local);
  }
  return st;
}

// Admit one score into a query's list.
__device__ __forceinline__ TopkState push_one(TopkState st, float s, int row, uint32_t list_a, int ksel, int lcap,
                                              const int64_t* ids) {
  const uint64_t key = make_key(s, row);
  if (st.nfill == lcap) st = compact_list(st, list_a, ksel, ids);
  if (st.nfill < lcap) {
    sts_u64(list_a + st.nfill * kSlot, key);
    ++st.nfill;
  } else if (key_before(key, st.min_key, ids)) {  // lcap == ksel and the list is full of live candidates
    sts_u64(list_a + st.minpos * kSlot, key);
    scan_min(list_a, ksel, ids, st.min_key, st.minpos);
    st.tau_local = key_score(st.min_key);
    st.tau = fmaxf(st.tau, st.tau_local);
  }
  return st;
}

// Examine four adjacent scores of one query (their max reached the threshold).  Out of
// line and small: at warp level some lane needs this about twice per tile, so it has to be
// cheap and its code has to stay resident next to the hot loop.
__device__ __noinline__ TopkState push_group4(TopkState st, float s0, float s1, float s2, float s3, int row,
                                              uint32_t list_a, int ksel, const int64_t* ids) {
  if (s0 >= st.tau) st = push_one(st, s0, row + 0, list_a, ksel, ksel, ids);   // `>=` also rejects NaN
  if (s1 >= st.tau) st = push_one(st, s1, row + 1, list_a, ksel, ksel, ids);
  if (s2 >= st.tau) st = push_one(st, s2, row + 2, list_a, ksel, ksel, ids);
  if (s3 >= st.tau) st = push_one(st, s3, row + 3, list_a, ksel, ksel, ids);
  return st;
}

// Running best four of the per-16-row chunk maxima.  Every chunk maximum belongs to a different corpus row, so
// top[m - 1] >= v certifies "this CTA has m rows scoring at least v" -- what the threshold exchange needs when fewer
// than k + slack CTAs scan the corpus (m = ceil((k + slack) / CTAs), up to 4).  Branch-free insertion network.
__device__ __forceinline__ void top4_insert(float (&t)[4], float v) {   // v is never NaN (fmaxf drops NaN upstream)
  float a = v;
  const float n0 = fmaxf(t[0], a); a = fminf(t[0], a);
  const float n1 = fmaxf(t[1], a); a = fminf(t[1], a);
  const float n2 = fmaxf(t[2], a); a = fminf(t[2], a);
  t[3] = fmaxf(t[3], a); t[0] = n0; t[1] = n1; t[2] = n2;
}

__device__ __forceinline__ float top4_get(const float (&t)[4], int m) {   // t[m - 1] without dynamic register indexing
  return m == 1 ? t[0] : (m == 2 ? t[1] : (m == 3 ? t[2] : t[3]));
}

// Deferred slow path.  The hot loop only parks a group of four adjacent scores whose max reached the
// threshold (two predicated shared-memory stores); this routine runs when a thread's FIFO is nearly
// full and once at the end, re-tests the parked scores against the threshold as it stands NOW (usually
// much tighter) and admits the survivors.  The cold code is entered a handful of times per kernel
// instead of ~100x per warp, and fewer scores pass.
__device__ __noinline__ TopkState drain_fifo(TopkState st, uint32_t fifo_a, uint32_t ftag_a, int fcnt, uint32_t list_a,
                                             int ksel, const int64_t* ids) {
#pragma unroll 1
  for (int rec = 0; rec < fcnt; ++rec) {
    int row;
    float s0, s1, s2, s3;
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(row) : "r"(ftag_a + rec * (kTcQRows * 4u)));
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(s0), "=f"(s1), "=f"(s2), "=f"(s3)
                 : "r"(fifo_a + rec * (kTcQRows * 16u)));
    if (s0 >= st.tau) st = push_one(st, s0, row + 0, list_a, ksel, ksel, ids);   // `>=` also rejects NaN
    if (s1 >= st.tau) st = push_one(st, s1, row + 1, list_a, ksel, ksel, ids);
    if (s2 >= st.tau) st = push_one(st, s2, row + 2, list_a, ksel, ksel, ids);
    if (s3 >= st.tau) st = push_one(st, s3, row + 3, list_a, ksel, ksel, ids);
  }
  return st;
}

// Warp-cooperative: R-th largest of the values published for one query by up to 96 CTAs
// (lane i holds entries i, i+32, i+64; entries of other launches or not yet written are
// skipped).  Bisection on the value with ballot counts.  Returns -inf when fewer than R CTAs
// have published.  All lanes return the same value.  The three entries are loaded by the caller
// (exchange_load) so that several rows' loads can be in flight before any is consumed.
struct PubEntries { unsigned long long e[3]; };
__device__ __forceinline__ PubEntries exchange_load(const unsigned long long* pubrow, int nuse, int lane) {
  PubEntries r;
#pragma unroll
  for (int k = 0; k < 3; ++k) { const int i = lane + 32 * k; r.e[k] = (i < nuse) ? __ldcg(pubrow + i) : 0ull; }
  return r;
}
__device__ float exchange_select(const PubEntries& ent, int nuse, int R, uint32_t epoch, int lane) {
  float v[3];
  float lo = INFINITY, hi = -INFINITY;
  int nvalid = 0;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int i = lane + 32 * k;
    const unsigned long long e = ent.e[k];
    const bool ok = (i < nuse) && static_cast<uint32_t>(e >> 32) == epoch;
    v[k] = ok ? ord_to_f32(static_cast<uint32_t>(e)) : __int_as_float(0x7FC00000);
    nvalid += __popc(__ballot_sync(0xffffffffu, ok));
    lo = fminf(lo, v[k]); hi = fmaxf(hi, v[k]);   // fminf / fmaxf skip NaN
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  if (nvalid < R) return -INFINITY;
  // invariant: count(v >= lo) >= R
  for (int round = 0; round < 12; ++round) {
    const float mid = 0.5f * (lo + hi);
    int c = 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) c += __popc(__ballot_sync(0xffffffffu, v[k] >= mid));
    if (c >= R) lo = mid; else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ float read_threshold(const unsigned long long* tq, uint32_t epoch) {
  const unsigned long long e = __ldcg(tq);
  return (static_cast<uint32_t>(e >> 32) == epoch) ? __uint_as_float(static_cast<uint32_t>(e)) : -INFINITY;
}

// Publishes value v of this launch into a CTA's exchange slot.  The slot's first publish of a launch REPLACES the entry
// (atomicExch), later ones keep the max.  A plain atomicMax would never get past an entry that another launch left with
// a numerically larger tag -- a bring-up launch (upper half of the tags) or any search before the counter wrapped --
// and the exchange would stay without a valid value for that slot until the table is reallocated.
__device__ __forceinline__ void publish_value(unsigned long long* slot, uint32_t epoch, float v, bool first) {
  const unsigned long long e = (static_cast<unsigned long long>(epoch) << 32) | f32_to_ord(v);
  if (first) atomicExch(slot, e);
  else atomicMax(slot, e);
}

constexpr uint32_t kNaNBits = 0x7FC00000u;

// kMask: the queries of the batch carry different tenant scopes (user_id == u OR org_id == o,
// weaviate_client.py:244-249).  A pre-pass has written one 32-bit word per corpus row -- bit s set when scope s of the
// batch may see the row -- and every query knows its scope's bit: scores of invisible rows become NaN before anything
// else looks at them, exactly like tombstones.  (One scope for the whole batch needs none of this: it folds into the
// inverse norms.)
//
// kQReg: the first kQReg query k-blocks are the MMA warpgroup's register A operand instead of shared-memory tiles
// (128-row tiles only; the host launches it only when dim / 64 >= kQReg).  Every two of them free one 16 KB ring stage.
//
// kI8: int8 corpus rows (AUR_I8).  A corpus k-block is still one 128-byte swizzled row of a ring stage, now 128 int8
// (UINT8 tensor map), so a stage carries twice the dimensions.  p.q is then the query image of launch_query_image_i8:
// each query as q16 = 256 hi + lo (hi, lo int8), laid out [dim / 128][hi 128 B | lo 128 B], dim * 2 bytes a query like
// a bf16 query row -- the staging below copies it unchanged, so query tile 2 kb is hi and 2 kb + 1 is lo of corpus
// k-block kb.  Per k-block the MMA warpgroup issues 4 wgmma m64nNk32 s8 into acc_hi and 4 into acc_lo, one commit group,
// and hands the epilogue fmaf(acc_hi, 256, acc_lo): |acc| <= 127 * 128 * 1024 < 2^24, so both convert exactly and the
// combination rounds once.  That is q16 . c, the cosine times a positive per-query factor: every comparison the
// epilogue, the threshold exchange and the candidate keys make is between scores of one query, so nothing else changes.
//
// kDump: the score dump of aur_debug_tc_scores (unmasked launches only).  Every CTA writes its first tile's scores, as
// the epilogue sees them before any selection, to p.dbg_scores.  A separate instantiation, so the kernels searches run
// carry none of its code.
template <int kCtaGroup, bool kMask, int kTileN, int kQReg, bool kI8 = false, bool kDump = false>
__global__ void __launch_bounds__(kThreads, 1)
simtopk_tc_kernel(const __grid_constant__ CUtensorMap tmap, const TcParams p) {
  static_assert(kTileN == kTcTileN || kTileN == kTcTileWide, "tile width");
  static_assert(kQReg == 0 || kTileN == kTcTileWide, "register-resident query k-blocks: 128-row tiles only");
  static_assert(!(kI8 && kQReg), "int8 rows: query image in shared memory only");
  constexpr uint32_t kStageBytes = stage_bytes(kTileN);
  constexpr int kScStride = sc_stride(kTileN);
  constexpr int kHalves = kTileN / 64;   // the epilogue examines a tile 64 scores (four 16-score chunks) at a time
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // SWIZZLE_128B tiles need 1024-byte alignment; the runtime only guarantees 16.  Offsetting
  // the declared array (rather than round-tripping through an integer) keeps the compiler's
  // shared-address-space inference, i.e. LDS/STS instead of generic loads.
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);

  const SmemLayout L = make_layout(p.num_stages, p.ksel, p.dim, kTileN, kMask, kQReg);
  float* normbuf = reinterpret_cast<float*>(smem + L.off_norm);      // [2 warps][2][kTileN]
  uint32_t* maskbuf = reinterpret_cast<uint32_t*>(smem + L.off_mask);  // [2 warps][2][kTileN]
  float* scbuf = reinterpret_cast<float*>(smem + L.off_sc);          // [64 queries][kScStride]
  volatile float* tau_s = reinterpret_cast<volatile float*>(smem + L.off_tau);   // [64]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L.off_bar);
  uint64_t* full_bar = bars;                              // [kTcMaxStages]
  uint64_t* empty_bar = bars + kTcMaxStages;              // [kTcMaxStages]
  uint64_t* acc_full = bars + 2 * kTcMaxStages;           // [1] score buffer written
  uint64_t* acc_empty = bars + 2 * kTcMaxStages + 2;      // [1] score buffer read into registers
  uint64_t* q_ready = bars + 2 * kTcMaxStages + 4;        // [1] the query block is in shared memory
  volatile int* epi_done = reinterpret_cast<volatile int*>(bars + 2 * kTcMaxStages + 5);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t rank = (kCtaGroup == 2) ? cluster_ctarank() : 0u;
  // launch counter tagging the exchange-table entries: read from device memory (the finalize kernel behind this launch
  // bumps it) so that a captured CUDA graph advances by itself when replayed
  const uint32_t epoch = p.epoch_ptr ? *p.epoch_ptr : p.epoch;

  // Work split.  tset = which set of corpus tiles this CTA (pair) walks; qblock = which 64 queries.
  // With more than 128 queries in a launch, S = n_qblocks / 2 CTA pairs ("query super-blocks") walk the SAME tile set
  // side by side, each with its own 128 queries: the first pair to ask for a tile pulls it from HBM, its
  // siblings hit L2, so the corpus crosses the HBM interface once per 128 * S queries instead of once per 128.
  int qblock, tset, n_tsets;
  if constexpr (kCtaGroup == 2) {
    const int n_super = p.n_qblocks >> 1, pair = blockIdx.x >> 1;
    qblock = (pair % n_super) * 2 + static_cast<int>(rank);
    tset = pair / n_super;
    n_tsets = (gridDim.x >> 1) / n_super;
  } else {
    qblock = blockIdx.x % p.n_qblocks;
    tset = blockIdx.x / p.n_qblocks;
    n_tsets = gridDim.x / p.n_qblocks;
  }
  const int my_tiles = (p.n_tiles > tset) ? (p.n_tiles - tset + n_tsets - 1) / n_tsets : 0;
  const int kbs = p.dim / kTcKBlock;  // 128-byte k-blocks per query row (bf16 row, or int8 query image)
  const int kbs_c = kI8 ? p.dim / kTcKBlockI8 : kbs;   // 128-byte k-blocks per corpus row

  // exchange geometry: R-th largest of the m-th best of `nuse` CTAs is a valid threshold
  const int ksel = p.ksel;
  const int nuse = min(n_tsets, 96);
  const int xm = (ksel + nuse - 1) / nuse;            // rows every publishing CTA vouches for (1 .. 4)
  const int xR = (ksel + xm - 1) / xm;
  // (only CTAs that own at least one tile ever publish)
  const bool xchg = (p.pub != nullptr) && xm <= 4 && (xR <= min(nuse, p.n_tiles));

  if (warp == kProducerWarp && lane == 0) {
    prefetch_tmap(&tmap);
    for (int i = 0; i < p.num_stages; ++i) {
      mbar_init(&full_bar[i], 1);          // this CTA's expect_tx arrive (the bytes may come from both CTAs)
      mbar_init(&empty_bar[i], kCtaGroup); // the MMA warpgroup of every CTA the stage is multicast to
    }
    mbar_init(acc_full, 128);              // every thread of the MMA warpgroup stores its part
    mbar_init(acc_empty, kEpiWarps);       // the epilogue warps read the buffer
    mbar_init(q_ready, kEpiWarps);
    *epi_done = 0;
    fence_mbar_init();
  } else if (warp < kThrWarps) {
    for (int i = lane; i < kTcQRows; i += 32) tau_s[i] = -INFINITY;
  }
  // both CTAs' barriers initialised before any multicast or remote arrive
  if constexpr (kCtaGroup == 2) cluster_sync_all(); else __syncthreads();
  grid_dep_launch();   // the exact re-rank kernel behind this one may start its prologue as CTAs here retire

  if (warp == kProducerWarp) {
    // ============================== TMA producer ==============================
    if (lane == 0) {
      // read once -> evict first; shared with sibling CTAs (two single CTAs or several query super-blocks) -> keep in L2
      const uint64_t hint = ((kCtaGroup == 2 && p.n_qblocks == 2) || p.n_qblocks == 1) ? kEvictFirst : kEvictNormal;
      int stage = 0; uint32_t phase = 0;
      long long tp_wait = 0;
      const long long tp_begin = TCLK();
#ifdef AUR_TC_PROFILE
      unsigned long long gt0; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt0));
#endif
      for (int it = 0; it < my_tiles; ++it) {
        const int tile = tset + it * n_tsets;
        const int row0 = tile * kTileN + static_cast<int>(rank) * (kTileN / kCtaGroup);
        for (int kb = 0; kb < kbs_c; ++kb) {
          {
            const long long t0 = TCLK();
            mbar_wait(&empty_bar[stage], phase ^ 1u);
            tp_wait += TCLK() - t0;
          }
          uint8_t* dst = smem + static_cast<uint32_t>(stage) * kStageBytes;
          mbar_arrive_expect_tx(&full_bar[stage], kStageBytes);   // the whole tile lands here, half of it from the peer
          constexpr int kKb = kI8 ? kTcKBlockI8 : kTcKBlock;   // elements of a 128-byte k-block
          if constexpr (kCtaGroup == 1)
            tma_load_2d(dst, &tmap, &full_bar[stage], kb * kKb, row0, hint);
          else
            tma_load_2d_mc(dst + rank * (kStageBytes / 2), &tmap, &full_bar[stage], kb * kKb, row0, 0x3, hint);
          if (++stage == p.num_stages) { stage = 0; phase ^= 1u; }
        }
      }
#ifdef AUR_TC_PROFILE
      if ((p.dbg_flags & 64) && p.dbg_scores != nullptr) {
        unsigned long long gt1; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt1));
        float* d = p.dbg_scores + static_cast<size_t>(blockIdx.x) * kTcQRows * kTcTileN + 36;
        d[0] = static_cast<float>(tp_wait); d[1] = static_cast<float>(TCLK() - tp_begin);
        d[2] = static_cast<float>(gt1 - gt0);     // ns: cycles / ns = the SM clock the kernel really ran at
      }
#endif
    }
  } else if (warp >= kMmaWarp0) {
    // ============================== MMA warpgroup ==============================
    // wgmma accumulator layout (m64nN): thread t = 32 w + l holds rows 16 w + l / 4 (+ 8) and columns
    // 8 j + 2 (l % 4) (+ 1), j = 0..N/8-1 -- stored into the score buffer as [query][corpus row].
    const int wt = threadIdx.x - kMmaWarp0 * 32;
    const int w4 = wt >> 5, l4 = wt & 31;
    // Register A operand: per k-block and K step the m64k16 fragment of this thread -- rows 16 w + l / 4 (+ 8), the
    // bf16 pairs at columns 16 s + 2 (l % 4) (+ 8) -- read straight from global memory while the epilogue warps stage
    // the other k-blocks.  Rows past nq are zeros, as in the staged tiles.  Written here and never again, and indexed by
    // compile-time constants only (a dynamic index would put the array in local memory).
    uint32_t qa[kQReg > 0 ? kQReg : 1][4][4];
    if constexpr (kQReg > 0) {
      const int qrow = qblock * kTcQRows + 16 * w4 + (l4 >> 2);
      const uint32_t* q0 = reinterpret_cast<const uint32_t*>(p.q + static_cast<size_t>(qrow) * p.dim) + (l4 & 3);
      const uint32_t* q8 = q0 + 4 * p.dim;   // row + 8, in 32-bit words
      const bool ok0 = qrow < p.nq, ok8 = qrow + 8 < p.nq;
#pragma unroll
      for (int kb = 0; kb < kQReg; ++kb)
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int wofs = kb * 32 + k * 8;
          qa[kb][k][0] = ok0 ? __ldg(q0 + wofs) : 0u;
          qa[kb][k][1] = ok8 ? __ldg(q8 + wofs) : 0u;
          qa[kb][k][2] = ok0 ? __ldg(q0 + wofs + 4) : 0u;
          qa[kb][k][3] = ok8 ? __ldg(q8 + wofs + 4) : 0u;
        }
    }
    mbar_wait(q_ready, 0);   // the staged query k-blocks are in shared memory (and visible to the async proxy)
    const uint32_t qs_a = smem_u32(smem + L.off_qs);
    const uint32_t ring_a = smem_u32(smem);
    // One commit group per k-block, then wait_group 1: the next k-block's MMAs are queued while the previous ones run,
    // so the tensor pipe drains once per tile instead of once per k-block.  The MMAs still accumulate in the order
    // k-block 0 .. kbs - 1, K step 0 .. 3: the scores are bit-identical to waiting after every group.
    // Stages are released in ring order (rel_stage trails stage), each exactly once and only after the wait_group that
    // retires the group reading it: k-block kb's stage after k-block kb + 1 is issued, the tile's last one after the
    // wait_group 0 that ends the tile.  So at most two stages are held (a 2-stage ring never waits on itself) and none
    // across the acc_empty wait, where the epilogue may hold buffer 0 until the first certified threshold.  Without MMAs
    // (dbg_flags & 2) the waits retire nothing and the same stages are released in the same order.  The wait_groups
    // are unconditional: ptxas serialises every wgmma of the kernel when a group may be in flight where paths merge.
    // (Overlapping the score-buffer store with the next tile's first k-block, through a second accumulator, makes
    // ptxas serialise every wgmma too: it does not track which accumulator a wait_group 1 retires across loops.)
    // A tile is kQReg unrolled k-blocks with register A, then the runtime loop with shared-memory A; both run the one
    // body below, so the stage, phase and release bookkeeping is the same for either operand source.
    int stage = 0, rel_stage = 0; uint32_t phase = 0;
    long long tm_empty = 0, tm_full = 0;
    const long long tm_begin = TCLK();
    // this CTA's tensor core is done with the oldest held stage; so may be the peer's producer
    auto release = [&]() {
      if (wt == 0) {
        mbar_arrive(&empty_bar[rel_stage]);
        if constexpr (kCtaGroup == 2) mbar_arrive_cluster(&empty_bar[rel_stage], rank ^ 1u);
      }
      if (++rel_stage == p.num_stages) rel_stage = 0;
    };
    // one k-block: mmas(db) issues its four K = 16 MMAs against the ring stage behind descriptor db
    auto kblock = [&](int kb, auto&& mmas) {
      {
        const long long t0 = TCLK();
        mbar_wait(&full_bar[stage], phase);
        tm_full += TCLK() - t0;
      }
      if (!(p.dbg_flags & 2)) {
        wgmma_fence();
        mmas(wgmma_desc_sw128(ring_a + static_cast<uint32_t>(stage) * kStageBytes));
        wgmma_commit();
      }
      wgmma_wait<1>();   // k-block kb - 1 has retired
      if (kb > 0) release();
      if (++stage == p.num_stages) { stage = 0; phase ^= 1u; }
    };
    for (int it = 0; it < my_tiles; ++it) {
      float d[kTileN / 2];
      if constexpr (kI8) {
        int32_t dh[kTileN / 2], dl[kTileN / 2];
#pragma unroll
        for (int i = 0; i < kTileN / 2; ++i) { dh[i] = 0; dl[i] = 0; }
        for (int kb = 0; kb < kbs_c; ++kb)
          kblock(kb, [&](uint64_t db) {
            const uint64_t dah = wgmma_desc_sw128(qs_a + static_cast<uint32_t>(2 * kb) * kQTileBytes);
            const uint64_t dal = wgmma_desc_sw128(qs_a + static_cast<uint32_t>(2 * kb + 1) * kQTileBytes);
#pragma unroll
            for (int k = 0; k < 4; ++k) {   // 4 x K=32 per 128-byte k-block, hi then lo
              if constexpr (kTileN == kTcTileWide) wgmma_m64n128_s8(dh, dah + 2 * k, db + 2 * k, 1u);
              else wgmma_m64n64_s8(dh, dah + 2 * k, db + 2 * k, 1u);
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              if constexpr (kTileN == kTcTileWide) wgmma_m64n128_s8(dl, dal + 2 * k, db + 2 * k, 1u);
              else wgmma_m64n64_s8(dl, dal + 2 * k, db + 2 * k, 1u);
            }
          });
        wgmma_wait<0>();
        wgmma_fence_regs(dh);
        wgmma_fence_regs(dl);
#pragma unroll
        for (int i = 0; i < kTileN / 2; ++i) d[i] = fmaf(static_cast<float>(dh[i]), 256.f, static_cast<float>(dl[i]));
      } else {
#pragma unroll
      for (int i = 0; i < kTileN / 2; ++i) d[i] = 0.f;
      if constexpr (kQReg > 0) {
#pragma unroll
        for (int kb = 0; kb < kQReg; ++kb)
          kblock(kb, [&](uint64_t db) {
#pragma unroll
            for (int k = 0; k < 4; ++k) wgmma_m64n128_rs(d, qa[kb][k], db + 2 * k, 1u);
          });
      }
      for (int kb = kQReg; kb < kbs; ++kb)
        kblock(kb, [&](uint64_t db) {
          const uint64_t da = wgmma_desc_sw128(qs_a + static_cast<uint32_t>(kb - kQReg) * kQTileBytes);
#pragma unroll
          for (int k = 0; k < 4; ++k) {   // 4 x K=16 per 128-byte k-block
            if constexpr (kTileN == kTcTileWide) wgmma_m64n128_ss(d, da + 2 * k, db + 2 * k, 1u);
            else wgmma_m64n64_ss(d, da + 2 * k, db + 2 * k, 1u);
          }
        });
      wgmma_wait<0>();
      wgmma_fence_regs(d);
      }
      release();
      {
        const long long t0 = TCLK();
        mbar_wait(acc_empty, (static_cast<uint32_t>(it) & 1u) ^ 1u);
        tm_empty += TCLK() - t0;
      }
#pragma unroll
      for (int j = 0; j < kTileN / 8; ++j) {
        const int row = 16 * w4 + (l4 >> 2), col = 8 * j + 2 * (l4 & 3);
        *reinterpret_cast<float2*>(scbuf + row * kScStride + col) = make_float2(d[4 * j + 0], d[4 * j + 1]);
        *reinterpret_cast<float2*>(scbuf + (row + 8) * kScStride + col) = make_float2(d[4 * j + 2], d[4 * j + 3]);
      }
      mbar_arrive(acc_full);
    }
    if ((p.dbg_flags & 64) && p.dbg_scores != nullptr && wt == 0) {
      float* dd = p.dbg_scores + static_cast<size_t>(blockIdx.x) * kTcQRows * kTcTileN + 32;
      dd[0] = static_cast<float>(tm_empty); dd[1] = static_cast<float>(tm_full);
      dd[2] = static_cast<float>(TCLK() - tm_begin);
    }
  } else if (warp < kProducerWarp) {
    // ================= threshold warp (0) and epilogue warps (1-2) =================
    const int ew = warp - kThrWarps;           // epilogue warp 0 .. 1 (the threshold warp: -1)
    const int quarter = ew & 1;                // which 32 queries of the block this warp owns
    const int r = (warp < kThrWarps) ? lane : quarter * 32 + lane;   // query row inside the CTA
    const int qglob = qblock * kTcQRows + r;   // query index inside this launch
    // exchange table: [qblock][query][CTA] -> a query's row is contiguous;
    // behind it, one published threshold per query
    const int pub_stride = (n_tsets + 1) & ~1;
    unsigned long long* pub_base =
        reinterpret_cast<unsigned long long*>(p.pub) + static_cast<size_t>(qblock) * kTcQRows * pub_stride;
    unsigned long long* thr_base = reinterpret_cast<unsigned long long*>(p.pub) +
                                   static_cast<size_t>(p.n_qblocks) * kTcQRows * pub_stride + qblock * kTcQRows;
    unsigned long long* pubrow = pub_base + static_cast<size_t>(r) * pub_stride;
    const unsigned long long* thr_q = thr_base + r;

    if (warp < kThrWarps) {
      // ============================== threshold warp ==============================
      // Serve the queries r = tset, tset + n_tsets, ... of this CTA's query block.
      constexpr int kSlots = 8;                      // queries one CTA may have to serve: ceil(128 / tile sets), tile sets >= 16
      float cur[kSlots];
#pragma unroll
      for (int sl = 0; sl < kSlots; ++sl) cur[sl] = -INFINITY;
      int polls = 0;
      while (xchg && my_tiles > 0) {
        // every epilogue thread of the grid waits for the FIRST threshold (bootstrap): poll fast until it is out
        __nanosleep(polls < 48 ? 150 : 1500);
        ++polls;
        const bool done = *epi_done >= kEpiWarps;
        // every global load of this round is issued before the first one is consumed: one L2 round trip per round
        unsigned long long cached[kTcQRows / 32];
#pragma unroll
        for (int j = 0; j < kTcQRows / 32; ++j) cached[j] = __ldcg(thr_base + j * 32 + lane);
        PubEntries ent[kSlots];
        int nslot = 0;
#pragma unroll
        for (int sl = 0; sl < kSlots; ++sl) {
          const int rq = tset + sl * n_tsets;
          if (rq < kTcQRows) { ent[sl] = exchange_load(pub_base + static_cast<size_t>(rq) * pub_stride, nuse, lane); nslot = sl + 1; }
        }
#pragma unroll
        for (int sl = 0; sl < kSlots; ++sl) {
          if (sl < nslot) {
            const int rq = tset + sl * n_tsets;
            const float t = exchange_select(ent[sl], nuse, xR, epoch, lane);
            if (t > cur[sl]) {
              cur[sl] = t;
              if (lane == 0) __stcg(thr_base + rq, (static_cast<unsigned long long>(epoch) << 32) | __float_as_uint(t));
            }
          }
        }
        // Refresh this CTA's cache of its 128 queries' certified thresholds.  The epilogue reads them from shared
        // memory once per tile; a global (L2) read there sat on the per-tile critical path with its full latency.
#pragma unroll
        for (int j = 0; j < kTcQRows / 32; ++j)
          if (static_cast<uint32_t>(cached[j] >> 32) == epoch) tau_s[j * 32 + lane] = __uint_as_float(static_cast<uint32_t>(cached[j]));   // only ever rises
        if (done) break;
      }
    } else {
      // ============================== epilogue warps ==============================
      const long long t_kernel0 = TCLK();
      // ---- the query block into shared memory: [64 queries x 128 B] K-major tiles with the 128-byte swizzle TMA
      //      would produce (16-byte chunk c of row r at c ^ (r & 7)).
      //      A warp reads its 32 rows coalesced (lane l takes 16-byte piece l of 4 consecutive rows per instruction).
      {
        const uint8_t* qbase = reinterpret_cast<const uint8_t*>(p.q);
        const size_t row_bytes = static_cast<size_t>(p.dim) * 2;
        const int wrow0 = qblock * kTcQRows + quarter * 32;   // first query of this warp
        auto load_kb = [&](int kb, uint4 (&x)[8]) {
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int id = i * 32 + lane, row = id >> 3, c = id & 7;
            x[i] = make_uint4(0, 0, 0, 0);
            if (kb < kbs && wrow0 + row < p.nq) x[i] = ldg_nc_v4(qbase + static_cast<size_t>(wrow0 + row) * row_bytes + kb * 128 + c * 16);
          }
        };
        // every CTA of a query block reads the same block at the same moment: start each at a different
        // k-block (rotation by tile set) so they do not all queue on the same L2 lines
        // (only the k-blocks the MMA warpgroup does not hold in registers: kQReg .. kbs - 1, tile index kb - kQReg)
        const int nst = kbs - kQReg;
        const int rot = nst > 0 ? tset % nst : 0;
        auto kb_of = [&](int j) { return (j < nst) ? kQReg + (j + rot) % nst : kbs; };
        // four k-blocks of loads (32 x 16 B per lane) are issued before the first is consumed
        constexpr int kDepth = 4;
        uint4 x[kDepth][8];
        for (int j0 = 0; j0 < nst; j0 += kDepth) {
#pragma unroll
          for (int u = 0; u < kDepth; ++u) load_kb(kb_of(j0 + u), x[u]);
#pragma unroll
          for (int u = 0; u < kDepth; ++u) {
            const int j = j0 + u;
            if (j >= nst) break;
            uint8_t* tile = smem + L.off_qs + static_cast<uint32_t>(kb_of(j) - kQReg) * kQTileBytes + quarter * 32 * 128;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int id = i * 32 + lane, row = id >> 3, c = id & 7;
              *reinterpret_cast<uint4*>(tile + row * 128 + ((c ^ (row & 7)) << 4)) = x[u][i];
            }
          }
        }
        fence_proxy_async_smem();   // the generic-proxy stores -> visible to the tensor core
        __syncwarp();
        if (lane == 0) mbar_arrive(q_ready);
      }
      const float* myrow = scbuf + r * kScStride;   // this query's row of the score buffer
      auto load_scores = [&](uint32_t (&acc)[4][16], int h) {   // scores 64 h .. 64 h + 63 of the tile
#pragma unroll
        for (int c = 0; c < 4; ++c)
#pragma unroll
          for (int j4 = 0; j4 < 4; ++j4) {
            const float4 v = *reinterpret_cast<const float4*>(myrow + h * 64 + c * 16 + j4 * 4);
            acc[c][j4 * 4 + 0] = __float_as_uint(v.x); acc[c][j4 * 4 + 1] = __float_as_uint(v.y);
            acc[c][j4 * 4 + 2] = __float_as_uint(v.z); acc[c][j4 * 4 + 3] = __float_as_uint(v.w);
          }
      };
      float* mynorm = normbuf + ew * 2 * kTileN;
      uint32_t* mymask = maskbuf + ew * 2 * kTileN;
      uint32_t mybit = 0u;                                       // this query's tenant-scope bit
      if constexpr (kMask) { if (qglob < p.nq) mybit = 1u << (p.q_scope[qglob] & 31); }
      const uint32_t list_a = smem_u32(smem + L.off_list) + static_cast<uint32_t>(r) * 8u;
      // deferred-candidate FIFO (see drain_fifo) whenever shared memory has room for it
      const bool use_fifo = L.fifo_recs > 0;
      const uint32_t fifo_a = smem_u32(smem + L.off_fifo) + r * 16u;
      const uint32_t ftag_a = smem_u32(smem + L.off_fifo) + L.fifo_recs * kTcQRows * 16u + r * 4u;
      int fcnt = 0;
      TopkState st;
      st.min_key = kKeyEmpty; st.tau_local = -INFINITY; st.tau = -INFINITY;
      st.top[0] = st.top[1] = st.top[2] = st.top[3] = -INFINITY; st.minpos = 0; st.nfill = 0;
      if (qglob >= p.nq) st.tau = INFINITY;   // padding row of a partial query block: admits nothing, appends nothing
      float published = -INFINITY;
      bool booted = false;   // the bootstrap has already fed the first tile's chunk maxima into st.top
      int nslow = 0;
      long long t_wait = 0, t_slow = 0, t_ld = 0, t_top = 0, t_fast = 0, t_chunks = 0, t_pub = 0;
      const long long t_begin = TCLK();
      long long t_boot = 0, t_loop_end = 0;

      // inverse norms: tile(0) into buffer 0, tile(1) in flight in registers (lane takes rows lane + 32 i)
      constexpr int kNv = kTileN / 32;
      float nn[kNv];
      uint32_t mm[kNv];                                         // (masks of the tile in flight, beside its norms)
      auto load_norms = [&](int it2) {
#pragma unroll
        for (int i = 0; i < kNv; ++i) { nn[i] = __uint_as_float(kNaNBits); mm[i] = 0u; }
        if (it2 < my_tiles) {
          const int64_t rbase = static_cast<int64_t>(tset + it2 * n_tsets) * kTileN;
#pragma unroll
          for (int i = 0; i < kNv; ++i)
            if (rbase + lane + 32 * i < p.n_rows) nn[i] = __ldg(p.inv_norm + rbase + lane + 32 * i);
          if constexpr (kMask) {
#pragma unroll
            for (int i = 0; i < kNv; ++i)
              if (rbase + lane + 32 * i < p.n_rows) mm[i] = __ldg(p.row_mask + rbase + lane + 32 * i);
          }
        }
      };
      auto store_norms = [&](int buf) {
#pragma unroll
        for (int i = 0; i < kNv; ++i) {
          mynorm[buf * kTileN + lane + 32 * i] = nn[i];
          if constexpr (kMask) mymask[buf * kTileN + lane + 32 * i] = mm[i];
        }
      };
      load_norms(0);
      store_norms(0);
      load_norms(1);
      __syncwarp();

      // Bootstrap on the first tile: nobody has a threshold yet, and pushing 64 arbitrary rows
      // through the list would be all waste.  Read the tile once just for its best score(s),
      // publish them, wait until enough CTAs have done the same (~5 us, once), and let the
      // main loop examine the tile against the first certified threshold.  The accumulator
      // buffer is not released here, so the MMA cannot overwrite it before the loop reads it again.
      if (xchg && my_tiles > 0) {
        mbar_wait(acc_full, 0);
#pragma unroll 1
        for (int c = 0; c < kTileN / 16; ++c) {
          uint32_t a16[16];
#pragma unroll
          for (int j4 = 0; j4 < 4; ++j4) {
            const float4 v = *reinterpret_cast<const float4*>(myrow + c * 16 + j4 * 4);
            a16[j4 * 4 + 0] = __float_as_uint(v.x); a16[j4 * 4 + 1] = __float_as_uint(v.y);
            a16[j4 * 4 + 2] = __float_as_uint(v.z); a16[j4 * 4 + 3] = __float_as_uint(v.w);
          }
          float m = -INFINITY;
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            float v = __uint_as_float(a16[j]) * mynorm[c * 16 + j];
            if constexpr (kMask) { if (!(mymask[c * 16 + j] & mybit)) v = __uint_as_float(kNaNBits); }
            m = fmaxf(m, v);
          }
          top4_insert(st.top, m);       // (the main loop skips the tracker for this tile: it is counted here)
        }
        const float pv0 = top4_get(st.top, xm);
        if (pv0 > -INFINITY) {
          publish_value(pubrow + tset, epoch, pv0, true);
          published = pv0;
        }
        booted = true;
        const long long tb = clock64();
        float tboot = -INFINITY;
        do {
          __nanosleep(100);
          tboot = tau_s[r];
        } while (__any_sync(0xffffffffu, tboot == -INFINITY) && clock64() - tb < 100000);
        st.tau = fmaxf(st.tau, tboot);
        t_boot = TCLK() - t_begin;
      }

      for (int it = 0; it < my_tiles; ++it) {
        const int tile = tset + it * n_tsets;
        const int row0 = tile * kTileN;
        const float* nbt = mynorm + (it & 1) * kTileN;
        const long long t_top0 = TCLK();
        const float thr_now = (xchg && !(p.dbg_flags & 16)) ? tau_s[r] : -INFINITY;   // shared-memory copy kept by the threshold warp

        // norms of the next tile (loaded one iteration ago) -> the other buffer; start the
        // loads for the tile after that.  A whole tile period hides the HBM latency.
        if (!(p.dbg_flags & 32)) {
          store_norms((it + 1) & 1);
          load_norms(it + 2);
          __syncwarp();
        }

        {
          const long long t0 = TCLK();
          mbar_wait(acc_full, (static_cast<uint32_t>(it)) & 1u);
          t_wait += TCLK() - t0;
        }
        // A wide tile is examined 64 scores at a time by the same code, half 0 while the buffer is still held.
#pragma unroll 1
        for (int h = 0; h < kHalves; ++h) {
          const int hrow0 = row0 + 64 * h;
          const float* nb = nbt + 64 * h;
          const long long t_ld0 = TCLK();
          uint32_t acc[4][16];
          if (!(p.dbg_flags & 1)) load_scores(acc, h);
          if (h == kHalves - 1) {   // the whole tile in registers or examined: hand the buffer back to the MMA warpgroup
            __syncwarp();
            if (lane == 0) mbar_arrive(acc_empty);
          }
          t_ld += TCLK() - t_ld0;
          if (p.dbg_flags & (1 | 4)) continue;
          const long long t_fast0 = TCLK();

          // Fast path: scale by 1/|c_j| in place and keep one running max per 16
          // scores.  (NaN norm = tombstone / out of range: fmaxf drops it, `>=` rejects it.)
          if constexpr (kMask) {   // rows this query's tenant scope may not see: NaN, like tombstones
            const uint32_t* mb = mymask + (it & 1) * kTileN + h * 64;
#pragma unroll
            for (int c = 0; c < 4; ++c)
#pragma unroll
              for (int j4 = 0; j4 < 4; ++j4) {
                const uint4 mk = *reinterpret_cast<const uint4*>(mb + c * 16 + j4 * 4);
                if (!(mk.x & mybit)) acc[c][j4 * 4 + 0] = kNaNBits;
                if (!(mk.y & mybit)) acc[c][j4 * 4 + 1] = kNaNBits;
                if (!(mk.z & mybit)) acc[c][j4 * 4 + 2] = kNaNBits;
                if (!(mk.w & mybit)) acc[c][j4 * 4 + 3] = kNaNBits;
              }
          }
          float cmax[4];
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            float m = -INFINITY;
#pragma unroll
            for (int j4 = 0; j4 < 4; ++j4) {
              const float4 nv = *reinterpret_cast<const float4*>(nb + c * 16 + j4 * 4);
              acc[c][j4 * 4 + 0] = __float_as_uint(__fmul_rn(__uint_as_float(acc[c][j4 * 4 + 0]), nv.x));
              acc[c][j4 * 4 + 1] = __float_as_uint(__fmul_rn(__uint_as_float(acc[c][j4 * 4 + 1]), nv.y));
              acc[c][j4 * 4 + 2] = __float_as_uint(__fmul_rn(__uint_as_float(acc[c][j4 * 4 + 2]), nv.z));
              acc[c][j4 * 4 + 3] = __float_as_uint(__fmul_rn(__uint_as_float(acc[c][j4 * 4 + 3]), nv.w));
              m = fmaxf(fmaxf(m, fmaxf(__uint_as_float(acc[c][j4 * 4 + 0]), __uint_as_float(acc[c][j4 * 4 + 1]))),
                        fmaxf(__uint_as_float(acc[c][j4 * 4 + 2]), __uint_as_float(acc[c][j4 * 4 + 3])));
            }
            cmax[c] = m;
          }
          if constexpr (kDump) {   // the score dump: the whole first tile, [CTA][query][kTileN]
            if (it == 0) {
#pragma unroll
              for (int c = 0; c < 4; ++c)
#pragma unroll
                for (int j = 0; j < 16; ++j)
                  p.dbg_scores[(static_cast<size_t>(blockIdx.x) * kTcQRows + r) * kTileN + h * 64 + c * 16 + j] =
                      __uint_as_float(acc[c][j]);
            }
          }

          t_fast += TCLK() - t_fast0;
          // what this CTA can vouch for (published below): chunk maxima are distinct rows
          if (!(booted && it == 0)) {
            if (xm == 1) st.top[0] = fmaxf(st.top[0], fmaxf(fmaxf(cmax[0], cmax[1]), fmaxf(cmax[2], cmax[3])));
            else { top4_insert(st.top, cmax[0]); top4_insert(st.top, cmax[1]); top4_insert(st.top, cmax[2]); top4_insert(st.top, cmax[3]); }
          }
          if (p.dbg_flags & 8) continue;
          const long long t_ch0 = TCLK();
          // A group of four scores whose max reaches this query's threshold goes out of line.
          st.tau = fmaxf(st.tau, thr_now);
          if (use_fifo) {
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              if (cmax[c] >= st.tau) {
                if (fcnt > static_cast<int>(L.fifo_recs) - 4) {   // no room for four more groups: make room (rare)
                  const long long t0 = TCLK();
                  st = drain_fifo(st, fifo_a, ftag_a, fcnt, list_a, ksel, p.ids);
                  fcnt = 0;
                  ++nslow;
                  t_slow += TCLK() - t0;
                }
#pragma unroll
                for (int g = 0; g < 4; ++g) {   // park the groups that reach the threshold: two stores each, no call
                  const float m4 = fmaxf(fmaxf(__uint_as_float(acc[c][4 * g]), __uint_as_float(acc[c][4 * g + 1])),
                                         fmaxf(__uint_as_float(acc[c][4 * g + 2]), __uint_as_float(acc[c][4 * g + 3])));
                  if (m4 >= st.tau) {
                    asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(fifo_a + static_cast<uint32_t>(fcnt) * (kTcQRows * 16u)),
                                 "r"(acc[c][4 * g]), "r"(acc[c][4 * g + 1]), "r"(acc[c][4 * g + 2]), "r"(acc[c][4 * g + 3]) : "memory");
                    asm volatile("st.shared.b32 [%0], %1;" ::"r"(ftag_a + static_cast<uint32_t>(fcnt) * (kTcQRows * 4u)),
                                 "r"(hrow0 + c * 16 + 4 * g) : "memory");
                    ++fcnt;
                  }
                }
              }
            }
          } else {
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            if (cmax[c] >= st.tau) {
              const long long t0 = TCLK();
#pragma unroll
              for (int g = 0; g < 4; ++g) {
                const float s0 = __uint_as_float(acc[c][4 * g]), s1 = __uint_as_float(acc[c][4 * g + 1]);
                const float s2 = __uint_as_float(acc[c][4 * g + 2]), s3 = __uint_as_float(acc[c][4 * g + 3]);
                if (fmaxf(fmaxf(s0, s1), fmaxf(s2, s3)) >= st.tau)
                  st = push_group4(st, s0, s1, s2, s3, hrow0 + c * 16 + 4 * g, list_a, ksel, p.ids);
              }
              ++nslow;
              t_slow += TCLK() - t0;
            }
          }
          }

          if (it < 8) t_top += TCLK() - t_ch0; else t_chunks += TCLK() - t_ch0;   // t_top reused: early tiles
        }
        if (p.dbg_flags & (1 | 4 | 8)) continue;
        const long long t_pub0 = TCLK();
        // publish this CTA's m-th best for the exchange (monotone, so stale reads stay valid)
        const float pv = top4_get(st.top, xm);
        if (xchg && pv > published) {
          publish_value(pubrow + tset, epoch, pv, published == -INFINITY);
          published = pv;
        }
        t_pub += TCLK() - t_pub0;
      }
      t_loop_end = TCLK();
      __syncwarp();
      if (lane == 0) atomicAdd(const_cast<int*>(epi_done), 1);   // lets the threshold warps go
      // one read of the certified threshold (a global round trip) serves both the parked candidates and the final cut
      float tau_end = -INFINITY;
      if (xchg && my_tiles > 0) tau_end = read_threshold(thr_q, epoch);
      st.tau = fmaxf(st.tau, tau_end);
      if (use_fifo) {   // whatever is still parked meets the final threshold
        if (__any_sync(0xffffffffu, fcnt > 0)) st = drain_fifo(st, fifo_a, ftag_a, fcnt, list_a, ksel, p.ids);
        fcnt = 0;
      }

      // ---- append the survivors (score >= the certified threshold, at most ksel of them)
      //      to this query's compact candidate row
      st = compact_list(st, list_a, ksel, p.ids);
      {
        const size_t cap = static_cast<size_t>(n_tsets) * ksel;
        uint64_t* out = p.cand + static_cast<size_t>(qglob) * cap;
        if (st.nfill > 0 && qglob < p.nq) {
          const uint32_t slot0 = atomicAdd(p.cand_count + qglob, static_cast<uint32_t>(st.nfill));
          for (int t = 0; t < st.nfill; ++t) out[slot0 + t] = lds_u64(list_a + t * kSlot);
        }
      }
      if ((p.dbg_flags & 64) && p.dbg_scores != nullptr) {
        float* d = p.dbg_scores + (static_cast<size_t>(blockIdx.x) * kTcQRows + r) * kTcTileN;
        d[0] = static_cast<float>(st.nfill); d[1] = static_cast<float>(nslow);
        d[2] = tau_end; d[3] = st.tau_local;
        d[8] = static_cast<float>(t_wait); d[9] = static_cast<float>(t_slow);
        d[10] = 0.f; d[11] = static_cast<float>(t_ld);
        d[12] = static_cast<float>(TCLK() - t_begin);
        d[13] = static_cast<float>(t_top); d[14] = static_cast<float>(t_fast);
        d[15] = static_cast<float>(t_chunks); d[16] = static_cast<float>(t_pub);
        d[17] = static_cast<float>(t_boot); d[18] = static_cast<float>(t_begin - t_kernel0);
        d[19] = static_cast<float>(TCLK() - t_loop_end);
      }
    }
  }

  // ============================== teardown ==============================
  __syncwarp();
  // no CTA of a pair exits while its peer may still multicast into it or arrive on its barriers
  if constexpr (kCtaGroup == 2) cluster_sync_all();
}

template <int kCtaGroup, bool kMask, int kTileN, int kQReg, bool kI8, bool kDump = false>
cudaError_t launch_variant(const cudaLaunchConfig_t& cfg, const CUtensorMap& tm, const TcParams& p, size_t smem) {
  auto kern = simtopk_tc_kernel<kCtaGroup, kMask, kTileN, kQReg, kI8, kDump>;
  // raised only: concurrent searches of the shards on one device ask for different sizes (raise_smem_limit)
  cudaError_t e = raise_smem_limit(reinterpret_cast<const void*>(kern), smem);
  if (e != cudaSuccess) return e;
  return cudaLaunchKernelEx(&cfg, kern, tm, p);
}

// The masked, the dumping (a score buffer without the per-thread counters of dbg_flags 64) or the plain kernel.
template <int kCtaGroup, int kTileN, int kQReg, bool kI8>
cudaError_t launch_kind(const cudaLaunchConfig_t& cfg, const CUtensorMap& tm, const TcParams& p, size_t smem) {
  if (p.row_mask != nullptr) return launch_variant<kCtaGroup, true, kTileN, kQReg, kI8>(cfg, tm, p, smem);
  if (p.dbg_scores != nullptr && !(p.dbg_flags & 64)) return launch_variant<kCtaGroup, false, kTileN, kQReg, kI8, true>(cfg, tm, p, smem);
  return launch_variant<kCtaGroup, false, kTileN, kQReg, kI8>(cfg, tm, p, smem);
}

}  // namespace

size_t tc_smem_bytes(int num_stages, int ksel, int dim, int tile_n, bool mask, int qregs) {
  return make_layout(num_stages, ksel, dim, tile_n, mask, qregs).total + 1024;  // + alignment slack
}

int tc_pick_stages(int ksel, int dim, size_t smem_limit, int tile_n, bool mask, int qregs) {
  for (int s = kTcMaxStages; s >= 2; --s)
    if (tc_smem_bytes(s, ksel, dim, tile_n, mask, qregs) <= smem_limit) return s;
  return 0;
}

cudaError_t tc_launch(int cta_group, int tile_n, int qregs, bool i8, int grid, const void* tmap, const TcParams& p, size_t smem,
                      cudaStream_t s) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cta_group;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  const CUtensorMap& tm = *reinterpret_cast<const CUtensorMap*>(tmap);
  if (i8) {
    if (qregs != 0 || p.dim % kTcKBlockI8 != 0) return cudaErrorInvalidValue;
    if (tile_n == kTcTileWide)
      return cta_group == 2 ? launch_kind<2, kTcTileWide, 0, true>(cfg, tm, p, smem) : launch_kind<1, kTcTileWide, 0, true>(cfg, tm, p, smem);
    return cta_group == 2 ? launch_kind<2, kTcTileN, 0, true>(cfg, tm, p, smem) : launch_kind<1, kTcTileN, 0, true>(cfg, tm, p, smem);
  }
  if (qregs != 0) {   // smem was sized without these k-blocks' tiles: only the matching kernel may run
    if (qregs != kTcQRegs || tile_n != kTcTileWide || p.dim / kTcKBlock < qregs) return cudaErrorInvalidValue;
    return cta_group == 2 ? launch_kind<2, kTcTileWide, kTcQRegs, false>(cfg, tm, p, smem) : launch_kind<1, kTcTileWide, kTcQRegs, false>(cfg, tm, p, smem);
  }
  if (tile_n == kTcTileWide)
    return cta_group == 2 ? launch_kind<2, kTcTileWide, 0, false>(cfg, tm, p, smem) : launch_kind<1, kTcTileWide, 0, false>(cfg, tm, p, smem);
  return cta_group == 2 ? launch_kind<2, kTcTileN, 0, false>(cfg, tm, p, smem) : launch_kind<1, kTcTileN, 0, false>(cfg, tm, p, smem);
}

}  // namespace aur
