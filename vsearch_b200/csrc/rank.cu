// rank.cu — k-mer index in HBM and the candidate ranker (sm_90a).
//
// Replaces, for whole batches of queries at once,
//   unique_count            (reference core/unique.cpp:155-353)   distinct unmasked k-mers of a sequence
//   Dbindex::prepare/add_*  (core/dbindex.cpp:121-255)            k-mer -> targets postings
//   search_topscores        (core/searchcore.cpp:260-340)         per-target shared-k-mer counts,
//                                                                 threshold, best `tophits` targets
//   minheap_*               (core/minheap.cpp:82-263)             order: count desc, length asc, seqno asc
//
// Layout.  The database is cut into SHARDS of at most 32766 consecutive targets (static index; 32768 for the cluster
// driver's incremental one).  A shard stores CSR postings; in the static index every k-mer has two sub-lists, its even
// and its odd targets, and a posting is the BYTE OFFSET of the target's counter word as a u16 (half the bytes of the
// reference's u32 lists; the reference's per-k-mer bitmaps for very frequent k-mers, dbindex.cpp:212-229, are a storage
// variant with the same meaning and are not needed).  --wordlength 3..10: list heads for all 2 * 4^k sub-lists;
// 11..15: only the sub-lists that exist, found by binary search (build_sparse_shard).
// One CTA ranks one query: for every shard it zeroes 32768 16-bit counters in SHARED memory, turns the postings of
// the query's distinct k-mers into shared-memory atomic adds — the runs of all k-mers laid end to end as one stream
// of 16-byte vectors that the 16 warps split evenly (every lane busy every round) —, scans the counters against a
// running threshold and appends the survivors as 64-bit sort keys to a candidate list that is sorted and cut to
// `tophits` at the end (and whenever a crowd of ties fills it up).  HBM traffic per query is the postings themselves
// (2 B each) — the counters never leave the SM.  Above TOPHITS_MAX candidates per query (rank_lists) the keys of every
// target at the threshold go to HBM instead and are sorted there per query.
#include "vsg_internal.h"
#include "rank_steps.cuh"

#include <cub/cub.cuh>
#include <thrust/iterator/transform_iterator.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <mutex>

namespace vsg {

constexpr int TOPHITS_MAX = RANK_TOPHITS_MAX;

// ---- index build: pass 1 counts, pass 2 fills; one CTA per target, shared-memory bitmap dedupe ----
template <bool FILL>
__global__ void index_build_kernel(DevSeqs db, int t0, int nt, int k, int mask_lower, int split,
                                   uint32_t * __restrict__ count /* pass1: counts; pass2: fill cursors */,
                                   const uint32_t * __restrict__ start, uint16_t * __restrict__ post)
{
  extern __shared__ uint32_t bitmap[];
  int const lt = blockIdx.x;
  if (lt >= nt) { return; }
  int const words = (1 << (2 * k)) >> 5;
  for (int i = threadIdx.x; i < (words > 0 ? words : 1); i += blockDim.x) { bitmap[i] = 0; }
  __syncthreads();
  int64_t const t = static_cast<int64_t>(t0) + lt;
  const uint8_t * __restrict__ s = db.sym + db.off[t];
  int const len = db.len[t];
  for (int p = k - 1 + threadIdx.x; p < len; p += blockDim.x) {
    uint32_t km;
    if (kmer_at(s, p, k, mask_lower, km)) {
      uint32_t const bit = 1u << (km & 31);
      uint32_t const old = atomicOr(&bitmap[km >> 5], bit);
      if ((old & bit) == 0) {  // first occurrence in this target
        uint32_t const list = split ? 2u * km + static_cast<uint32_t>(lt & 1) : km;   // static index: even / odd targets apart
        if (FILL) {
          uint32_t const pos = atomicAdd(&count[list], 1u);
          post[static_cast<size_t>(start[list]) + pos] = static_cast<uint16_t>((lt & ~1) << 1);
        } else {
          atomicAdd(&count[list], 1u);
        }
      }
    }
  }
}

// lists are padded to a multiple of 8 entries so that every list starts on a 16-byte boundary
__global__ void pad_counts_kernel(uint32_t * __restrict__ count, int n)
{
  int const i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { count[i] = (count[i] + 7u) & ~7u; }
}
__global__ void fill_u16_kernel(uint16_t * __restrict__ p, size_t n, uint16_t v)
{
  size_t const i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) { p[i] = v; }
}

// per-k-mer totals over the shards built so far (vsg_udb_load checks them against the file's word counts)
__global__ void add_totals_kernel(const uint32_t * __restrict__ count /* 2 per k-mer */, uint32_t * __restrict__ totals, size_t hashsize)
{
  size_t const i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < hashsize) { totals[i] += count[2 * i] + count[2 * i + 1]; }
}

// the same totals from a built shard: sub-list i holds its k-mer's targets plus up to 7 POST_PAD entries (dense: k-mer
// i >> 1; sparse: rkeys[i] >> 1)
__global__ void shard_word_counts_kernel(ShardDev S, uint32_t nlists, uint32_t * __restrict__ totals)
{
  uint32_t const i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nlists) { return; }
  uint32_t n = 0;
  for (uint32_t j = S.start[i]; j < S.start[i + 1]; j++) { n += S.post[j] != POST_PAD ? 1u : 0u; }
  if (n > 0) { atomicAdd(&totals[(S.nr != 0 ? S.rkeys[i] : i) >> 1], n); }
}

// ---- sparse build (--wordlength 11..15: 4^k list heads per shard would dwarf the postings) --------------------------
// One 46-bit key per window: k-mer (30 bits) | target parity | local target >> 1 (14 bits); windows that hold a masked
// symbol, and the first k-1 positions of a target, get SPARSE_INVALID, which sorts behind every real key.  Sorting the
// keys and dropping duplicates IS the per-target de-duplication (unique_count_hash, core/unique.cpp:243-334: its
// CityHash table is only the device that finds the distinct k-mers) and the grouping by list in one go.
constexpr uint64_t SPARSE_INVALID = 1ull << 45;
__global__ void sparse_keys_kernel(DevSeqs db, int t0, int nt, int k, int mask_lower, const int64_t * __restrict__ cum,
                                   uint64_t * __restrict__ keys)
{
  int const lt = blockIdx.x;
  if (lt >= nt) { return; }
  int64_t const t = static_cast<int64_t>(t0) + lt;
  const uint8_t * __restrict__ s = db.sym + db.off[t];
  int const len = db.len[t];
  uint64_t * __restrict__ out = keys + cum[lt];
  uint64_t const low = (static_cast<uint64_t>(lt & 1) << 14) | static_cast<uint64_t>(lt >> 1);
  for (int p = threadIdx.x; p < len; p += blockDim.x) {
    uint64_t key = SPARSE_INVALID;
    uint32_t km;
    if (p >= k - 1 && kmer_at(s, p, k, mask_lower, km)) { key = (static_cast<uint64_t>(km) << 15) | low; }
    out[p] = key;
  }
}
struct SparseRunOf {   // key -> sub-list id (k-mer << 1 | parity); the invalid key maps to 0x80000000
  __host__ __device__ uint32_t operator()(uint64_t key) const { return static_cast<uint32_t>(key >> 14); }
};
struct PadTo8 {
  __host__ __device__ uint32_t operator()(uint32_t n) const { return (n + 7u) & ~7u; }
};
// sub-list r: its distinct keys ukeys[src[r] .. src[r] + cnt[r]) become counter offsets at post[dst[r] ...]
__global__ void sparse_scatter_kernel(const uint64_t * __restrict__ ukeys, const uint32_t * __restrict__ rkeys,
                                      const uint32_t * __restrict__ cnt, const uint32_t * __restrict__ src,
                                      const uint32_t * __restrict__ dst, uint32_t nr, uint16_t * __restrict__ post,
                                      uint32_t * __restrict__ totals)
{
  uint32_t const r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= nr) { return; }
  uint32_t const n = cnt[r], a = src[r], b = dst[r];
  for (uint32_t i = 0; i < n; i++) { post[b + i] = static_cast<uint16_t>((ukeys[a + i] & 0x3fffu) << 2); }
  if (totals != nullptr) { atomicAdd(&totals[rkeys[r] >> 1], n); }
}

// Order inside a list does not matter to the counts, only to the speed of the shared-memory atomics that apply it:
// the ranker's warp turns a list into counter updates 32 postings at a time — lane L holds vector blk*32 + L of the
// list and instruction j of a vector round updates posting 8*(blk*32 + L) + j of every lane.  Those 32 postings are a
// "row"; a row whose postings fall into 32 different shared-memory banks (bank = bits 2..6 of the stored counter offset) is applied in one pass, one with collisions is replayed.  This kernel sorts every list
// by bank and deals the sorted postings out down the rows' lanes, so that the members of one row lie a whole
// list / 32 apart in bank order: a row only collides where a bank holds more than 1/32 of the list.
constexpr int BANK_ORDER_CAP = 8192;   // longer lists (a k-mer in a quarter of the shard) are left as they are

__global__ void __launch_bounds__(128)
list_bank_order_kernel(const uint32_t * __restrict__ start, uint16_t * __restrict__ post, int nlists)
{
  __shared__ uint16_t src[BANK_ORDER_CAP];
  __shared__ uint32_t hist[32], cursor[32];
  for (int li = blockIdx.x; li < nlists; li += gridDim.x) {
    uint32_t const b = start[li];
    int const n = static_cast<int>(start[li + 1] - b);   // a multiple of 8
    if (n <= 32 || n > BANK_ORDER_CAP) { continue; }      // uniform per block
    uint16_t * const lp = post + b;
    if (threadIdx.x < 32) { hist[threadIdx.x] = 0; }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      uint16_t const x = lp[i];
      src[i] = x;
      atomicAdd(&hist[(x >> 2) & 31], 1u);
    }
    __syncthreads();
    if (threadIdx.x < 32) {
      uint32_t const v = hist[threadIdx.x];
      cursor[threadIdx.x] = warp_inclusive_sum(v) - v;
    }
    __syncthreads();
    int const nv = n >> 3, full = nv >> 5, rem = nv & 31;   // vectors; whole 32-vector blocks; lanes used in the last block
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      uint16_t const x = src[i];
      int const si = static_cast<int>(atomicAdd(&cursor[(x >> 2) & 31], 1u));   // rank in bank order
      // positions in the order (lane, block, posting of the vector)
      int const vr = si >> 3, j = si & 7;
      int lane, blk;
      if (vr < rem * (full + 1)) { lane = vr / (full + 1); blk = vr % (full + 1); }
      else { int const v2 = vr - rem * (full + 1); lane = rem + v2 / full; blk = v2 % full; }
      lp[8 * (blk * 32 + lane) + j] = x;
    }
    __syncthreads();
  }
}

// ---- bitonic sort helpers on shared memory (descending for keys, ascending for k-mers) ----------
template <typename T, bool DESC>
__device__ void bitonic_sort_shared(T * a, int n /* power of two */)
{
  for (int size = 2; size <= n; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int i = threadIdx.x; i < (n >> 1); i += blockDim.x) {
        int const lo = 2 * i - (i & (stride - 1));
        int const hi = lo + stride;
        bool const up = ((lo & size) == 0);
        T const x = a[lo], y = a[hi];
        bool const sw = DESC ? (up ? (x < y) : (x > y)) : (up ? (x > y) : (x < y));
        if (sw) { a[lo] = y; a[hi] = x; }
      }
    }
  }
  __syncthreads();
}

__device__ __forceinline__ int next_pow2(int v)
{
  int p = 1;
  while (p < v) { p <<= 1; }
  return p;
}

// ---- block-wide building blocks of the ranker -------------------------------------------------------------------------

// Warp 0 only.  hist[c] = how many targets have count c.  Returns the largest T in [floor, top] with at least `tophits`
// targets at or above it (floor if there is none), and in K how many targets in hist[T .. top] there are.
__device__ __forceinline__ int threshold_from_hist(const uint32_t * hist, int top, int floor, int tophits, int & K)
{
  int const lane = threadIdx.x & 31;
  int acc = 0;
  for (; top >= floor; top -= 32) {
    int const b = top - lane;
    // inclusive prefix over lanes = suffix over bins (lane 0 is the highest bin)
    int const v = warp_inclusive_sum(b >= floor ? static_cast<int>(hist[b]) : 0);
    unsigned const hit = __ballot_sync(0xffffffffu, acc + v >= tophits);
    if (hit != 0u) {
      int const first = __ffs(hit) - 1;
      K = acc + __shfl_sync(0xffffffffu, v, first);
      return top - first;
    }
    acc += __shfl_sync(0xffffffffu, v, 31);
  }
  K = acc;   // fewer than tophits targets: all of them
  return floor;
}

// Compacts the keys >= tkey of cand[0, m) (m <= CAND) in place to its front (in no order) and returns how many there
// are.  Every thread reads its keys before any is written back.
template <int CAND>
__device__ __forceinline__ int keep_keys_from(uint64_t * cand, int m, uint64_t tkey, int & s_ncand)
{
  uint64_t mine[(CAND + RANK_THREADS - 1) / RANK_THREADS];
  int cnt = 0;
  for (int i = threadIdx.x; i < m; i += blockDim.x) { uint64_t const kx = cand[i]; if (kx >= tkey) { mine[cnt++] = kx; } }
  if (threadIdx.x == 0) { s_ncand = 0; }
  __syncthreads();
  int const base = cnt > 0 ? atomicAdd(&s_ncand, cnt) : 0;
  for (int i = 0; i < cnt; i++) { cand[base + i] = mine[i]; }
  __syncthreads();
  return s_ncand;
}

// Sorts cand[0, m) best first (padded with zero keys to a power of two) and returns how many of them to keep,
// min(m, tophits).  Starts and ends with a barrier.
__device__ __forceinline__ int sort_and_cut(uint64_t * cand, int m, int tophits)
{
  int const p2 = next_pow2(m);
  for (int i = m + threadIdx.x; i < p2; i += blockDim.x) { cand[i] = 0; }
  bitonic_sort_shared<uint64_t, true>(cand, p2);
  return m < tophits ? m : tophits;
}

// ---- the steps of rank_kernel ------------------------------------------------------------------------------------------

// 1. A query of at most KMER_CAP windows: its k-mers in kmers[0, np2), sorted, np2 = the windows rounded up to a power
//    of two, duplicates and masked windows invalidated (0xffffffff).  flag: np2 words of scratch.  Returns the number
//    of distinct k-mers.
__device__ __forceinline__ int query_kmers_smem(const uint8_t * __restrict__ s, int nwin, int k, int mask_lower,
                                                uint32_t * kmers, uint32_t * flag, int & s_nk, int & np2)
{
  np2 = next_pow2(nwin > 1 ? nwin : 1);
  for (int i = threadIdx.x; i < np2; i += blockDim.x) {
    uint32_t km = 0xffffffffu;
    if (i < nwin) {
      uint32_t v;
      if (kmer_at(s, i + k - 1, k, mask_lower, v)) { km = v; }
    }
    kmers[i] = km;
  }
  bitonic_sort_shared<uint32_t, false>(kmers, np2);
  int mine = 0;
  for (int i = threadIdx.x; i < np2; i += blockDim.x) {
    uint32_t const v = kmers[i];
    bool const keep = (v != 0xffffffffu) && (i == 0 || kmers[i - 1] != v);
    flag[i] = keep ? 1u : 0u;
    mine += keep;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < np2; i += blockDim.x) { if (flag[i] == 0u) { kmers[i] = 0xffffffffu; } }
  atomicAdd(&s_nk, mine);
  __syncthreads();
  return s_nk;
}

// 1'. A longer query: its distinct k-mers, in no order, to gk[0, nk) in this CTA's HBM scratch, de-duplicated through
//     `words` words at bm: a 4^k-bit map, or for wordlength 11..15, where a 4^k-bit map per CTA is out of reach, an
//     open-addressing table of `words` (a power of two >= twice the windows) slots that does what unique_count_hash's
//     table does (core/unique.cpp:243-334).  Returns nk.
__device__ __forceinline__ int query_kmers_hbm(const uint8_t * __restrict__ s, int nwin, int k, int mask_lower,
                                               uint32_t * bm, int words, uint32_t * gk, int & s_nk)
{
  if (k <= 10) {
    for (int i = threadIdx.x; i < words; i += blockDim.x) { bm[i] = 0; }
    __syncthreads();
    for (int p = threadIdx.x; p < nwin; p += blockDim.x) {
      uint32_t v;
      if (kmer_at(s, p + k - 1, k, mask_lower, v)) {
        uint32_t const bit = 1u << (v & 31);
        uint32_t const old = atomicOr(&bm[v >> 5], bit);
        if ((old & bit) == 0) { gk[atomicAdd(&s_nk, 1)] = v; }
      }
    }
  } else {
    uint32_t const hmask = static_cast<uint32_t>(words) - 1u;
    for (int i = threadIdx.x; i < words; i += blockDim.x) { bm[i] = 0xffffffffu; }
    __syncthreads();
    for (int p = threadIdx.x; p < nwin; p += blockDim.x) {
      uint32_t v;
      if (kmer_at(s, p + k - 1, k, mask_lower, v)) {
        uint32_t slot = (v * 2654435761u) >> 7 & hmask;
        for (;;) {
          uint32_t const old = atomicCAS(&bm[slot], 0xffffffffu, v);
          if (old == 0xffffffffu) { gk[atomicAdd(&s_nk, 1)] = v; break; }
          if (old == v) { break; }
          slot = (slot + 1u) & hmask;
        }
      }
    }
  }
  __threadfence_block();
  __syncthreads();
  return s_nk;
}

// 3. Postings -> counters, incremental index: unpadded lists of 32-bit target numbers, one warp per list, coalesced
//    loads, shared-memory atomics (targets within a list are distinct, lists collide).
__device__ __forceinline__ void postings_incr(const ShardDev & S, int n, const uint32_t * lbeg, const uint32_t * llen,
                                              uint32_t * counters)
{
  int const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int li = warp; li < n; li += RANK_THREADS / 32) {
    uint32_t const len = llen[li];
    const uint32_t * __restrict__ pl = S.post32 + lbeg[li];
    for (uint32_t e = lane; e < len; e += 32) {
      uint32_t const a = __ldg(pl + e) - static_cast<uint32_t>(S.t0);
      atomicAdd(&counters[a >> 1], (a & 1) ? 0x10000u : 1u);
    }
  }
}

// RANK_TOP: the best `tophits` of every query in shared memory (tophits <= TOPHITS_MAX).  The unbounded path
// (rank_lists) runs the same k-mer extraction and posting stream twice: RANK_COUNT writes to out_n how many targets of
// each query reach the reference's threshold, RANK_EMIT writes their keys to keys[key_off[qi] ...] in no order.
enum { RANK_TOP = 0, RANK_COUNT = 1, RANK_EMIT = 2 };

// The shapes rank_kernel is compiled for, both of RANK_THREADS threads: CTAS per SM (the register bound of
// __launch_bounds__), KCAP k-mer slots per query, CAND candidate keys and SEG counter words per segment of the sort-and-cut scan (each
// segment appends at most 2 * SEG keys, so tophits + 2 * SEG <= CAND must hold).
//   RankFull: every mode and both indexes; queries of up to KCAP windows in shared memory, longer ones through HBM
//     scratch.  114 708 B of shared memory: two CTAs per SM.
//   RankShort: RANK_TOP on the static index with tophits <= 64, every query of the launch with np2 + nwin + 1 <= 512
//     (so its k-mers and the running threshold's histogram fit the k-mer array: at wordlength 8, queries of up to
//     262 nt).  75 796 B of shared memory and <= 40 registers (ptxas: 40, and 36 B of spill stores, none of them in
//     postings_stream's loop, whose code matches RankFull's): three CTAs per SM, 1.5x the posting loads in flight of
//     RankFull.  (256-thread CTAs with 8 vectors per lane would allow 80 registers; at 40 nothing in the loop spills.)
struct RankFull { static constexpr int CTAS = 2, KCAP = KMER_CAP, CAND = 2048, SEG = 512; };
struct RankShort { static constexpr int CTAS = 3, KCAP = 512, CAND = 256, SEG = 64, TOPHITS = 64; };

template <typename CFG>
constexpr size_t rank_smem() { return CFG::CAND * 8 + (COUNTER_WORDS + 3) * 4 + CFG::KCAP * 4 * 4 + 4; }
static_assert(rank_smem<RankFull>() == 114708 && rank_smem<RankShort>() == 75796, "rank_kernel's shared memory");
static_assert(RankShort::TOPHITS + 2 * RankShort::SEG <= RankShort::CAND, "a sort-and-cut segment must fit behind tophits keys");

template <typename CFG, bool INCR, int MODE = RANK_TOP>
__global__ void __launch_bounds__(RANK_THREADS, CFG::CTAS)
rank_kernel(DevSeqs qs, int64_t q0, int nq, DevSeqs db, const ShardDev * __restrict__ shards, int nshards,
            int k, int mask_lower, int minwordmatches, int tophits,
            uint32_t * __restrict__ out_seqno, uint32_t * __restrict__ out_count, int32_t * __restrict__ out_n,
            int32_t * __restrict__ status, uint32_t * __restrict__ scratch, size_t scratch_stride, int bitmap_words,
            const int64_t * __restrict__ key_off, uint64_t * __restrict__ keys)
{
  extern __shared__ __align__(16) unsigned char smem[];
  constexpr int KCAP = CFG::KCAP, CAND = CFG::CAND, SEG = CFG::SEG;
  uint64_t * const cand = reinterpret_cast<uint64_t *>(smem);                 // CAND
  uint32_t * const counters = reinterpret_cast<uint32_t *>(smem + CAND * 8);  // COUNTER_WORDS (+pad)
  uint32_t * const kmers = counters + COUNTER_WORDS + 3;                      // KCAP
  uint32_t * const lbeg = kmers + KCAP;                                       // KCAP
  uint32_t * const llen = lbeg + KCAP;                                        // KCAP
  uint32_t * const cum = llen + KCAP;                                         // KCAP + 1 (static index, flat stream)
  __shared__ int s_ncand, s_nk, s_T, s_K;
  __shared__ int s_wsum[RANK_THREADS / 32];

  int const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  bool clean = false;   // the counters are all zero (left so by the previous shard's last scan)
  for (int qi = blockIdx.x; qi < nq; qi += gridDim.x) {
    int64_t const q = q0 + qi;
    const uint8_t * __restrict__ s = qs.sym + qs.off[q];
    int const len = qs.len[q];
    int const nwin = len - k + 1;
    if (threadIdx.x == 0) { s_ncand = 0; s_nk = 0; }
    bool const longq = nwin > KCAP;
    if (longq && (scratch == nullptr || nwin > 65535)) {
      if (threadIdx.x == 0) { out_n[qi] = 0; atomicExch(status, 1); }
      continue;
    }
    // 1. the query's distinct k-mers: in shared memory, or in HBM scratch, fed through shared memory KCAP at a time
    int np2, nk, nchunks = 1;
    uint32_t * gk = nullptr;
    if (!longq) {
      nk = query_kmers_smem(s, nwin, k, mask_lower, kmers, lbeg, s_nk, np2);
    } else {
      uint32_t * const bm = scratch + static_cast<size_t>(blockIdx.x) * scratch_stride;
      gk = bm + bitmap_words;
      nk = query_kmers_hbm(s, nwin, k, mask_lower, bm, bitmap_words, gk, s_nk);
      nchunks = nk > 0 ? (nk + KCAP - 1) / KCAP : 1;
      np2 = 1;
    }
    // search_topscores: count >= min(minwordmatches, kmersamplecount)  (searchcore.cpp:320)
    uint32_t const minmatches = static_cast<uint32_t>(minwordmatches < nk ? minwordmatches : nk);
    // RUNNING THRESHOLD (queries with np2 + nk + 1 <= KCAP, i.e. up to ~1000 nt in RankFull): hist[c] counts,
    // over the shards seen so far, the targets whose k-mer count is c; T = the largest count with at
    // least `tophits` targets at or above it.  A target below T can never reach the final list, so
    // only counts >= T are turned into candidate keys: a few dozen per shard instead of the ~3 % of
    // all targets that pass the reference's fixed threshold (searchcore.cpp:320), no overflow sorts.
    bool const running = MODE == RANK_TOP && !longq && (np2 + nk + 1 <= KCAP);
    uint32_t * const hist = kmers + np2;  // nk + 1 bins in the unused tail of the k-mer array
    if (running) {
      for (int i = threadIdx.x; i <= nk; i += blockDim.x) { hist[i] = 0; }
      if (threadIdx.x == 0) { s_T = static_cast<int>(minmatches); }
    }

    for (int sh = 0; sh < nshards; sh++) {
      ShardDev const S = shards[sh];
      // 2. zero the counters; 3. for every chunk of k-mers, the bounds of their lists in this shard, then their postings
      if (!clean) { for (int i = threadIdx.x; i < COUNTER_WORDS; i += blockDim.x) { counters[i] = 0; } }
      clean = false;
      for (int chunk = 0; chunk < nchunks; chunk++) {
        if (longq) {
          int const cn = nk > 0 ? min(KCAP, nk - chunk * KCAP) : 1;
          for (int i = threadIdx.x; i < cn; i += blockDim.x) { kmers[i] = nk > 0 ? gk[chunk * KCAP + i] : 0xffffffffu; }
          np2 = cn;
          __syncthreads();
        }
        list_bounds<INCR>(S, kmers, np2, lbeg, llen);
        __syncthreads();
        if constexpr (INCR) { postings_incr(S, np2, lbeg, llen, counters); }
        else { postings_stream<KCAP>(S, np2, lbeg, llen, cum, counters, s_wsum); }
        __syncthreads();
      }
      // 4. collect this shard's candidates
      int const nwords = (S.nt + 1) >> 1;
      uint32_t thr = minmatches;
      if constexpr (MODE != RANK_TOP) {
        // 4u. every target at or above the threshold; the counters are cleared behind the scan
        visit_counters<4>(counters, 0, nwords, S.nt, minmatches, true, [&](uint32_t c, int lt) {
          int const pos = atomicAdd(&s_ncand, 1);
          if (MODE == RANK_EMIT) { keys[key_off[qi] + pos] = target_key(db, S, c, lt); }
        });
        clean = true;
        __syncthreads();
        continue;  // next shard
      }
      if (running) {
        // 4r. histogram of this shard's counts >= T, new T, then keys for counts >= new T only
        uint32_t const T0 = static_cast<uint32_t>(s_T);
        visit_counters<4>(counters, 0, nwords, S.nt, T0, false, [&](uint32_t c, int) { atomicAdd(&hist[c], 1u); });
        __syncthreads();
        if (warp == 0) {
          int K;
          int const T = threshold_from_hist(hist, nk, static_cast<int>(T0), tophits, K);
          if (lane == 0) { s_T = T; s_K = K; }
        }
        int const level = s_ncand;
        __syncthreads();
        uint32_t const T1 = static_cast<uint32_t>(s_T);
        if (level + s_K <= CAND) {
          // at most K targets (all shards so far) are >= T1, so at most K keys are appended here
          visit_counters<4>(counters, 0, nwords, S.nt, T1, true, [&](uint32_t c, int lt) {
            cand[atomicAdd(&s_ncand, 1)] = target_key(db, S, c, lt);
          });
          clean = true;
          __syncthreads();
          continue;  // next shard
        }
        thr = T1;  // a crowd of ties at T1: the sort-and-cut path below, from T1 up
      } else {
        // 4. threshold scan.  Common case: count the survivors, one block-wide prefix sum, write them straight to
        //    their slots (no barrier per segment).  Only if they would not fit does the sort-and-cut path below run.
        int mine = 0;
        visit_counters<1>(counters, 0, nwords, S.nt, minmatches, false, [&](uint32_t, int) { mine++; });
        int total;
        int pos = block_exclusive_sum(mine, s_wsum, total);
        int const level = s_ncand;
        __syncthreads();
        if (level + total <= CAND) {
          pos += level;
          visit_counters<1>(counters, 0, nwords, S.nt, minmatches, false, [&](uint32_t c, int lt) {
            cand[pos++] = target_key(db, S, c, lt);
          });
          if (threadIdx.x == 0) { s_ncand = level + total; }
          __syncthreads();
          continue;  // next shard
        }
      }
      // 4b. segmented scan with sort-and-cut when the candidate list could overflow
      for (int seg = 0; seg < nwords; seg += SEG) {
        // every thread must take the same decision: read the fill level, then fence the read off
        // from the appends of threads that are already past this point
        int const level = s_ncand;
        __syncthreads();
        if (level + 2 * SEG > CAND) {
          int const nkeep = sort_and_cut(cand, level, tophits);
          if (threadIdx.x == 0) { s_ncand = nkeep; }
          __syncthreads();
        }
        visit_counters<1>(counters, seg, min(seg + SEG, nwords), S.nt, thr, false, [&](uint32_t c, int lt) {
          cand[atomicAdd(&s_ncand, 1)] = target_key(db, S, c, lt);
        });
        __syncthreads();
      }
    }
    // 5. finish the query
    if constexpr (MODE != RANK_TOP) {
      if (threadIdx.x == 0) { out_n[qi] = s_ncand; }
      __syncthreads();
      continue;  // next query
    }
    // Usually far more targets pass the k-mer threshold than are wanted: find the count T of the tophits-th best,
    // keep count >= T, sort only those.  (A running query has nk < KCAP and its T already.)
    int m = s_ncand;
    __syncthreads();
    if (m > 2 * tophits && nk + 1 <= 2 * KCAP) {
      if (!running) {
        uint32_t * const hist5 = lbeg;  // 2 * KCAP words available, counts are <= nk
        for (int i = threadIdx.x; i <= nk; i += blockDim.x) { hist5[i] = 0; }
        __syncthreads();
        for (int i = threadIdx.x; i < m; i += blockDim.x) { atomicAdd(&hist5[static_cast<uint32_t>(cand[i] >> 49)], 1u); }
        __syncthreads();
        if (warp == 0) {
          int K;
          int const T = threshold_from_hist(hist5, nk, 0, tophits, K);
          if (lane == 0) { s_T = T; }
        }
        __syncthreads();
      }
      // running: the keys below the final T were appended while T was still lower
      m = keep_keys_from<CAND>(cand, m, count_key(s_T), s_ncand);
    }
    int const nout = sort_and_cut(cand, m, tophits);
    for (int i = threadIdx.x; i < nout; i += blockDim.x) {
      uint64_t const key = cand[i];
      out_seqno[static_cast<size_t>(qi) * tophits + i] = 0xffffffu - static_cast<uint32_t>(key & 0xffffffu);
      out_count[static_cast<size_t>(qi) * tophits + i] = static_cast<uint32_t>(key >> 49);
    }
    if (threadIdx.x == 0) { out_n[qi] = nout; }
    __syncthreads();
  }
}


}  // namespace vsg

using namespace vsg;

struct vsg_index {
  int device = 0;
  int k = 8;
  int mask_lower = 0;
  int64_t ntargets = 0;
  const vsg_seqset * db = nullptr;
  std::vector<DevBuf> b_start, b_post, b_rkeys;
  std::vector<ShardDev> h_shards;
  DevBuf b_shards;
  int64_t total_postings = 0;
  // per k-mer, the number of targets holding it (Dbindex::getmatchcount), 4^k words: built on first use by
  // index_word_counts, under the lock because an index is shared read-only by several contexts and threads
  mutable std::mutex words_lock;
  mutable DevBuf b_words;
  mutable bool words_ready = false;
};

extern "C" void vsg_index_destroy(vsg_index * ix);
namespace vsg {

static void shard_bank_order(vsg_ctx * c, const uint32_t * start, uint16_t * post, size_t nlists)
{
  if (nlists == 0) { return; }
  int sms = 132;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device);
  list_bank_order_kernel<<<static_cast<int>(std::min<size_t>(nlists, static_cast<size_t>(sms) * 32)), 128, 0, c->stream>>>(start, post, static_cast<int>(nlists));
  count_launch();
}

// dense shard (k <= 10): start[2 * 4^k + 1], two sub-lists per k-mer
static int build_dense_shard(vsg_ctx * c, vsg_index * ix, int sh, int t0, int nt, DevBuf & cnt, DevBuf & tmp, uint32_t * d_totals)
{
  const vsg_seqset * db = ix->db;
  int const k = ix->k;
  size_t const hashsize = static_cast<size_t>(1) << (2 * k);
  size_t const bitmap_bytes = std::max<size_t>(hashsize / 8, 4);
  size_t const nlists = 2 * hashsize;   // even and odd targets of every k-mer
  int rc;
  // list offsets are 32-bit: a shard's postings (at most one per nucleotide) plus the padding of its lists must fit
  int64_t nuc = 0;
  for (int i = 0; i < nt; i++) { nuc += db->h_len[static_cast<size_t>(t0) + static_cast<size_t>(i)]; }
  if (nuc + 7 * static_cast<int64_t>(nlists) >= (static_cast<int64_t>(1) << 32) - 64) {
    Error::set("vsg_index_create: a shard of 32766 targets holds 2^32 nucleotides or more");
    return VSG_EINVAL;
  }
  DevBuf & bs = ix->b_start[static_cast<size_t>(sh)];
  if ((rc = bs.reserve(sizeof(uint32_t) * (nlists + 1))) != VSG_OK) { return rc; }
  VSG_CUDA_OK(cudaMemsetAsync(cnt.p, 0, sizeof(uint32_t) * (nlists + 1), c->stream));
  index_build_kernel<false><<<nt, 128, bitmap_bytes, c->stream>>>(db->d, t0, nt, k, ix->mask_lower, 1,
                                                                  static_cast<uint32_t *>(cnt.p), nullptr, nullptr);
  count_launch();
  if (d_totals != nullptr) {
    add_totals_kernel<<<static_cast<unsigned>((hashsize + 255) / 256), 256, 0, c->stream>>>(static_cast<const uint32_t *>(cnt.p), d_totals, hashsize);
    count_launch();
  }
  pad_counts_kernel<<<static_cast<unsigned>((nlists + 255) / 256), 256, 0, c->stream>>>(static_cast<uint32_t *>(cnt.p), static_cast<int>(nlists));
  count_launch();
  size_t tb = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tb, static_cast<uint32_t *>(cnt.p), static_cast<uint32_t *>(bs.p),
                                static_cast<int>(nlists + 1), c->stream);
  if ((rc = tmp.reserve(tb + 16)) != VSG_OK) { return rc; }
  cub::DeviceScan::ExclusiveSum(tmp.p, tb, static_cast<uint32_t *>(cnt.p), static_cast<uint32_t *>(bs.p),
                                static_cast<int>(nlists + 1), c->stream);
  count_launch();
  uint32_t total = 0;
  VSG_CUDA_OK(cudaMemcpyAsync(&total, static_cast<uint32_t *>(bs.p) + nlists, sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
  VSG_CUDA_OK(cudaStreamSynchronize(c->stream));
  DevBuf & bp = ix->b_post[static_cast<size_t>(sh)];
  if ((rc = bp.reserve(sizeof(uint16_t) * (static_cast<size_t>(total) + 64))) != VSG_OK) { return rc; }
  VSG_CUDA_OK(cudaMemsetAsync(cnt.p, 0, sizeof(uint32_t) * (nlists + 1), c->stream));
  if (total > 0) {
    fill_u16_kernel<<<static_cast<unsigned>((static_cast<size_t>(total) + 255) / 256), 256, 0, c->stream>>>(
        static_cast<uint16_t *>(bp.p), static_cast<size_t>(total), POST_PAD);
    count_launch();
  }
  index_build_kernel<true><<<nt, 128, bitmap_bytes, c->stream>>>(db->d, t0, nt, k, ix->mask_lower, 1,
                                                                 static_cast<uint32_t *>(cnt.p),
                                                                 static_cast<uint32_t *>(bs.p),
                                                                 static_cast<uint16_t *>(bp.p));
  count_launch();
  if (total > 0) { shard_bank_order(c, static_cast<const uint32_t *>(bs.p), static_cast<uint16_t *>(bp.p), nlists); }
  ShardDev sd{};
  sd.start = static_cast<uint32_t *>(bs.p); sd.post = static_cast<uint16_t *>(bp.p); sd.t0 = t0; sd.nt = nt;
  ix->h_shards.push_back(sd);
  ix->total_postings += total;
  return VSG_OK;
}

// sparse shard (k 11..15): sort the windows' keys, drop duplicates, run-length encode the sub-lists
struct SparseScratch { DevBuf keys0, keys1, runs, cum, num, tmp; void release() { keys0.release(); keys1.release(); runs.release(); cum.release(); num.release(); tmp.release(); } };
static int build_sparse_shard(vsg_ctx * c, vsg_index * ix, int sh, int t0, int nt, SparseScratch & w, uint32_t * d_totals)
{
  const vsg_seqset * db = ix->db;
  int rc;
  // window slots of the shard's targets back to back, whatever the layout of the sequence set
  std::vector<int64_t> cum(static_cast<size_t>(nt) + 1, 0);
  for (int i = 0; i < nt; i++) { cum[static_cast<size_t>(i) + 1] = cum[static_cast<size_t>(i)] + db->h_len[static_cast<size_t>(t0) + static_cast<size_t>(i)]; }
  int64_t const W = cum[static_cast<size_t>(nt)];
  if (W >= (static_cast<int64_t>(1) << 31) - 64) { Error::set("vsg_index_create: a shard of 32766 targets holds 2^31 nucleotides or more (wordlength > 10)"); return VSG_EINVAL; }
  DevBuf & bs = ix->b_start[static_cast<size_t>(sh)];
  DevBuf & bp = ix->b_post[static_cast<size_t>(sh)];
  DevBuf & bk = ix->b_rkeys[static_cast<size_t>(sh)];
  int const n = static_cast<int>(W);
  uint32_t nr = 0, total = 0;
  if (n > 0) {
    if ((rc = w.keys0.reserve(sizeof(uint64_t) * (static_cast<size_t>(n) + 8))) != VSG_OK ||
        (rc = w.keys1.reserve(sizeof(uint64_t) * (static_cast<size_t>(n) + 8))) != VSG_OK ||
        (rc = w.cum.reserve(sizeof(int64_t) * (static_cast<size_t>(nt) + 1))) != VSG_OK ||
        (rc = w.num.reserve(64)) != VSG_OK) { return rc; }
    uint64_t * const k0 = static_cast<uint64_t *>(w.keys0.p);
    uint64_t * const k1 = static_cast<uint64_t *>(w.keys1.p);
    uint32_t * const d_num = static_cast<uint32_t *>(w.num.p);
    VSG_CUDA_OK(cudaMemcpyAsync(w.cum.p, cum.data(), sizeof(int64_t) * (static_cast<size_t>(nt) + 1), cudaMemcpyHostToDevice, c->stream));
    sparse_keys_kernel<<<nt, 128, 0, c->stream>>>(db->d, t0, nt, ix->k, ix->mask_lower, static_cast<const int64_t *>(w.cum.p), k0);
    count_launch();
    VSG_CUDA_OK(cudaStreamSynchronize(c->stream));   // `cum` (pageable) has been consumed
    size_t tb = 0, tb2 = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, tb, k0, k1, n, 0, 46, c->stream);
    cub::DeviceSelect::Unique(nullptr, tb2, k1, k0, d_num, n, c->stream);
    if ((rc = w.tmp.reserve(std::max(tb, tb2) + 64)) != VSG_OK) { return rc; }
    cub::DeviceRadixSort::SortKeys(w.tmp.p, tb, k0, k1, n, 0, 46, c->stream);
    count_launch();
    cub::DeviceSelect::Unique(w.tmp.p, tb2, k1, k0, d_num, n, c->stream);
    count_launch();
    uint32_t nu = 0;
    VSG_CUDA_OK(cudaMemcpyAsync(&nu, d_num, sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    VSG_CUDA_OK(cudaStreamSynchronize(c->stream));
    // k0[0 .. nu): the distinct keys in order, closed by the invalid key if any window was unusable.
    // Sub-lists = runs of key >> 14; the invalid key's run has id 0x80000000 and comes last.
    if ((rc = w.runs.reserve(sizeof(uint32_t) * 2 * (static_cast<size_t>(nu) + 2))) != VSG_OK ||
        (rc = bk.reserve(sizeof(uint32_t) * (static_cast<size_t>(nu) + 2))) != VSG_OK) { return rc; }
    uint32_t * const rcnt = static_cast<uint32_t *>(w.runs.p);
    uint32_t * const rsrc = rcnt + nu + 2;
    uint32_t * const rkeys = static_cast<uint32_t *>(bk.p);
    VSG_CUDA_OK(cudaMemsetAsync(rcnt, 0, sizeof(uint32_t) * 2 * (static_cast<size_t>(nu) + 2), c->stream));
    uint32_t nruns = 0;
    if (nu > 0) {
      auto runs_in = thrust::make_transform_iterator(static_cast<const uint64_t *>(k0), SparseRunOf());
      size_t tb3 = 0;
      cub::DeviceRunLengthEncode::Encode(nullptr, tb3, runs_in, rkeys, rcnt, d_num, static_cast<int>(nu), c->stream);
      if ((rc = w.tmp.reserve(tb3 + 64)) != VSG_OK) { return rc; }
      cub::DeviceRunLengthEncode::Encode(w.tmp.p, tb3, runs_in, rkeys, rcnt, d_num, static_cast<int>(nu), c->stream);
      count_launch();
      VSG_CUDA_OK(cudaMemcpyAsync(&nruns, d_num, sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
      VSG_CUDA_OK(cudaStreamSynchronize(c->stream));
      if (nruns > 0) {
        uint32_t lastkey = 0;
        VSG_CUDA_OK(cudaMemcpyAsync(&lastkey, rkeys + (nruns - 1), sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
        VSG_CUDA_OK(cudaStreamSynchronize(c->stream));
        if (lastkey >= 0x80000000u) { nruns--; }
      }
    }
    nr = nruns;
    if (nr > 0) {
      if ((rc = bs.reserve(sizeof(uint32_t) * (static_cast<size_t>(nr) + 2))) != VSG_OK) { return rc; }
      // source offsets (plain counts) and destination offsets (counts padded to vectors of 8) of every sub-list
      size_t tb4 = 0, tb5 = 0;
      auto padded = thrust::make_transform_iterator(static_cast<const uint32_t *>(rcnt), PadTo8());
      cub::DeviceScan::ExclusiveSum(nullptr, tb4, rcnt, rsrc, static_cast<int>(nr + 1), c->stream);
      cub::DeviceScan::ExclusiveSum(nullptr, tb5, padded, static_cast<uint32_t *>(bs.p), static_cast<int>(nr + 1), c->stream);
      if ((rc = w.tmp.reserve(std::max(tb4, tb5) + 64)) != VSG_OK) { return rc; }
      cub::DeviceScan::ExclusiveSum(w.tmp.p, tb4, rcnt, rsrc, static_cast<int>(nr + 1), c->stream);
      count_launch();
      cub::DeviceScan::ExclusiveSum(w.tmp.p, tb5, padded, static_cast<uint32_t *>(bs.p), static_cast<int>(nr + 1), c->stream);
      count_launch();
      VSG_CUDA_OK(cudaMemcpyAsync(&total, static_cast<uint32_t *>(bs.p) + nr, sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
      VSG_CUDA_OK(cudaStreamSynchronize(c->stream));
      if ((rc = bp.reserve(sizeof(uint16_t) * (static_cast<size_t>(total) + 64))) != VSG_OK) { return rc; }
      fill_u16_kernel<<<static_cast<unsigned>((static_cast<size_t>(total) + 255) / 256), 256, 0, c->stream>>>(
          static_cast<uint16_t *>(bp.p), static_cast<size_t>(total), POST_PAD);
      count_launch();
      sparse_scatter_kernel<<<(nr + 127) / 128, 128, 0, c->stream>>>(k0, rkeys, rcnt, rsrc, static_cast<const uint32_t *>(bs.p), nr,
                                                                    static_cast<uint16_t *>(bp.p), d_totals);
      count_launch();
      shard_bank_order(c, static_cast<const uint32_t *>(bs.p), static_cast<uint16_t *>(bp.p), nr);
      VSG_CUDA_OK(cudaStreamSynchronize(c->stream));
    }
  }
  if (nr == 0) {
    // no usable window in the whole shard: one empty sub-list under a key no k-mer has
    if ((rc = bs.reserve(16)) != VSG_OK || (rc = bp.reserve(128)) != VSG_OK || (rc = bk.reserve(16)) != VSG_OK) { return rc; }
    VSG_CUDA_OK(cudaMemsetAsync(bs.p, 0, 16, c->stream));
    VSG_CUDA_OK(cudaMemsetAsync(bk.p, 0xff, 16, c->stream));
    nr = 1;
  }
  ShardDev sd{};
  sd.t0 = t0; sd.nt = nt;
  sd.start = static_cast<uint32_t *>(bs.p); sd.post = static_cast<uint16_t *>(bp.p);
  sd.rkeys = static_cast<uint32_t *>(bk.p); sd.nr = nr;
  ix->h_shards.push_back(sd);
  ix->total_postings += total;
  return VSG_OK;
}

// d_totals (optional): 4^k words on the device, zeroed by the caller; receives the number of targets holding each k-mer
int index_create_counts(vsg_ctx * c, const vsg_seqset * db, int wordlength, int mask_lower, uint32_t * d_totals, vsg_index ** out)
{
  if (c == nullptr || db == nullptr || out == nullptr) { Error::set("vsg_index_create: null argument"); return VSG_EINVAL; }
  *out = nullptr;
  if (wordlength < 3 || wordlength > 15) {
    Error::set("vsg_index_create: --wordlength must be in 3..15");
    return VSG_EINVAL;
  }
  if (db->device != c->device) { Error::set("vsg_index_create: the sequence set lives on another device than the context"); return VSG_EINVAL; }
  if (db->d.n > (1 << 24)) { Error::set("vsg_index_create: more than 2^24 targets"); return VSG_EINVAL; }
  VSG_CUDA_OK(cudaSetDevice(c->device));
  int const k = wordlength;
  bool const sparse = k > 10;
  size_t const hashsize = static_cast<size_t>(1) << (2 * k);
  if (!sparse) {
    size_t const bitmap_bytes = std::max<size_t>(hashsize / 8, 4);
    if (bitmap_bytes > 48 * 1024) {
      VSG_CUDA_OK(cudaFuncSetAttribute(index_build_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bitmap_bytes)));
      VSG_CUDA_OK(cudaFuncSetAttribute(index_build_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bitmap_bytes)));
    }
  }
  vsg_index * ix = new (std::nothrow) vsg_index();
  if (ix == nullptr) { Error::set("out of host memory"); return VSG_ENOMEM; }
  ix->device = c->device; ix->k = wordlength; ix->mask_lower = mask_lower; ix->ntargets = db->d.n; ix->db = db;
  int const nshards = static_cast<int>((db->d.n + SHARD_STATIC - 1) / SHARD_STATIC);
  ix->b_start.resize(static_cast<size_t>(nshards));
  ix->b_post.resize(static_cast<size_t>(nshards));
  ix->b_rkeys.resize(static_cast<size_t>(nshards));
  DevBuf cnt, tmp;
  SparseScratch w;
  int rc = VSG_OK;
  if (!sparse) { rc = cnt.reserve(sizeof(uint32_t) * (2 * hashsize + 1)); }
  for (int sh = 0; sh < nshards && rc == VSG_OK; sh++) {
    int const t0 = sh * SHARD_STATIC;
    int const nt = static_cast<int>(std::min<int64_t>(SHARD_STATIC, db->d.n - t0));
    rc = sparse ? build_sparse_shard(c, ix, sh, t0, nt, w, d_totals) : build_dense_shard(c, ix, sh, t0, nt, cnt, tmp, d_totals);
  }
  if (rc == VSG_OK) { rc = ix->b_shards.reserve(sizeof(ShardDev) * (ix->h_shards.size() + 1)); }
  cudaError_t e = cudaSuccess;
  if (rc == VSG_OK && !ix->h_shards.empty()) {
    e = cudaMemcpyAsync(ix->b_shards.p, ix->h_shards.data(), sizeof(ShardDev) * ix->h_shards.size(), cudaMemcpyHostToDevice, c->stream);
  }
  if (rc == VSG_OK && e == cudaSuccess) { e = cudaStreamSynchronize(c->stream); }
  if (rc == VSG_OK && e == cudaSuccess) { e = cudaGetLastError(); }
  cnt.release(); tmp.release(); w.release();
  if (rc == VSG_OK && e != cudaSuccess) { Error::set(std::string("vsg_index_create: ") + cudaGetErrorString(e)); rc = VSG_ECUDA; }
  if (rc != VSG_OK) { vsg_index_destroy(ix); return rc; }
  *out = ix;
  return VSG_OK;
}
}  // namespace vsg

extern "C" int vsg_index_create(vsg_ctx * c, const vsg_seqset * db, int wordlength, int mask_lower,
                                vsg_index ** out)
{
  return vsg::index_create_counts(c, db, wordlength, mask_lower, nullptr, out);
}

extern "C" void vsg_index_destroy(vsg_index * ix)
{
  if (ix == nullptr) { return; }
  cudaSetDevice(ix->device);
  for (auto & b : ix->b_start) { b.release(); }
  for (auto & b : ix->b_post) { b.release(); }
  for (auto & b : ix->b_rkeys) { b.release(); }
  ix->b_shards.release();
  ix->b_words.release();
  delete ix;
}

namespace vsg {
const vsg_seqset * index_db(const vsg_index * ix) { return ix->db; }
int index_wordlength(const vsg_index * ix) { return ix->k; }

int index_word_counts(vsg_ctx * c, const vsg_index * ix, const uint32_t ** out)
{
  std::lock_guard<std::mutex> const lock(ix->words_lock);
  if (!ix->words_ready) {
    size_t const hashsize = static_cast<size_t>(1) << (2 * ix->k);
    int const rc = ix->b_words.reserve(sizeof(uint32_t) * hashsize);
    if (rc != VSG_OK) { return rc; }
    uint32_t * const words = static_cast<uint32_t *>(ix->b_words.p);
    VSG_CUDA_OK(cudaMemsetAsync(words, 0, sizeof(uint32_t) * hashsize, c->stream));
    for (ShardDev const & S : ix->h_shards) {
      uint32_t const nlists = S.nr != 0 ? S.nr : static_cast<uint32_t>(2 * hashsize);
      shard_word_counts_kernel<<<(nlists + 255) / 256, 256, 0, c->stream>>>(S, nlists, words);
      count_launch();
    }
    VSG_CUDA_OK(cudaStreamSynchronize(c->stream));
    VSG_CUDA_OK(cudaGetLastError());
    ix->words_ready = true;
  }
  *out = static_cast<const uint32_t *>(ix->b_words.p);
  return VSG_OK;
}
const ShardDev * index_shards(const vsg_index * ix, int & nshards)
{
  nshards = static_cast<int>(ix->h_shards.size());
  return static_cast<const ShardDev *>(ix->b_shards.p);
}

// call after the stream has been synchronised
static void rank_collect_time(vsg_ctx * c)
{
  if (c->rank_pending) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, c->ev[4], c->ev[5]) == cudaSuccess) { c->prof_rank_ms += ms; }
    c->rank_pending = false;
  }
}

// Room for the bounded ranker's results of nq queries in ctx->rank_tmp, laid out as [seqno nq*tophits]
// [count nq*tophits][n nq][status 1], the status cleared.  tophits 0: n and status only.
static int rank_top_alloc(vsg_ctx * c, int64_t nq, int tophits, RankTop & r)
{
  size_t const cells = static_cast<size_t>(nq) * tophits;
  int rc;
  if ((rc = c->rank_tmp.reserve(sizeof(uint32_t) * (2 * cells + nq + 4))) != VSG_OK) { return rc; }
  r.seqno = static_cast<uint32_t *>(c->rank_tmp.p);
  r.count = r.seqno + cells;
  r.n = reinterpret_cast<int32_t *>(r.count + cells);
  r.status = r.n + nq;
  VSG_CUDA_OK(cudaMemsetAsync(r.status, 0, sizeof(int32_t), c->stream));
  return VSG_OK;
}

static int rank_status(int32_t status, const char * caller)
{
  if (status == 0) { return VSG_OK; }
  Error::set(std::string(caller) + ": a query is longer than the device ranker supports (65 534 + wordlength nt)");
  return VSG_EINVAL;
}

RankTargets index_targets(const vsg_index * ix, int mask_lower)
{
  RankTargets t;
  t.shards = static_cast<const ShardDev *>(ix->b_shards.p); t.nshards = static_cast<int>(ix->h_shards.size());
  t.lens = ix->db->d; t.k = ix->k; t.mask_lower = mask_lower; t.device = ix->device;
  t.incr = false; t.timed = true;
  return t;
}

// Whether rank_kernel<RankShort> can rank a launch of RANK_TOP on the static index whose longest query has maxlen nt:
// every query's np2 + nwin + 1 must fit RankShort::KCAP, and np2 + nwin grows with the length.
static bool rank_short_fits(bool incr, int tophits, int maxlen, int k)
{
  int const nwin = std::max(1, maxlen - k + 1);
  int np2 = 1;
  while (np2 < nwin) { np2 <<= 1; }
  return !incr && tophits <= RankShort::TOPHITS && np2 + nwin + 1 <= RankShort::KCAP;
}

// Launches rank_kernel on c's stream over queries [q0, q0 + nq) (nq >= 1) against t's shards: rank_kernel<RankShort>
// (three CTAs per SM) when rank_short_fits, else rank_kernel<RankFull, t.incr, MODE> (two CTAs per SM) with HBM
// scratch when a query has more than KMER_CAP windows.  t.timed: ev[4..5] around the launch, added to
// vsg_profile.rank_ms by rank_collect_time.
template <int MODE>
static int rank_launch(vsg_ctx * c, const RankTargets & t, const vsg_seqset * queries, int64_t q0, int64_t nq,
                       int minwordmatches, int tophits, const RankTop & out, const int64_t * d_key_off, uint64_t * d_keys)
{
  int rc;
  int const k = t.k;
  int maxlen = 0;
  for (int64_t q = q0; q < q0 + nq; q++) { maxlen = std::max(maxlen, queries->h_len[static_cast<size_t>(q)]); }
  bool const small = MODE == RANK_TOP && rank_short_fits(t.incr, tophits, maxlen, k);
  auto const kernel = small ? rank_kernel<RankShort, false, RANK_TOP>
                            : t.incr ? rank_kernel<RankFull, true, MODE> : rank_kernel<RankFull, false, MODE>;
  size_t const smem = small ? rank_smem<RankShort>() : rank_smem<RankFull>();
  VSG_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  int sms = 132;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device);
  int const grid = static_cast<int>(std::min<int64_t>(nq, static_cast<int64_t>(sms) * (small ? RankShort::CTAS : RankFull::CTAS)));
  // queries with more than KMER_CAP windows de-duplicate their k-mers in HBM scratch
  uint32_t * d_scratch = nullptr;
  size_t stride = 0;
  int bitmap_words = std::max(1, (1 << (2 * std::min(k, 10))) >> 5);
  if (k > 10) { bitmap_words = 4096; while (bitmap_words < 2 * maxlen) { bitmap_words <<= 1; } }   // hash slots (power of two)
  if (maxlen - k + 1 > KMER_CAP) {
    stride = static_cast<size_t>(bitmap_words) + static_cast<size_t>(maxlen) + 8;
    if ((rc = c->rank_scratch.reserve(sizeof(uint32_t) * stride * static_cast<size_t>(grid))) != VSG_OK) { return rc; }
    d_scratch = static_cast<uint32_t *>(c->rank_scratch.p);
  }
  if (t.timed) { VSG_CUDA_OK(cudaEventRecord(c->ev[4], c->stream)); }
  kernel<<<grid, RANK_THREADS, smem, c->stream>>>(
      queries->d, q0, static_cast<int>(nq), t.lens, t.shards, t.nshards, k, t.mask_lower, minwordmatches, tophits,
      out.seqno, out.count, out.n, out.status, d_scratch, stride, bitmap_words, d_key_off, d_keys);
  count_launch();
  if (t.timed) {
    VSG_CUDA_OK(cudaEventRecord(c->ev[5], c->stream));
    c->rank_pending = true;
  }
  return VSG_OK;
}

// the static index's ranker over queries [q0, q0 + nq) on c's stream; results as RankTop in ctx->rank_tmp
int rank_enqueue(vsg_ctx * c, const vsg_index * ix, const vsg_seqset * queries, int64_t q0, int64_t nq,
                 int minwordmatches, int tophits, int mask_lower, RankTop & out)
{
  if (tophits < 1 || tophits > TOPHITS_MAX) { Error::set("vsg_rank: tophits must be in 1..1024"); return VSG_EINVAL; }
  if (q0 < 0 || nq < 0 || q0 + nq > queries->d.n) { Error::set("vsg_rank: query range out of bounds"); return VSG_EINVAL; }
  if (queries->device != c->device || ix->device != c->device) { Error::set("vsg_rank: sequence set / index lives on another device than the context"); return VSG_EINVAL; }
  if (nq > (1 << 30) / tophits) { Error::set("vsg_rank: batch too large"); return VSG_EINVAL; }
  int rc;
  if ((rc = rank_top_alloc(c, nq, tophits, out)) != VSG_OK || nq == 0) { return rc; }
  return rank_launch<RANK_TOP>(c, index_targets(ix, mask_lower), queries, q0, nq, minwordmatches, tophits, out, nullptr, nullptr);
}

int rank_download(vsg_ctx * c, const RankTop & r, int64_t nq, int tophits, uint32_t * h_seqno, uint32_t * h_count,
                  int32_t * h_n, const char * caller)
{
  size_t const cells = static_cast<size_t>(nq) * tophits;
  int32_t status = 0;
  if (nq > 0) {
    VSG_CUDA_OK(cudaMemcpyAsync(h_seqno, r.seqno, sizeof(uint32_t) * cells, cudaMemcpyDeviceToHost, c->stream));
    VSG_CUDA_OK(cudaMemcpyAsync(h_count, r.count, sizeof(uint32_t) * cells, cudaMemcpyDeviceToHost, c->stream));
    VSG_CUDA_OK(cudaMemcpyAsync(h_n, r.n, sizeof(int32_t) * static_cast<size_t>(nq), cudaMemcpyDeviceToHost, c->stream));
  }
  VSG_CUDA_OK(cudaMemcpyAsync(&status, r.status, sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
  VSG_CUDA_OK(cudaStreamSynchronize(c->stream));
  rank_collect_time(c);
  return rank_status(status, caller);
}

// the first min(n, tophits) sorted keys of every query of a chunk as (target, count): one block per query
__global__ void cut_lists_kernel(const uint64_t * __restrict__ keys, const int64_t * __restrict__ key_off,
                                 const int64_t * __restrict__ out_off, uint32_t * __restrict__ seqno, uint32_t * __restrict__ count)
{
  int const q = blockIdx.x;
  int64_t const a = key_off[q], n = out_off[q + 1] - out_off[q], o = out_off[q];
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    uint64_t const key = keys[a + i];
    seqno[o + i] = 0xffffffu - static_cast<uint32_t>(key & 0xffffffu);
    count[o + i] = static_cast<uint32_t>(key >> 49);
  }
}

// The count pass of the unbounded ranker: n[i] = the number of targets query q0 + i has at or above the reference's
// threshold, min(minwordmatches, distinct k-mers) (its whole candidate list before any cut)
int rank_counts(vsg_ctx * c, const RankTargets & t, const vsg_seqset * queries, int64_t q0, int64_t nq, int minwordmatches,
                std::vector<int32_t> & n)
{
  if (q0 < 0 || nq < 0 || q0 + nq > queries->d.n) { Error::set("vsg_rank: query range out of bounds"); return VSG_EINVAL; }
  if (queries->device != c->device || t.device != c->device) { Error::set("vsg_rank: sequence set / index lives on another device than the context"); return VSG_EINVAL; }
  if (nq > (1 << 30)) { Error::set("vsg_rank: batch too large"); return VSG_EINVAL; }
  n.assign(static_cast<size_t>(nq), 0);
  if (nq == 0) { return VSG_OK; }
  RankTop r;
  int rc;
  if ((rc = rank_top_alloc(c, nq, 0, r)) != VSG_OK ||
      (rc = rank_launch<RANK_COUNT>(c, t, queries, q0, nq, minwordmatches, 1, r, nullptr, nullptr)) != VSG_OK) { return rc; }
  int32_t status = 0;
  VSG_CUDA_OK(cudaMemcpyAsync(n.data(), r.n, sizeof(int32_t) * static_cast<size_t>(nq), cudaMemcpyDeviceToHost, c->stream));
  VSG_CUDA_OK(cudaMemcpyAsync(&status, r.status, sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
  VSG_CUDA_OK(cudaStreamSynchronize(c->stream));
  rank_collect_time(c);
  return rank_status(status, "vsg_rank");
}

// The unbounded ranker (any tophits): query i's list is seqno / count[first[i] .. first[i + 1]), best first, the
// targets with count >= min(minwordmatches, distinct k-mers) cut to tophits.  A count pass sizes every list; then, for
// as many queries as the key budget holds at a time, an emit pass writes the keys, a segmented sort orders each
// query's keys and cut_lists_kernel keeps the first tophits.  Keys, sort buffers and lists take 24 bytes per candidate
// from a quarter of the context's direction-bit budget (a share of the device's free memory, vsg_ctx_create).  When
// t.timed, the context's ranker time (vsg_profile.rank_ms) covers the count pass and, per chunk, the emit pass, sort and
// cut.
int rank_lists(vsg_ctx * c, const RankTargets & t, const vsg_seqset * queries, int64_t q0, int64_t nq, int minwordmatches,
               int64_t tophits, std::vector<int64_t> & first, std::vector<uint32_t> & seqno, std::vector<uint32_t> & count)
{
  if (tophits < 1) { Error::set("vsg_rank: tophits must be at least 1"); return VSG_EINVAL; }
  std::vector<int32_t> n;
  int rc = rank_counts(c, t, queries, q0, nq, minwordmatches, n);
  if (rc != VSG_OK) { return rc; }
  first.assign(static_cast<size_t>(nq) + 1, 0);
  seqno.clear(); count.clear();
  if (nq == 0) { return VSG_OK; }
  int const th = static_cast<int>(std::min<int64_t>(tophits, INT32_MAX));
  for (int64_t i = 0; i < nq; i++) { first[static_cast<size_t>(i) + 1] = first[static_cast<size_t>(i)] + std::min<int64_t>(n[static_cast<size_t>(i)], tophits); }
  seqno.resize(static_cast<size_t>(first[static_cast<size_t>(nq)]));
  count.resize(seqno.size());
  // 2. chunks of consecutive queries whose keys fit the budget (one query at least)
  int64_t const budget = std::min<int64_t>(static_cast<int64_t>(c->dir_budget / 4 / 24), INT32_MAX / 2);
  std::vector<int64_t> koff, ooff;
  for (int64_t a = 0; a < nq;) {
    int64_t b = a, keys = 0;
    while (b < nq && (b == a || keys + n[static_cast<size_t>(b)] <= budget)) { keys += n[static_cast<size_t>(b)]; b++; }
    int64_t const m = b - a;
    koff.assign(static_cast<size_t>(m) + 1, 0); ooff.assign(static_cast<size_t>(m) + 1, 0);
    for (int64_t i = 0; i < m; i++) {
      koff[static_cast<size_t>(i) + 1] = koff[static_cast<size_t>(i)] + n[static_cast<size_t>(a + i)];
      ooff[static_cast<size_t>(i) + 1] = first[static_cast<size_t>(a + i) + 1] - first[static_cast<size_t>(a)];
    }
    int64_t const nout = ooff[static_cast<size_t>(m)];
    if (keys > 0) {
      size_t const offs_b = sizeof(int64_t) * 2 * (static_cast<size_t>(m) + 1);
      size_t const keys_b = sizeof(uint64_t) * static_cast<size_t>(keys);
      if ((rc = c->rank_tmp.reserve(offs_b + 2 * keys_b + sizeof(uint32_t) * (2 * static_cast<size_t>(nout) + static_cast<size_t>(m) + 4) + 64)) != VSG_OK) { return rc; }
      int64_t * const d_koff = static_cast<int64_t *>(c->rank_tmp.p);
      int64_t * const d_ooff = d_koff + m + 1;
      uint64_t * const d_k0 = reinterpret_cast<uint64_t *>(d_ooff + m + 1);
      uint64_t * const d_k1 = d_k0 + keys;
      uint32_t * const d_seq = reinterpret_cast<uint32_t *>(d_k1 + keys);
      uint32_t * const d_cnt = d_seq + nout;
      int32_t * const d_n2 = reinterpret_cast<int32_t *>(d_cnt + nout);   // the emit pass's counts (not read back)
      VSG_CUDA_OK(cudaMemcpyAsync(d_koff, koff.data(), sizeof(int64_t) * (static_cast<size_t>(m) + 1), cudaMemcpyHostToDevice, c->stream));
      VSG_CUDA_OK(cudaMemcpyAsync(d_ooff, ooff.data(), sizeof(int64_t) * (static_cast<size_t>(m) + 1), cudaMemcpyHostToDevice, c->stream));
      RankTop const emit{nullptr, nullptr, d_n2, d_n2 + m};
      if ((rc = rank_launch<RANK_EMIT>(c, t, queries, q0 + a, m, minwordmatches, th, emit, d_koff, d_k0)) != VSG_OK) { return rc; }
      cub::DoubleBuffer<uint64_t> db(d_k0, d_k1);
      size_t tb = 0;
      cub::DeviceSegmentedSort::SortKeysDescending(nullptr, tb, db, static_cast<int>(keys), static_cast<int>(m), d_koff, d_koff + 1, c->stream);
      if ((rc = c->cub_tmp.reserve(tb + 64)) != VSG_OK) { return rc; }
      cub::DeviceSegmentedSort::SortKeysDescending(c->cub_tmp.p, tb, db, static_cast<int>(keys), static_cast<int>(m), d_koff, d_koff + 1, c->stream);
      count_launch();
      if (nout > 0) {
        cut_lists_kernel<<<static_cast<unsigned>(m), 256, 0, c->stream>>>(db.Current(), d_koff, d_ooff, d_seq, d_cnt);
        count_launch();
        if (t.timed) { VSG_CUDA_OK(cudaEventRecord(c->ev[5], c->stream)); }   // the chunk's ranker time runs from its emit pass to here
        size_t const o = static_cast<size_t>(first[static_cast<size_t>(a)]);
        VSG_CUDA_OK(cudaMemcpyAsync(seqno.data() + o, d_seq, sizeof(uint32_t) * static_cast<size_t>(nout), cudaMemcpyDeviceToHost, c->stream));
        VSG_CUDA_OK(cudaMemcpyAsync(count.data() + o, d_cnt, sizeof(uint32_t) * static_cast<size_t>(nout), cudaMemcpyDeviceToHost, c->stream));
      }
      VSG_CUDA_OK(cudaStreamSynchronize(c->stream));
      VSG_CUDA_OK(cudaGetLastError());
      rank_collect_time(c);
    }
    a = b;
  }
  return VSG_OK;
}

}  // namespace vsg

extern "C" int vsg_rank(vsg_ctx * c, const vsg_index * ix, const vsg_seqset * queries, int64_t q0, int64_t nq,
                        int minwordmatches, int tophits, int mask_lower, uint32_t * cand_seqno,
                        uint32_t * cand_count, int32_t * ncand)
{
  if (c == nullptr || ix == nullptr || queries == nullptr || cand_seqno == nullptr || cand_count == nullptr || ncand == nullptr) {
    Error::set("vsg_rank: null argument");
    return VSG_EINVAL;
  }
  VSG_CUDA_OK(cudaSetDevice(c->device));
  if (tophits > TOPHITS_MAX) {
    std::vector<int64_t> first;
    std::vector<uint32_t> seqno, count;
    int const rc = rank_lists(c, index_targets(ix, mask_lower), queries, q0, nq, minwordmatches, tophits, first, seqno, count);
    if (rc != VSG_OK) { return rc; }
    for (int64_t i = 0; i < nq; i++) {
      size_t const a = static_cast<size_t>(first[static_cast<size_t>(i)]), n = static_cast<size_t>(first[static_cast<size_t>(i) + 1]) - a;
      std::memcpy(cand_seqno + static_cast<size_t>(i) * tophits, seqno.data() + a, sizeof(uint32_t) * n);
      std::memcpy(cand_count + static_cast<size_t>(i) * tophits, count.data() + a, sizeof(uint32_t) * n);
      ncand[i] = static_cast<int32_t>(n);
    }
    return VSG_OK;
  }
  RankTop r;
  int rc = rank_enqueue(c, ix, queries, q0, nq, minwordmatches, tophits, mask_lower, r);
  if (rc == VSG_OK) { rc = rank_download(c, r, nq, tophits, cand_seqno, cand_count, ncand, "vsg_rank"); }
  if (rc != VSG_OK) { return rc; }
  VSG_CUDA_OK(cudaGetLastError());
  return VSG_OK;
}

extern "C" int vsg_rank_occupancy(vsg_ctx * c, int * ctas_full, int * ctas_short)
{
  if (c == nullptr || ctas_full == nullptr || ctas_short == nullptr) { Error::set("vsg_rank_occupancy: null argument"); return VSG_EINVAL; }
  VSG_CUDA_OK(cudaSetDevice(c->device));
  auto const full = rank_kernel<RankFull, false, RANK_TOP>;
  auto const small = rank_kernel<RankShort, false, RANK_TOP>;
  VSG_CUDA_OK(cudaFuncSetAttribute(full, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(rank_smem<RankFull>())));
  VSG_CUDA_OK(cudaFuncSetAttribute(small, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(rank_smem<RankShort>())));
  VSG_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(ctas_full, full, RANK_THREADS, rank_smem<RankFull>()));
  VSG_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(ctas_short, small, RANK_THREADS, rank_smem<RankShort>()));
  return VSG_OK;
}


// ---------------------------------------------------------------------------------------------
// Incremental index of the cluster driver: replaces Dbindex::prepare + Dbindex::add_sequence
// (core/dbindex.cpp:121-148, 163-255) for a set of targets that GROWS (the centroids).  Targets get
// dense numbers in creation order; list km holds the numbers of the targets containing k-mer km, in
// creation order, inside a CSR whose per-list CAPACITY is the number of sequences of the whole set that
// contain km (every sequence could become a centroid) — counted once, as the reference's counting pass
// does for its bitmap/list sizing.  Shards of 32768 targets are contiguous ranges of every list; the
// list positions at a shard boundary are snapshotted when the boundary is crossed.
// ---------------------------------------------------------------------------------------------
namespace vsg {

__global__ void cindex_append_kernel(DevSeqs db, const uint32_t * __restrict__ seqnos, int n, uint32_t first_id, int k,
                                     int mask_lower, uint32_t * __restrict__ cursor, uint32_t * __restrict__ post32,
                                     int32_t * __restrict__ clen)
{
  extern __shared__ uint32_t bitmap[];
  int const ci = blockIdx.x;
  if (ci >= n) { return; }
  int const words = (1 << (2 * k)) >> 5;
  for (int i = threadIdx.x; i < (words > 0 ? words : 1); i += blockDim.x) { bitmap[i] = 0; }
  __syncthreads();
  int64_t const t = seqnos[ci];
  const uint8_t * __restrict__ s = db.sym + db.off[t];
  int const len = db.len[t];
  if (threadIdx.x == 0) { clen[first_id + ci] = len; }
  for (int p = k - 1 + threadIdx.x; p < len; p += blockDim.x) {
    uint32_t km;
    if (kmer_at(s, p, k, mask_lower, km)) {
      uint32_t const bit = 1u << (km & 31);
      uint32_t const old = atomicOr(&bitmap[km >> 5], bit);
      if ((old & bit) == 0) { post32[atomicAdd(&cursor[km], 1u)] = first_id + static_cast<uint32_t>(ci); }
    }
  }
}

struct CIndex {
  int device = 0, k = 8, mask_lower = 0;
  const vsg_seqset * set = nullptr;
  int64_t ncent = 0;                 // targets added so far
  DevBuf b_start, b_cursor, b_post, b_clen, b_shards, b_seqnos;
  std::vector<DevBuf> b_begin;       // list positions at the start of shard s >= 1
  std::vector<uint32_t> h_seqno;     // dense target number -> sequence number
};

int cindex_create(vsg_ctx * c, const vsg_seqset * set, int wordlength, int mask_lower, CIndex ** out)
{
  *out = nullptr;
  if (wordlength < 3 || wordlength > 10) { Error::set("cluster index: the device index supports --wordlength 3..10"); return VSG_EINVAL; }
  VSG_CUDA_OK(cudaSetDevice(c->device));
  CIndex * ix = new (std::nothrow) CIndex();
  if (ix == nullptr) { Error::set("out of host memory"); return VSG_ENOMEM; }
  ix->device = c->device; ix->k = wordlength; ix->mask_lower = mask_lower; ix->set = set;
  size_t const hashsize = static_cast<size_t>(1) << (2 * wordlength);
  size_t const bitmap_bytes = std::max<size_t>(hashsize / 8, 4);
  if (bitmap_bytes > 48 * 1024) {
    VSG_CUDA_OK(cudaFuncSetAttribute(index_build_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bitmap_bytes)));
    VSG_CUDA_OK(cudaFuncSetAttribute(cindex_append_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bitmap_bytes)));
  }
  int rc;
  DevBuf cnt, tmp;
  if ((rc = cnt.reserve(sizeof(uint32_t) * (hashsize + 1))) != VSG_OK ||
      (rc = ix->b_start.reserve(sizeof(uint32_t) * (hashsize + 1))) != VSG_OK ||
      (rc = ix->b_cursor.reserve(sizeof(uint32_t) * (hashsize + 1))) != VSG_OK ||
      (rc = ix->b_clen.reserve(sizeof(int32_t) * (static_cast<size_t>(set->d.n) + 1))) != VSG_OK) { delete ix; return rc; }
  // capacity of every list = the number of sequences of the whole set that contain the k-mer
  VSG_CUDA_OK(cudaMemsetAsync(cnt.p, 0, sizeof(uint32_t) * (hashsize + 1), c->stream));
  int64_t const n = set->d.n;
  for (int64_t t0 = 0; t0 < n; t0 += 1 << 20) {
    int const nt = static_cast<int>(std::min<int64_t>(1 << 20, n - t0));
    index_build_kernel<false><<<nt, 128, bitmap_bytes, c->stream>>>(set->d, static_cast<int>(t0), nt, wordlength, mask_lower, 0,
                                                                    static_cast<uint32_t *>(cnt.p), nullptr, nullptr);
    count_launch();
  }
  size_t tb = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tb, static_cast<uint32_t *>(cnt.p), static_cast<uint32_t *>(ix->b_start.p), static_cast<int>(hashsize + 1), c->stream);
  if ((rc = tmp.reserve(tb + 16)) != VSG_OK) { delete ix; return rc; }
  cub::DeviceScan::ExclusiveSum(tmp.p, tb, static_cast<uint32_t *>(cnt.p), static_cast<uint32_t *>(ix->b_start.p), static_cast<int>(hashsize + 1), c->stream);
  count_launch();
  // 64-bit check of the total: offsets are 32-bit
  {
    std::vector<uint32_t> h(hashsize);
    VSG_CUDA_OK(cudaMemcpyAsync(h.data(), cnt.p, sizeof(uint32_t) * hashsize, cudaMemcpyDeviceToHost, c->stream));
    VSG_CUDA_OK(cudaStreamSynchronize(c->stream));
    uint64_t total = 0;
    for (uint32_t v : h) { total += v; }
    if (total > 0xfffffff0ull) { cnt.release(); tmp.release(); delete ix; Error::set("cluster index: more than 2^32 k-mer occurrences in the sequence set"); return VSG_EINVAL; }
    if ((rc = ix->b_post.reserve(sizeof(uint32_t) * (total + 64))) != VSG_OK) { cnt.release(); tmp.release(); delete ix; return rc; }
  }
  VSG_CUDA_OK(cudaMemcpyAsync(ix->b_cursor.p, ix->b_start.p, sizeof(uint32_t) * (hashsize + 1), cudaMemcpyDeviceToDevice, c->stream));
  VSG_CUDA_OK(cudaStreamSynchronize(c->stream));
  cnt.release(); tmp.release();
  *out = ix;
  return VSG_OK;
}

void cindex_destroy(CIndex * ix)
{
  if (ix == nullptr) { return; }
  cudaSetDevice(ix->device);
  for (DevBuf * b : {&ix->b_start, &ix->b_cursor, &ix->b_post, &ix->b_clen, &ix->b_shards, &ix->b_seqnos}) { b->release(); }
  for (auto & b : ix->b_begin) { b.release(); }
  delete ix;
}

// Dbindex::add_sequence for a batch of new targets (ascending sequence numbers); enqueued on c->stream
int cindex_append(vsg_ctx * c, CIndex * ix, const uint32_t * seqnos, int n)
{
  if (n <= 0) { return VSG_OK; }
  size_t const hashsize = static_cast<size_t>(1) << (2 * ix->k);
  size_t const bitmap_bytes = std::max<size_t>(hashsize / 8, 4);
  int rc;
  int done = 0;
  while (done < n) {
    // never across a shard boundary in one launch: a shard's part of every list must be contiguous
    int64_t const room = SHARD - (ix->ncent % SHARD);
    int const m = static_cast<int>(std::min<int64_t>(n - done, room));
    if (sizeof(uint32_t) * static_cast<size_t>(m) + 16 > ix->b_seqnos.cap) {
      VSG_CUDA_OK(cudaStreamSynchronize(c->stream));   // the buffer is about to be replaced: let earlier launches finish with it
      if ((rc = ix->b_seqnos.reserve(sizeof(uint32_t) * static_cast<size_t>(std::max(m, 4096)) + 16)) != VSG_OK) { return rc; }
    }
    // the upload below reuses one small buffer: order it after the previous launch on the same stream
    VSG_CUDA_OK(cudaMemcpyAsync(ix->b_seqnos.p, seqnos + done, sizeof(uint32_t) * static_cast<size_t>(m), cudaMemcpyHostToDevice, c->stream));
    cindex_append_kernel<<<m, 128, bitmap_bytes, c->stream>>>(ix->set->d, static_cast<const uint32_t *>(ix->b_seqnos.p), m,
                                                              static_cast<uint32_t>(ix->ncent), ix->k, ix->mask_lower,
                                                              static_cast<uint32_t *>(ix->b_cursor.p), static_cast<uint32_t *>(ix->b_post.p),
                                                              static_cast<int32_t *>(ix->b_clen.p));
    count_launch();   // (the copy above is from pageable memory: staged before cudaMemcpyAsync returns)
    for (int i = 0; i < m; i++) { ix->h_seqno.push_back(seqnos[done + i]); }
    ix->ncent += m;
    done += m;
    if (ix->ncent % SHARD == 0) {
      ix->b_begin.emplace_back();
      if ((rc = ix->b_begin.back().reserve(sizeof(uint32_t) * (hashsize + 1))) != VSG_OK) { return rc; }
      VSG_CUDA_OK(cudaMemcpyAsync(ix->b_begin.back().p, ix->b_cursor.p, sizeof(uint32_t) * (hashsize + 1), cudaMemcpyDeviceToDevice, c->stream));
    }
  }
  return VSG_OK;
}

const std::vector<uint32_t> & cindex_seqnos(const CIndex * ix) { return ix->h_seqno; }

// The ranker's view of the targets added so far: their shard table, uploaded to ix->b_shards, and their lengths by
// dense number.  Not timed.  t.nshards == 0 (nothing uploaded) while nothing is indexed.
static int cindex_targets(vsg_ctx * c, CIndex * ix, RankTargets & t)
{
  int const nshards = static_cast<int>((ix->ncent + SHARD - 1) / SHARD);
  t.shards = nullptr; t.nshards = nshards;
  t.lens = DevSeqs{nullptr, nullptr, static_cast<const int32_t *>(ix->b_clen.p), ix->ncent};
  t.k = ix->k; t.mask_lower = ix->mask_lower; t.device = ix->device;
  t.incr = true; t.timed = false;
  if (nshards == 0) { return VSG_OK; }
  std::vector<ShardDev> sh(static_cast<size_t>(nshards));
  for (int s = 0; s < nshards; s++) {
    ShardDev & sd = sh[static_cast<size_t>(s)];
    sd.start = static_cast<const uint32_t *>(s == 0 ? ix->b_start.p : ix->b_begin[static_cast<size_t>(s) - 1].p);
    sd.end = static_cast<const uint32_t *>(s + 1 < nshards || ix->ncent % SHARD == 0 ? ix->b_begin[static_cast<size_t>(s)].p : ix->b_cursor.p);
    sd.post = nullptr; sd.post32 = static_cast<const uint32_t *>(ix->b_post.p);
    sd.rkeys = nullptr; sd.nr = 0; sd.reserved = 0;
    sd.t0 = s * SHARD;
    sd.nt = static_cast<int32_t>(std::min<int64_t>(SHARD, ix->ncent - static_cast<int64_t>(s) * SHARD));
  }
  int rc;
  if ((rc = ix->b_shards.reserve(sizeof(ShardDev) * sh.size())) != VSG_OK) { return rc; }
  // pageable source: staged before the call returns, so `sh` may go out of scope
  VSG_CUDA_OK(cudaMemcpyAsync(ix->b_shards.p, sh.data(), sizeof(ShardDev) * sh.size(), cudaMemcpyHostToDevice, c->stream));
  t.shards = static_cast<const ShardDev *>(ix->b_shards.p);
  return VSG_OK;
}

// search_topscores of queries [q0, q0+nq) of `queries` against the targets added so far; results as rank_enqueue's,
// candidate numbers are DENSE target numbers (CIndex::h_seqno maps them back).  Not timed.
int cindex_rank_enqueue(vsg_ctx * c, CIndex * ix, const vsg_seqset * queries, int64_t q0, int64_t nq, int minwordmatches,
                        int tophits, RankTop & out)
{
  if (tophits < 1 || tophits > TOPHITS_MAX) { Error::set("cluster ranker: tophits must be in 1..1024"); return VSG_EINVAL; }
  int rc;
  if ((rc = rank_top_alloc(c, nq, tophits, out)) != VSG_OK || nq == 0) { return rc; }
  RankTargets t;
  if ((rc = cindex_targets(c, ix, t)) != VSG_OK) { return rc; }
  if (t.nshards == 0) {   // nothing indexed yet: no candidates
    VSG_CUDA_OK(cudaMemsetAsync(out.n, 0, sizeof(int32_t) * nq, c->stream));
    return VSG_OK;
  }
  return rank_launch<RANK_TOP>(c, t, queries, q0, nq, minwordmatches, tophits, out, nullptr, nullptr);
}

// rank_lists of queries [q0, q0+nq) of `queries` against the targets added so far (any tophits); candidate numbers are
// DENSE target numbers.  Not timed.
int cindex_rank_lists(vsg_ctx * c, CIndex * ix, const vsg_seqset * queries, int64_t q0, int64_t nq, int minwordmatches,
                      int64_t tophits, std::vector<int64_t> & first, std::vector<uint32_t> & seqno, std::vector<uint32_t> & count)
{
  RankTargets t;
  int const rc = cindex_targets(c, ix, t);
  if (rc != VSG_OK) { return rc; }
  if (t.nshards == 0) {   // nothing indexed yet: no candidates
    first.assign(static_cast<size_t>(nq) + 1, 0);
    seqno.clear(); count.clear();
    return VSG_OK;
  }
  return rank_lists(c, t, queries, q0, nq, minwordmatches, tophits, first, seqno, count);
}

}  // namespace vsg

// ---- the cluster driver's incremental index on its own (include/vsg.h), so its candidate lists can be compared with a
//      plain index of the same targets ----
struct vsg_cluster_index {
  vsg::CIndex * ix = nullptr;
  int64_t nseq = 0;        // sequences in the set
  int64_t last = -1;       // the last sequence number appended
};

extern "C" int vsg_cluster_index_create(vsg_ctx * c, const vsg_seqset * set, int wordlength, int mask_lower, vsg_cluster_index ** out)
{
  if (c == nullptr || set == nullptr || out == nullptr) { Error::set("vsg_cluster_index_create: null argument"); return VSG_EINVAL; }
  *out = nullptr;
  if (set->device != c->device) { Error::set("vsg_cluster_index_create: sequence set lives on another device than the context"); return VSG_EINVAL; }
  vsg_cluster_index * h = new (std::nothrow) vsg_cluster_index();
  if (h == nullptr) { Error::set("out of host memory"); return VSG_ENOMEM; }
  int const rc = cindex_create(c, set, wordlength, mask_lower, &h->ix);
  if (rc != VSG_OK) { delete h; return rc; }
  h->nseq = set->d.n;
  *out = h;
  return VSG_OK;
}

extern "C" int vsg_cluster_index_append(vsg_ctx * c, vsg_cluster_index * h, const uint32_t * seqnos, int64_t n)
{
  if (c == nullptr || h == nullptr || (n > 0 && seqnos == nullptr)) { Error::set("vsg_cluster_index_append: null argument"); return VSG_EINVAL; }
  if (n < 0 || n > INT32_MAX) { Error::set("vsg_cluster_index_append: count out of range"); return VSG_EINVAL; }
  if (h->ix->device != c->device) { Error::set("vsg_cluster_index_append: index lives on another device than the context"); return VSG_EINVAL; }
  // cindex_append takes new targets in ascending sequence order, each once, after every earlier one
  int64_t prev = h->last;
  for (int64_t i = 0; i < n; i++) {
    int64_t const s = seqnos[i];
    if (s <= prev || s >= h->nseq) {
      Error::set("vsg_cluster_index_append: sequence numbers must be strictly ascending, after the last one appended and inside the set");
      return VSG_EINVAL;
    }
    prev = s;
  }
  VSG_CUDA_OK(cudaSetDevice(c->device));
  int const rc = cindex_append(c, h->ix, seqnos, static_cast<int>(n));
  if (rc != VSG_OK) { return rc; }
  VSG_CUDA_OK(cudaGetLastError());
  h->last = prev;
  return VSG_OK;
}

extern "C" int64_t vsg_cluster_index_count(const vsg_cluster_index * h)
{
  return h == nullptr ? 0 : static_cast<int64_t>(cindex_seqnos(h->ix).size());
}

extern "C" int vsg_cluster_index_rank(vsg_ctx * c, vsg_cluster_index * h, const vsg_seqset * queries, int64_t q0, int64_t nq,
                                      int minwordmatches, int tophits, uint32_t * cand, uint32_t * count, int32_t * ncand)
{
  if (c == nullptr || h == nullptr || queries == nullptr || (nq > 0 && (cand == nullptr || count == nullptr || ncand == nullptr))) {
    Error::set("vsg_cluster_index_rank: null argument");
    return VSG_EINVAL;
  }
  if (tophits < 1) { Error::set("vsg_cluster_index_rank: tophits must be at least 1"); return VSG_EINVAL; }
  if (q0 < 0 || nq < 0 || q0 + nq > queries->d.n) { Error::set("vsg_cluster_index_rank: query range out of bounds"); return VSG_EINVAL; }
  if (queries->device != c->device || h->ix->device != c->device) {
    Error::set("vsg_cluster_index_rank: sequence set / index lives on another device than the context");
    return VSG_EINVAL;
  }
  if (nq > (1 << 30) / tophits) { Error::set("vsg_cluster_index_rank: batch too large"); return VSG_EINVAL; }
  VSG_CUDA_OK(cudaSetDevice(c->device));
  int rc;
  if (tophits > TOPHITS_MAX) {
    std::vector<int64_t> first;
    std::vector<uint32_t> seqno, cnt;
    if ((rc = cindex_rank_lists(c, h->ix, queries, q0, nq, minwordmatches, tophits, first, seqno, cnt)) != VSG_OK) { return rc; }
    for (int64_t i = 0; i < nq; i++) {
      size_t const a = static_cast<size_t>(first[static_cast<size_t>(i)]), n = static_cast<size_t>(first[static_cast<size_t>(i) + 1]) - a;
      std::memcpy(cand + static_cast<size_t>(i) * tophits, seqno.data() + a, sizeof(uint32_t) * n);
      std::memcpy(count + static_cast<size_t>(i) * tophits, cnt.data() + a, sizeof(uint32_t) * n);
      ncand[i] = static_cast<int32_t>(n);
    }
    return VSG_OK;
  }
  RankTop r;
  if ((rc = cindex_rank_enqueue(c, h->ix, queries, q0, nq, minwordmatches, tophits, r)) != VSG_OK ||
      (rc = rank_download(c, r, nq, tophits, cand, count, ncand, "vsg_cluster_index_rank")) != VSG_OK) { return rc; }
  VSG_CUDA_OK(cudaGetLastError());
  return VSG_OK;
}

extern "C" void vsg_cluster_index_destroy(vsg_cluster_index * h)
{
  if (h == nullptr) { return; }
  cindex_destroy(h->ix);
  delete h;
}
