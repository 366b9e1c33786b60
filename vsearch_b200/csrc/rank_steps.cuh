// rank_steps.cuh — the device steps of the k-mer ranker that rank.cu and sintax.cu both run: the static index's
// shard layout, symbol and k-mer helpers, the per-target sort key, block scans, and the posting-list walk that turns a
// set of query k-mers into shared-memory counters of one shard (see rank.cu for the index and the ranker).
#pragma once

#include "vsg_internal.h"

namespace vsg {

constexpr int SHARD_BITS = 15;
constexpr int SHARD = 1 << SHARD_BITS;  // targets per shard
constexpr int RANK_THREADS = 512;
constexpr int KMER_CAP = 2048;          // distinct-k-mer capacity per query (query length <= 2047 + k)

constexpr int COUNTER_WORDS = SHARD / 2 + 1;
// Static index: a shard holds 32766 targets and its postings are stored as the BYTE OFFSET of the target's counter
// word (two 16-bit counters per word: offset = (local target & ~1) * 2 <= 65528); every k-mer has two sub-lists,
// the even and the odd targets, each padded to a multiple of 8 entries with offset 65532 = word 16383, which no
// target owns.  Turning a posting into its counter update then takes no arithmetic at all: the address is the
// posting, the increment (1 or 0x10000) is a constant of the sub-list.
constexpr int SHARD_STATIC = SHARD - 2;
constexpr uint16_t POST_PAD = 65532;

struct ShardDev {
  const uint32_t * start;  // 4^k + 1 list offsets (incremental index: where this shard's part of every list begins)
  const uint16_t * post;   // shard-local target numbers (static index)
  int32_t t0;              // first target of the shard
  int32_t nt;              // targets in the shard
  // incremental index (cluster driver): lists of 32-bit target numbers in creation order, this shard's part of
  // list km is post32[start[km] .. end[km])
  const uint32_t * end;
  const uint32_t * post32;
  // sparse static index (--wordlength 11..15): the sorted (k-mer << 1 | target parity) keys of the sub-lists that
  // exist in this shard; sub-list i is post[start[i] .. start[i + 1]).  nr == 0: dense (start indexed by 2 * k-mer)
  const uint32_t * rkeys;
  uint32_t nr;
  uint32_t reserved;
};

__device__ __forceinline__ bool sym_bad(int s, int mask_lower)
{
  int const c = s & 15;
  bool const single = (c == 1) | (c == 2) | (c == 4) | (c == 8);
  return !single || (mask_lower && (s & 16));
}
__device__ __forceinline__ uint32_t sym_2bit(int s)
{
  int const c = s & 15;
  return (c == 2) ? 1u : (c == 4) ? 2u : (c == 8) ? 3u : 0u;
}

// k-mer ending at position p (p >= k-1); returns false when the window holds a masked symbol
__device__ __forceinline__ bool kmer_at(const uint8_t * __restrict__ s, int p, int k, int mask_lower,
                                        uint32_t & out)
{
  uint32_t v = 0;
  bool bad = false;
  for (int j = p - k + 1; j <= p; j++) {
    int const c = s[j];
    bad |= sym_bad(c, mask_lower);
    v = (v << 2) | sym_2bit(c);
  }
  out = v;
  return !bad;
}

// inclusive prefix sum of v over the lanes of the (whole) warp
template <typename T>
__device__ __forceinline__ T warp_inclusive_sum(T v)
{
  int const lane = threadIdx.x & 31;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { T const o = __shfl_up_sync(0xffffffffu, v, d); if (lane >= d) { v += o; } }
  return v;
}

// key: larger = better.  count (15 bits) | ~length (25 bits) | ~seqno (24 bits)
__device__ __forceinline__ uint64_t make_key(uint32_t count, uint32_t len, uint32_t seqno)
{
  uint32_t const l = len > 0x1ffffffu ? 0x1ffffffu : len;
  if (count > 32767u) { count = 32767u; }  // the reference saturates its counters (searchcore.cpp:306-315)
  return (static_cast<uint64_t>(count) << 49) | (static_cast<uint64_t>(0x1ffffffu - l) << 24) |
         static_cast<uint64_t>(0xffffffu - seqno);
}
// the key of local target lt of shard S with k-mer count `count`
__device__ __forceinline__ uint64_t target_key(const DevSeqs & db, const ShardDev & S, uint32_t count, int lt)
{
  int const t = S.t0 + lt;
  return make_key(count, static_cast<uint32_t>(db.len[t]), static_cast<uint32_t>(t));
}
// the smallest key with k-mer count `count`
__device__ __forceinline__ uint64_t count_key(int count) { return static_cast<uint64_t>(static_cast<uint32_t>(count)) << 49; }

// Exclusive prefix sum of x over the block, and the block's total.  s_wsum holds one word per warp; the caller's next
// barrier must come before the next call writes it again.
template <typename T>
__device__ __forceinline__ T block_exclusive_sum(T x, int * s_wsum, T & total)
{
  int const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T const incl = warp_inclusive_sum(x);
  if (lane == 31) { s_wsum[warp] = static_cast<int>(incl); }
  __syncthreads();
  T wbase = 0;
  total = 0;
#pragma unroll
  for (int w = 0; w < RANK_THREADS / 32; w++) { T const v = static_cast<T>(s_wsum[w]); if (w < warp) { wbase += v; } total += v; }
  return wbase + incl - x;
}

// 2. The posting lists of kmers[0, n) in shard S: lbeg[i] = where k-mer i's list begins; llen[i] = its length
//    (incremental index), or the lengths of its even and its odd sub-list in vectors of 8, one per 16-bit half
//    (static index).  Invalid k-mers get empty lists.
template <bool INCR>
__device__ __forceinline__ void list_bounds(const ShardDev & S, const uint32_t * kmers, int n, uint32_t * lbeg, uint32_t * llen)
{
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    uint32_t const km = kmers[i];
    uint32_t b = 0, len = 0;
    if (km != 0xffffffffu) {
      if (INCR) { b = S.start[km]; len = S.end[km] - b; }
      else if (S.nr == 0u) {
        // even sub-list [b, mid), odd sub-list [mid, end)
        b = S.start[2 * km];
        uint32_t const mid = S.start[2 * km + 1], e = S.start[2 * km + 2];
        len = ((mid - b) >> 3) | (((e - mid) >> 3) << 16);
      } else {
        // sparse shard: lower bound of the even sub-list's key among the sub-lists that exist; the odd one, if
        // present, is its neighbour, so the pair is one contiguous run of postings either way
        uint32_t const want = km << 1;
        uint32_t lo = 0, hi = S.nr;
        while (lo < hi) {
          uint32_t const mid = (lo + hi) >> 1;
          if (__ldg(S.rkeys + mid) < want) { lo = mid + 1; } else { hi = mid; }
        }
        b = S.start[lo];
        uint32_t na = 0, nb = 0, j = lo;
        if (j < S.nr && __ldg(S.rkeys + j) == want) { na = (S.start[j + 1] - S.start[j]) >> 3; j++; }
        if (j < S.nr && __ldg(S.rkeys + j) == (want | 1u)) { nb = (S.start[j + 1] - S.start[j]) >> 3; }
        len = na | (nb << 16);
      }
    }
    lbeg[i] = b; llen[i] = len;
  }
}

// 3. Postings -> counters, static index: the FLAT VECTOR STREAM.  Lists are 16-byte aligned and padded, so a lane
//    pulls 8 targets per 128-bit load; padding entries land in counter word 16383, which no target of a static shard
//    owns.  The even and the odd sub-list of a k-mer are one contiguous run of 16-byte vectors, and the runs of all
//    the query's k-mers, laid end to end, form one virtual stream of Vtot vectors.  Each warp takes a contiguous 1/16
//    of the stream and walks it 32 vectors per round — every lane always has a vector (a per-k-mer loop leaves most
//    lanes idle on the second trip of a 36-vector sub-list and pays its set-up 243 times per shard).  Per run i, with
//    c_i its position in the stream:
//      cum[i]  = c_i + n_i          where the run ends
//      lbeg[i] = first vector - c_i  so that stream position + lbeg = the vector's index in the shard's postings
//      llen[i] = c_i + na_i         positions below it hold even targets (increment 1), the rest odd ones (0x10000)
//    A lane finds its first run by one binary search and then walks forward (runs average two rounds).
//    KCAP: the capacity of the run arrays (n <= KCAP); llen and cum must lie KCAP and 2 * KCAP words behind lbeg: the
//    walk addresses them from lbeg.
template <int KCAP = KMER_CAP>
__device__ __forceinline__ void postings_stream(const ShardDev & S, int n, uint32_t * lbeg, uint32_t * llen, uint32_t * cum,
                                                uint32_t * counters, int * s_wsum)
{
  constexpr int NWARPS = RANK_THREADS / 32;
  int const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t Vtot;
  {
    // 3a. exclusive prefix sum of the run lengths (in vectors)
    int const per = (n + RANK_THREADS - 1) / RANK_THREADS;   // <= KCAP / RANK_THREADS
    int const i0 = threadIdx.x * per;
    uint32_t nn[KCAP / RANK_THREADS], bb[KCAP / RANK_THREADS];
    uint32_t sum = 0;
#pragma unroll
    for (int u = 0; u < KCAP / RANK_THREADS; u++) {
      bool const in = u < per && i0 + u < n;
      nn[u] = in ? llen[i0 + u] : 0u;
      bb[u] = in ? lbeg[i0 + u] : 0u;
      sum += (nn[u] & 0xffffu) + (nn[u] >> 16);
    }
    uint32_t c0 = block_exclusive_sum(sum, s_wsum, Vtot);
#pragma unroll
    for (int u = 0; u < KCAP / RANK_THREADS; u++) {
      if (u < per && i0 + u < n) {
        uint32_t const na = nn[u] & 0xffffu, nv = na + (nn[u] >> 16);
        lbeg[i0 + u] = (bb[u] >> 3) - c0;
        llen[i0 + u] = c0 + na;
        cum[i0 + u] = c0 + nv;
        c0 += nv;
      }
    }
    __syncthreads();
  }
  uint32_t const per_w = ((Vtot + NWARPS * 32 - 1) / (NWARPS * 32)) * 32;
  uint32_t const wbeg = static_cast<uint32_t>(warp) * per_w;
  uint32_t const wend = min(Vtot, wbeg + per_w);
  if (wbeg < wend) {
    constexpr int U = 4;   // vectors (of 8 postings) held per lane
    const uint4 * __restrict__ pbase = reinterpret_cast<const uint4 *>(S.post);
    uint32_t const cnt_sa = static_cast<uint32_t>(__cvta_generic_to_shared(counters));
    // the run holding this lane's first vector: the first whose end lies beyond it
    uint32_t const v_first = min(wbeg + static_cast<uint32_t>(lane), wend - 1);
    int lo = 0, hi = n - 1;
    while (lo < hi) {
      int const mid = (lo + hi) >> 1;
      if (cum[mid] <= v_first) { lo = mid + 1; } else { hi = mid; }
    }
    // sa walks the run arrays as a shared-memory byte address of lbeg[s]; llen and cum lie KCAP words further each
    uint32_t sa = static_cast<uint32_t>(__cvta_generic_to_shared(lbeg + lo));
    uint32_t ce = cum[lo];
    // U loads per lane are issued back to back, then turned into counter updates; the other 31 warps of the SM
    // cover the wait
    uint4 cur[U];
    uint32_t inc[U];
    auto fetch = [&](int u, uint32_t vv) {
      inc[u] = 0u;
      if (vv < wend) {
        while (vv >= ce) {
          sa += 4u;
          asm("ld.shared.u32 %0, [%1+%2];" : "=r"(ce) : "r"(sa), "n"(2 * KCAP * 4));
        }
        uint32_t vb, sp;
        asm("ld.shared.u32 %0, [%1];" : "=r"(vb) : "r"(sa));
        asm("ld.shared.u32 %0, [%1+%2];" : "=r"(sp) : "r"(sa), "n"(KCAP * 4));
        cur[u] = __ldg(pbase + static_cast<uint32_t>(vb + vv));
        inc[u] = vv < sp ? 1u : 0x10000u;
      }
    };
    auto apply = [&](int u) {
      if (inc[u] != 0u) {
        uint32_t const w[4] = {cur[u].x, cur[u].y, cur[u].z, cur[u].w};
#pragma unroll
        for (int k2 = 0; k2 < 4; k2++) {
          // the postings ARE the byte offsets of their counter words
          asm volatile("red.shared.add.u32 [%0], %1;" :: "r"(cnt_sa + (w[k2] & 0xffffu)), "r"(inc[u]));
          asm volatile("red.shared.add.u32 [%0], %1;" :: "r"(cnt_sa + (w[k2] >> 16)), "r"(inc[u]));
        }
      }
    };
    for (uint32_t v0 = wbeg; v0 < wend; v0 += 32u * U) {
#pragma unroll
      for (int u = 0; u < U; u++) { fetch(u, v0 + 32u * u + static_cast<uint32_t>(lane)); }
#pragma unroll
      for (int u = 0; u < U; u++) { apply(u); }
    }
  }
}

// 4. Visits every counter >= thr in counter words [w0, w1) (w0 a multiple of W) of a shard of nt targets: f(count,
//    local target).  Thread i reads W words at a time, step w0 / W + i, + blockDim.x, ..., so two calls over the same
//    range visit each thread's counters in the same order.  W = 4 (one 16-byte load) for the scans of the running
//    threshold and the unbounded ranker; W = 1 for the fixed-threshold scans, whose appends keep more state live
//    (four words per thread there spill).  zero: the words are cleared behind the scan, and so is the word the padding
//    entries of the lists land in (the next shard then skips its clearing pass).  That word holds the counters of
//    targets 32766 and 32767 in an incremental shard of more than SHARD_STATIC targets: there the scan itself reads and
//    clears it, and clearing it up front would race with that read.
template <int W, typename F>
__device__ __forceinline__ void visit_counters(uint32_t * counters, int w0, int w1, int nt, uint32_t thr, bool zero, F && f)
{
  static_assert(W == 1 || W == 4, "counter words per load");
  int const v1 = (w1 + W - 1) / W;
  uint32_t const below = thr > 0 ? ((thr - 1) | ((thr - 1) << 16)) : 0u;
  if (zero && threadIdx.x == 0 && nt <= SHARD_STATIC) { counters[(POST_PAD >> 2)] = 0; }
  for (int vi = w0 / W + threadIdx.x; vi < v1; vi += blockDim.x) {
    uint32_t w[W];
    if constexpr (W == 4) {
      uint4 * __restrict__ cv = reinterpret_cast<uint4 *>(counters);
      uint4 const x = cv[vi];
      if (zero) { cv[vi] = make_uint4(0u, 0u, 0u, 0u); }
      w[0] = x.x; w[1] = x.y; w[2] = x.z; w[3] = x.w;
    } else {
      w[0] = counters[vi];
      if (zero) { counters[vi] = 0u; }
    }
#pragma unroll
    for (int u = 0; u < W; u++) {
      // some half above thr-1?  (thr == 0: everything passes)
      if (W == 4 && thr > 0 && __vmaxu2(w[u], below) == below) { continue; }
      uint32_t const c0 = w[u] & 0xffffu, c1 = w[u] >> 16;
      int const lt0 = 2 * (W * vi + u), lt1 = lt0 + 1;
      if (c0 >= thr && lt0 < nt) { f(c0, lt0); }
      if (c1 >= thr && lt1 < nt) { f(c1, lt1); }
    }
  }
}

}  // namespace vsg
