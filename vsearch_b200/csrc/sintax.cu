// sintax.cu — SINTAX taxonomy classification on the static k-mer index (sm_90a).
//
// Replaces, for whole batches of queries at once,
//   unique_count(..., Masking::none)  (reference core/unique.cpp:155-353)     distinct k-mers in first-occurrence order
//   the subsampling of sintax_query   (commands/sintax.cpp:405-478)           100 bootstraps of 32 draws per strand
//   sintax_search_topscores           (commands/sintax.cpp:299-402)           the best target of every bootstrap
//   sintax_analyse                    (commands/sintax.cpp:138-296)           the vote and the --tabbedout row (host)
//
// Per chunk of queries four kernels run:
//   1. sintax_kmers_kernel: one CTA per (query, strand) writes the strand's distinct k-mers in the order of their first
//      window.  Every window's k-mer goes into an open-addressing table that keeps the smallest window per k-mer
//      (shared memory up to KMER_CAP windows, this CTA's HBM scratch beyond); a second pass keeps the windows that are
//      their k-mer's first and compacts them in window order with block scans.
//   2. sintax_draw_kernel: one warp per query makes the draws of both strands.  The reference's generator is SplitMix64,
//      whose call i returns mix(state + i * gamma), so lane L evaluates call `calls + L + 1` and the warp makes 32 calls
//      per round; Lemire's bounded method rejects a call exactly when its low product word is below 2^64 mod c, which
//      depends on that call alone, so the draws are the accepted calls in call order.  A repeated index is dropped
//      (match_any), and the sampled k-mers go to HBM.
//   3. sintax_count_kernel: one CTA per (query, strand, index shard) loops over the bootstraps: the ranker's posting
//      stream (rank_steps.cuh) turns the sample's postings into shared-memory counters, the scan that clears them
//      behind keeps the best make_key(count, length, seqno) of the counts >= 2 (the key orders exactly as the tie rule
//      of sintax_search_topscores), and one 64-bit atomicMax per (query, strand, bootstrap) combines the shards.
//   4. sintax_finish_kernel: one warp per query compacts the winners in bootstrap order and picks the strand.
#include "vsg_internal.h"
#include "rank_steps.cuh"

#include <algorithm>
#include <cctype>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

namespace vsg {

namespace {

constexpr int BOOTS = VSG_SINTAX_BOOTSTRAPS;
constexpr int SUBSET = 32;                           // draws per bootstrap (sintax.cpp subset_size)
constexpr uint64_t GAMMA = 0x9E3779B97F4A7C15ull;     // SplitMix64's increment
constexpr int SMEM_SLOTS = 2 * KMER_CAP;             // first-occurrence table in shared memory (<= KMER_CAP windows)
constexpr int DRAW_WARPS = 8;

__host__ __device__ __forceinline__ uint64_t splitmix_mix(uint64_t z)
{
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

__device__ __forceinline__ uint32_t slot_of(uint32_t v, uint32_t hmask) { return (v * 2654435761u) >> 7 & hmask; }

// 1. item = query * nstrands + strand; its list goes to lists[list_off[item] ...], nlist[item] entries
__global__ void __launch_bounds__(RANK_THREADS)
sintax_kmers_kernel(DevSeqs plus, int64_t q0, DevSeqs minus, int nq, int nstrands, int k,
                    const int64_t * __restrict__ list_off, uint32_t * __restrict__ lists, int32_t * __restrict__ nlist,
                    uint32_t * __restrict__ scratch, int scratch_slots)
{
  __shared__ uint32_t s_key[SMEM_SLOTS], s_pos[SMEM_SLOTS];
  __shared__ int s_wsum[RANK_THREADS / 32];
  for (int item = blockIdx.x; item < nq * nstrands; item += gridDim.x) {
    int const qi = item / nstrands;
    bool const minus_strand = (item % nstrands) != 0;
    int64_t const q = minus_strand ? qi : q0 + qi;
    DevSeqs const & qs = minus_strand ? minus : plus;
    const uint8_t * __restrict__ s = qs.sym + qs.off[q];
    int const nwin = qs.len[q] - k + 1;
    int slots = SMEM_SLOTS;
    uint32_t * hk = s_key;
    uint32_t * hp = s_pos;
    if (nwin > KMER_CAP) {
      slots = scratch_slots;
      hk = scratch + static_cast<size_t>(blockIdx.x) * 2 * static_cast<size_t>(scratch_slots);
      hp = hk + scratch_slots;
    }
    uint32_t const hmask = static_cast<uint32_t>(slots) - 1u;
    for (int i = threadIdx.x; i < slots; i += blockDim.x) { hk[i] = 0xffffffffu; hp[i] = 0xffffffffu; }
    __syncthreads();
    // the smallest window of every k-mer
    for (int p = threadIdx.x; p < nwin; p += blockDim.x) {
      uint32_t v;
      if (kmer_at(s, p + k - 1, k, 0, v)) {
        uint32_t slot = slot_of(v, hmask);
        for (;;) {
          uint32_t const old = atomicCAS(&hk[slot], 0xffffffffu, v);
          if (old == 0xffffffffu || old == v) { atomicMin(&hp[slot], static_cast<uint32_t>(p)); break; }
          slot = (slot + 1u) & hmask;
        }
      }
    }
    __syncthreads();
    // the windows that hold their k-mer's first occurrence, in window order
    uint32_t * __restrict__ out = lists + list_off[item];
    int base = 0;
    for (int p0 = 0; p0 < nwin; p0 += RANK_THREADS) {
      int const p = p0 + static_cast<int>(threadIdx.x);
      uint32_t v = 0;
      int first = 0;
      if (p < nwin && kmer_at(s, p + k - 1, k, 0, v)) {
        uint32_t slot = slot_of(v, hmask);
        while (hk[slot] != v) { slot = (slot + 1u) & hmask; }
        first = hp[slot] == static_cast<uint32_t>(p) ? 1 : 0;
      }
      int total;
      int const pos = block_exclusive_sum(first, s_wsum, total);
      if (first != 0) { out[base + pos] = v; }
      base += total;
      __syncthreads();
    }
    if (threadIdx.x == 0) { nlist[item] = base; }
    __syncthreads();
  }
}

// 2. one warp per query: the sampled k-mers of bootstrap b of item i at samp[(i * BOOTS + b) * SUBSET ...],
//    nsamp[i * BOOTS + b] of them (0 for a strand with fewer than SUBSET distinct k-mers)
__global__ void __launch_bounds__(DRAW_WARPS * 32)
sintax_draw_kernel(int nq, int nstrands, uint64_t seed, int64_t qnum0, const int64_t * __restrict__ list_off,
                   const uint32_t * __restrict__ lists, const int32_t * __restrict__ nlist, uint32_t * __restrict__ samp,
                   uint8_t * __restrict__ nsamp)
{
  __shared__ uint32_t s_x[DRAW_WARPS][SUBSET];
  int const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int const qi = blockIdx.x * DRAW_WARPS + warp;
  if (qi >= nq) { return; }   // whole warps
  // random_substream_seed(seed, n) = the first output of SplitMix64(seed ^ n * gamma)
  uint64_t const state = splitmix_mix((seed ^ (static_cast<uint64_t>(qnum0 + qi) * GAMMA)) + GAMMA);
  uint64_t calls = 0;   // generator calls so far, both strands
  unsigned const below = (1u << lane) - 1u;
  for (int st = 0; st < nstrands; st++) {
    int const item = qi * nstrands + st;
    uint64_t const c = static_cast<uint64_t>(nlist[item]);
    if (c < SUBSET) {
      for (int b = lane; b < BOOTS; b += 32) { nsamp[static_cast<size_t>(item) * BOOTS + b] = 0; }
      continue;
    }
    uint64_t const reject_below = (0ull - c) % c;   // 2^64 mod c (random_bounded's threshold)
    const uint32_t * __restrict__ list = lists + list_off[item];
    for (int b = 0; b < BOOTS; b++) {
      int have = 0;
      while (have < SUBSET) {
        uint64_t const z = splitmix_mix(state + (calls + static_cast<uint64_t>(lane) + 1u) * GAMMA);
        bool const ok = z * c >= reject_below;
        unsigned const acc = __ballot_sync(0xffffffffu, ok);
        int const rank = __popc(acc & below);
        int const need = SUBSET - have;
        if (ok && rank < need) { s_x[warp][have + rank] = static_cast<uint32_t>(__umul64hi(z, c)); }
        unsigned const last = __ballot_sync(0xffffffffu, ok && rank == need - 1);
        calls += last != 0u ? static_cast<uint64_t>(__ffs(last)) : 32u;
        have += min(__popc(acc), need);
      }
      __syncwarp();
      uint32_t const x = s_x[warp][lane];
      unsigned const same = __match_any_sync(0xffffffffu, x);
      bool const keep = (__ffs(same) - 1) == lane;   // the first draw of this index
      unsigned const kept = __ballot_sync(0xffffffffu, keep);
      size_t const cell = static_cast<size_t>(item) * BOOTS + b;
      if (keep) { samp[cell * SUBSET + __popc(kept & below)] = list[x]; }
      if (lane == 0) { nsamp[cell] = static_cast<uint8_t>(__popc(kept)); }
      __syncwarp();
    }
  }
}

// 3. one CTA per (item, shard): keys[item * BOOTS + b] = the best key of bootstrap b over all shards (0: no target
//    holds two of the sampled k-mers)
constexpr size_t COUNT_SMEM = (COUNTER_WORDS + 3) * 4 + SUBSET * 4 + 3 * KMER_CAP * 4;   // 90 244 B: two CTAs per SM

__global__ void __launch_bounds__(RANK_THREADS, 2)
sintax_count_kernel(DevSeqs db, const ShardDev * __restrict__ shards, const int32_t * __restrict__ nlist,
                    const uint32_t * __restrict__ samp, const uint8_t * __restrict__ nsamp,
                    unsigned long long * __restrict__ keys)
{
  extern __shared__ __align__(16) unsigned char smem[];
  uint32_t * const counters = reinterpret_cast<uint32_t *>(smem);   // COUNTER_WORDS (+pad)
  uint32_t * const kmers = counters + COUNTER_WORDS + 3;            // SUBSET
  uint32_t * const lbeg = kmers + SUBSET;                           // postings_stream: lbeg, llen, cum KMER_CAP apart
  uint32_t * const llen = lbeg + KMER_CAP;
  uint32_t * const cum = llen + KMER_CAP;
  __shared__ unsigned long long s_best;
  __shared__ int s_wsum[RANK_THREADS / 32];
  int const item = blockIdx.x;
  if (nlist[item] < SUBSET) { return; }   // no bootstraps on this strand
  ShardDev const S = shards[blockIdx.y];
  int const nwords = (S.nt + 1) >> 1;
  for (int i = threadIdx.x; i < COUNTER_WORDS; i += blockDim.x) { counters[i] = 0; }   // later cleared by each scan
  for (int b = 0; b < BOOTS; b++) {
    size_t const cell = static_cast<size_t>(item) * BOOTS + b;
    int const n = nsamp[cell];
    if (static_cast<int>(threadIdx.x) < n) { kmers[threadIdx.x] = samp[cell * SUBSET + threadIdx.x]; }
    if (threadIdx.x == 0) { s_best = 0; }
    __syncthreads();
    list_bounds<false>(S, kmers, n, lbeg, llen);
    __syncthreads();
    postings_stream(S, n, lbeg, llen, cum, counters, s_wsum);
    __syncthreads();
    // the winner must hold at least two sampled k-mers (sintax.cpp:399)
    unsigned long long best = 0;
    visit_counters<4>(counters, 0, nwords, S.nt, 2u, true, [&](uint32_t cnt, int lt) {
      unsigned long long const key = target_key(db, S, cnt, lt);
      best = key > best ? key : best;
    });
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      unsigned long long const v = __shfl_xor_sync(0xffffffffu, best, o);
      best = v > best ? v : best;
    }
    if ((threadIdx.x & 31) == 0 && best != 0) { atomicMax(&s_best, best); }
    __syncthreads();
    if (threadIdx.x == 0 && s_best != 0) { atomicMax(keys + cell, s_best); }
  }
}

// 4. one warp per query: winners in bootstrap order, per-strand counts, the strand (sintax.cpp:480-507)
__global__ void __launch_bounds__(DRAW_WARPS * 32)
sintax_finish_kernel(int nq, int nstrands, const unsigned long long * __restrict__ keys, vsg_sintax_result * __restrict__ out)
{
  int const lane = threadIdx.x & 31;
  int const qi = blockIdx.x * DRAW_WARPS + (threadIdx.x >> 5);
  if (qi >= nq) { return; }
  vsg_sintax_result & r = out[qi];
  unsigned const below = (1u << lane) - 1u;
  int nb[2] = {0, 0}, bc[2] = {0, 0};
  for (int st = 0; st < 2; st++) {
    int n = 0, best = 0;
    for (int b0 = 0; b0 < BOOTS; b0 += 32) {
      int const b = b0 + lane;
      unsigned long long const key = (st < nstrands && b < BOOTS) ? keys[(static_cast<size_t>(qi) * nstrands + st) * BOOTS + b] : 0ull;
      int const cnt = static_cast<int>(key >> 49);
      unsigned const won = __ballot_sync(0xffffffffu, cnt > 1);
      if (cnt > 1) { r.seqno[st][n + __popc(won & below)] = static_cast<int32_t>(0xffffffu - static_cast<uint32_t>(key & 0xffffffu)); }
      n += __popc(won);
      best = max(best, cnt);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { best = max(best, __shfl_xor_sync(0xffffffffu, best, o)); }
    for (int i = n + lane; i < BOOTS; i += 32) { r.seqno[st][i] = -1; }
    nb[st] = n; bc[st] = best;
  }
  if (lane == 0) {
    int strand = 0;
    if (nstrands == 2) {
      if (bc[1] > bc[0]) { strand = 1; }
      else if (bc[1] == bc[0] && nb[1] > nb[0]) { strand = 1; }
    }
    r.strand = strand;
    r.nboot[0] = nb[0]; r.nboot[1] = nb[1];
    r.best_count[0] = bc[0]; r.best_count[1] = bc[1];
  }
}

// ---- the vote and the row (host) ----------------------------------------------------------------------------------
constexpr int TAX_LEVELS = 9;
constexpr char TAX_FIELDS[TAX_LEVELS] = {'d', 'k', 'p', 'c', 'o', 'f', 'g', 's', 't'};

// tax_parse (core/tax.cpp:70-125): the first (^|;)tax= and where its value ends (';' or the end of the header)
bool tax_parse(const char * h, int hl, int & start, int & end)
{
  int offset = 0;
  while (offset < hl - 4) {
    const char * const f = std::strstr(h + offset, "tax=");
    if (f == nullptr) { break; }
    offset = static_cast<int>(f - h);
    if (offset > 0 && h[offset - 1] != ';') { offset += 5; continue; }
    start = offset;
    const char * const t = std::strchr(h + offset + 4, ';');
    end = t == nullptr ? hl : static_cast<int>(t - h);
    return true;
  }
  return false;
}

// tax_split (core/tax.cpp:128-186), including its reading of a level's name up to the next ',' of the whole header
void tax_split(const char * h, int * lstart, int * llen)
{
  int start = 0, end = 0;
  if (!tax_parse(h, static_cast<int>(std::strlen(h)), start, end)) { return; }
  int offset = start + 4;
  while (offset < end) {
    int const c = std::tolower(h[offset]);
    const char * const lv = std::find(TAX_FIELDS, TAX_FIELDS + TAX_LEVELS, c);
    if (lv != TAX_FIELDS + TAX_LEVELS && h[offset + 1] == ':') {
      int const level = static_cast<int>(lv - TAX_FIELDS);
      lstart[level] = offset + 2;
      const char * const comma = std::strchr(h + offset + 2, ',');
      llen[level] = comma != nullptr ? static_cast<int>(comma - h) - offset - 2 : end - offset - 2;
    }
    const char * const next = std::strchr(h + offset, ',');
    offset = next != nullptr ? static_cast<int>(next - h) + 1 : end;
  }
}

// sintax_analyse (sintax.cpp:138-296): one --tabbedout row
void sintax_row(const vsg_sintax_result & r, const char * qhead, const char * const * theads, double cutoff, std::string & out)
{
  int const strand = r.strand;
  int const count = r.nboot[strand];
  bool const enough = count >= (BOOTS + 1) / 2;
  out += qhead;
  out += '\t';
  if (!enough) {
    out += cutoff > 0.0 ? "\t\t\n" : "\t\n";
    return;
  }
  const char * name[BOOTS][TAX_LEVELS];
  int nlen[BOOTS][TAX_LEVELS];
  for (int i = 0; i < count; i++) {
    const char * const h = theads[r.seqno[strand][i]];
    int ls[TAX_LEVELS] = {0}, ll[TAX_LEVELS] = {0};
    tax_split(h, ls, ll);
    for (int l = 0; l < TAX_LEVELS; l++) { name[i][l] = h + ls[l]; nlen[i][l] = ll[l]; }
  }
  int level_best[TAX_LEVELS], level_matchcount[TAX_LEVELS];
  bool included[BOOTS];
  std::fill(included, included + BOOTS, true);
  for (int l = 0; l < TAX_LEVELS; l++) {
    level_best[l] = -1;
    level_matchcount[l] = 0;
    int match[BOOTS], matchcount[BOOTS];
    std::fill(match, match + BOOTS, -1);
    std::fill(matchcount, matchcount + BOOTS, 0);
    for (int i = 0; i < count; i++) {
      if (!included[i]) { continue; }
      for (int j = 0; j <= i; j++) {
        if (included[j] && nlen[i][l] == nlen[j][l] && std::strncmp(name[i][l], name[j][l], static_cast<size_t>(nlen[i][l])) == 0) {
          match[i] = j;
          matchcount[j]++;
          break;
        }
      }
    }
    for (int i = 0; i < count; i++) {
      if (matchcount[i] > level_matchcount[l]) { level_best[l] = i; level_matchcount[l] = matchcount[i]; }
    }
    for (int i = 0; i < count; i++) { if (match[i] != level_best[l]) { included[i] = false; } }
  }
  char num[64];
  bool comma = false;
  for (int l = 0; l < TAX_LEVELS; l++) {
    int const b = level_best[l];
    if (b < 0 || nlen[b][l] <= 0) { continue; }
    if (comma) { out += ','; }
    out += TAX_FIELDS[l]; out += ':';
    out.append(name[b][l], static_cast<size_t>(nlen[b][l]));
    int const w = std::snprintf(num, sizeof num, "(%.2f)", 1.0 * level_matchcount[l] / count);
    out.append(num, static_cast<size_t>(w));
    comma = true;
  }
  out += '\t';
  out += strand != 0 ? '-' : '+';
  if (cutoff > 0.0) {
    out += '\t';
    bool c2 = false;
    for (int l = 0; l < TAX_LEVELS; l++) {
      int const b = level_best[l];
      if (b < 0 || nlen[b][l] <= 0 || !(1.0 * level_matchcount[l] / count >= cutoff)) { continue; }
      if (c2) { out += ','; }
      out += TAX_FIELDS[l]; out += ':';
      out.append(name[b][l], static_cast<size_t>(nlen[b][l]));
      c2 = true;
    }
  }
  out += '\n';
}

}  // namespace

int sintax_check_opts(const vsg_sintax_opts * o, const char * caller)
{
  if (o->random_ties != 0) {
    Error::set(std::string(caller) + ": --sintax_random is not supported (its tie draws interleave with the subsample draws)");
    return VSG_EINVAL;
  }
  if (!(o->cutoff >= 0.0 && o->cutoff <= 1.0)) { Error::set(std::string(caller) + ": cutoff must be in 0..1"); return VSG_EINVAL; }
  return VSG_OK;
}

int sintax_rows_string(const vsg_sintax_result * res, int64_t nq, const char * const * qheads, const char * const * theads,
                       const vsg_sintax_opts * opts, std::string & out)
{
  if (res == nullptr && nq > 0) { Error::set("vsg_sintax_rows: null argument"); return VSG_EINVAL; }
  if (opts == nullptr || nq < 0 || (nq > 0 && (qheads == nullptr || theads == nullptr))) {
    Error::set("vsg_sintax_rows: bad argument");
    return VSG_EINVAL;
  }
  int rc = sintax_check_opts(opts, "vsg_sintax_rows");
  if (rc != VSG_OK) { return rc; }
  for (int64_t i = 0; i < nq; i++) {
    vsg_sintax_result const & r = res[i];
    if (r.strand < 0 || r.strand > 1 || r.nboot[r.strand] < 0 || r.nboot[r.strand] > BOOTS || qheads[i] == nullptr) {
      Error::set("vsg_sintax_rows: malformed result record");
      return VSG_EINVAL;
    }
    sintax_row(r, qheads[i], theads, opts->cutoff, out);
  }
  return VSG_OK;
}

}  // namespace vsg

using namespace vsg;

extern "C" int vsg_sintax(vsg_ctx * c, const vsg_index * ix, const vsg_seqset * queries, int64_t q0, int64_t nq,
                          const vsg_sintax_opts * opts, vsg_sintax_result * out)
{
  if (c == nullptr || ix == nullptr || queries == nullptr || opts == nullptr || (out == nullptr && nq > 0)) {
    Error::set("vsg_sintax: null argument");
    return VSG_EINVAL;
  }
  int rc = sintax_check_opts(opts, "vsg_sintax");
  if (rc != VSG_OK) { return rc; }
  if (q0 < 0 || nq < 0 || q0 + nq > queries->d.n) { Error::set("vsg_sintax: query range out of bounds"); return VSG_EINVAL; }
  if (queries->device != c->device || index_db(ix)->device != c->device) {
    Error::set("vsg_sintax: sequence set / index lives on another device than the context");
    return VSG_EINVAL;
  }
  if (nq == 0) { return VSG_OK; }
  int const k = index_wordlength(ix);
  int maxwin = 0;
  for (int64_t q = q0; q < q0 + nq; q++) { maxwin = std::max(maxwin, queries->h_len[static_cast<size_t>(q)] - k + 1); }
  if (maxwin > 65535) {   // the ranker's limit
    Error::set("vsg_sintax: a query is longer than the device ranker supports (65 534 + wordlength nt)");
    return VSG_EINVAL;
  }
  VSG_CUDA_OK(cudaSetDevice(c->device));
  int nshards = 0;
  const ShardDev * const d_shards = index_shards(ix, nshards);
  int const ns = opts->strand_both != 0 ? 2 : 1;
  int sms = 132;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device);
  VSG_CUDA_OK(cudaFuncSetAttribute(sintax_count_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(COUNT_SMEM)));
  // Chunks of consecutive queries whose scratch fits a quarter of the context's direction-bit budget (a share of the
  // device's free memory, vsg_ctx_create), capped at 1 GiB: per strand the k-mer list (4 B per window), the samples
  // (12.8 kB), their counts and the bootstrap keys; per query its result record.
  size_t const budget = std::min<size_t>(c->dir_budget / 4, static_cast<size_t>(1) << 30);
  size_t const per_boot = sizeof(uint32_t) * SUBSET + 1 + sizeof(unsigned long long);
  std::vector<int64_t> list_off;
  for (int64_t a = 0; a < nq;) {
    int64_t b = a;
    size_t bytes = 0, words = 0;
    int chunk_maxwin = 0;
    while (b < nq) {
      int const win = std::max(0, queries->h_len[static_cast<size_t>(q0 + b)] - k + 1);
      size_t const add = ns * (sizeof(uint32_t) * static_cast<size_t>(win) + BOOTS * per_boot + 16) + sizeof(vsg_sintax_result);
      if (b > a && (bytes + add > budget || b - a >= (1 << 20))) { break; }
      bytes += add; words += ns * static_cast<size_t>(win);
      chunk_maxwin = std::max(chunk_maxwin, win);
      b++;
    }
    int const m = static_cast<int>(b - a);
    int const items = m * ns;
    SeqsetPtr rc_set;
    if (ns == 2 && (rc = seqset_revcomp(c, queries, q0 + a, m, rc_set)) != VSG_OK) { return rc; }
    list_off.assign(static_cast<size_t>(items) + 1, 0);
    for (int i = 0; i < items; i++) {
      int const win = std::max(0, queries->h_len[static_cast<size_t>(q0 + a + i / ns)] - k + 1);
      list_off[static_cast<size_t>(i) + 1] = list_off[static_cast<size_t>(i)] + win;
    }
    // rank_tmp: [list_off items+1][keys items*BOOTS][lists words][samp items*BOOTS*SUBSET][nlist items][results m][nsamp]
    size_t const cells = static_cast<size_t>(items) * BOOTS;
    size_t const off_b = sizeof(int64_t) * (static_cast<size_t>(items) + 1);
    size_t const keys_b = sizeof(unsigned long long) * cells;
    size_t const lists_b = sizeof(uint32_t) * (words + 4);
    size_t const samp_b = sizeof(uint32_t) * cells * SUBSET;
    size_t const nlist_b = sizeof(int32_t) * (static_cast<size_t>(items) + 4);
    size_t const res_b = sizeof(vsg_sintax_result) * static_cast<size_t>(m);
    auto up16 = [](size_t x) { return (x + 15) & ~static_cast<size_t>(15); };
    size_t const total = up16(off_b) + up16(keys_b) + up16(lists_b) + up16(samp_b) + up16(nlist_b) + up16(res_b) + cells + 64;
    if ((rc = c->rank_tmp.reserve(total)) != VSG_OK) { return rc; }
    unsigned char * p = static_cast<unsigned char *>(c->rank_tmp.p);
    int64_t * const d_off = reinterpret_cast<int64_t *>(p); p += up16(off_b);
    unsigned long long * const d_keys = reinterpret_cast<unsigned long long *>(p); p += up16(keys_b);
    uint32_t * const d_lists = reinterpret_cast<uint32_t *>(p); p += up16(lists_b);
    uint32_t * const d_samp = reinterpret_cast<uint32_t *>(p); p += up16(samp_b);
    int32_t * const d_nlist = reinterpret_cast<int32_t *>(p); p += up16(nlist_b);
    vsg_sintax_result * const d_res = reinterpret_cast<vsg_sintax_result *>(p); p += up16(res_b);
    uint8_t * const d_nsamp = p;
    // queries of more than KMER_CAP windows build their first-occurrence table in HBM, one per CTA
    int const kgrid = std::min(items, sms * 4);
    uint32_t * d_scratch = nullptr;
    int scratch_slots = 0;
    if (chunk_maxwin > KMER_CAP) {
      scratch_slots = SMEM_SLOTS;
      while (scratch_slots < 2 * chunk_maxwin) { scratch_slots <<= 1; }
      if ((rc = c->rank_scratch.reserve(sizeof(uint32_t) * 2 * static_cast<size_t>(scratch_slots) * static_cast<size_t>(kgrid))) != VSG_OK) { return rc; }
      d_scratch = static_cast<uint32_t *>(c->rank_scratch.p);
    }
    VSG_CUDA_OK(cudaMemcpyAsync(d_off, list_off.data(), off_b, cudaMemcpyHostToDevice, c->stream));
    VSG_CUDA_OK(cudaMemsetAsync(d_keys, 0, keys_b, c->stream));
    DevSeqs const minus = rc_set ? rc_set->d : DevSeqs{nullptr, nullptr, nullptr, 0};
    sintax_kmers_kernel<<<kgrid, RANK_THREADS, 0, c->stream>>>(queries->d, q0 + a, minus, m, ns, k, d_off, d_lists, d_nlist,
                                                               d_scratch, scratch_slots);
    count_launch();
    unsigned const wgrid = static_cast<unsigned>((m + DRAW_WARPS - 1) / DRAW_WARPS);
    sintax_draw_kernel<<<wgrid, DRAW_WARPS * 32, 0, c->stream>>>(m, ns, opts->seed, opts->query_number0 + a, d_off, d_lists,
                                                                  d_nlist, d_samp, d_nsamp);
    count_launch();
    VSG_CUDA_OK(cudaEventRecord(c->ev[4], c->stream));
    sintax_count_kernel<<<dim3(static_cast<unsigned>(items), static_cast<unsigned>(nshards)), RANK_THREADS, COUNT_SMEM, c->stream>>>(
        index_db(ix)->d, d_shards, d_nlist, d_samp, d_nsamp, d_keys);
    count_launch();
    VSG_CUDA_OK(cudaEventRecord(c->ev[5], c->stream));
    sintax_finish_kernel<<<wgrid, DRAW_WARPS * 32, 0, c->stream>>>(m, ns, d_keys, d_res);
    count_launch();
    VSG_CUDA_OK(cudaMemcpyAsync(out + a, d_res, res_b, cudaMemcpyDeviceToHost, c->stream));
    VSG_CUDA_OK(cudaStreamSynchronize(c->stream));
    VSG_CUDA_OK(cudaGetLastError());
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, c->ev[4], c->ev[5]) == cudaSuccess) { c->prof_rank_ms += ms; }   // vsg_profile.rank_ms
    a = b;
  }
  return VSG_OK;
}

extern "C" int vsg_sintax_rows(const vsg_sintax_result * results, int64_t nq, const char * const * query_headers,
                               const char * const * target_headers, const vsg_sintax_opts * opts, char * buf, int64_t cap,
                               int64_t * len)
{
  if (len == nullptr || cap < 0 || (cap > 0 && buf == nullptr)) { Error::set("vsg_sintax_rows: bad argument"); return VSG_EINVAL; }
  *len = 0;
  std::string out;
  int const rc = sintax_rows_string(results, nq, query_headers, target_headers, opts, out);
  if (rc != VSG_OK) { return rc; }
  *len = static_cast<int64_t>(out.size());
  if (*len > cap) { Error::set("vsg_sintax_rows: the rows do not fit the buffer"); return VSG_ECAP; }
  if (!out.empty()) { std::memcpy(buf, out.data(), out.size()); }
  return VSG_OK;
}
