// chimera.cu — reference-based chimera detection: the --uchime_ref command (core/chimera.cpp:2003-2402 with
// find_best_parents :627-750 and eval_parents :1245-1880, run as `vsearch --uchime_ref --threads 1` orders its output).
//
// For a batch of queries:
//   1. each query of 4 nt or more is cut into four pieces (partition_query): piece i has length
//      (rest + 3 - i) / (4 - i).  The pieces of the batch are one sequence set;
//   2. the pieces are searched against the database's static index with the detection parameters
//      (chimera_detection_parameters, :2805-2823): --id 0.55 = --weak_id, maxaccepts 4, maxrejects 16
//      (search_hits_host: the device ranker and the lock-step candidate loop of the search driver);
//   3. the candidates are the accepted hits of the four pieces in order, without duplicates (:2045-2071);
//   4. the whole query is aligned with every candidate in one vsg_align_pairs call that returns CIGARs;
//   5. parents_kernel (below) selects the two parents of every query of the batch on the device;
//   6. eval_parents runs on the host over worker threads: its doubles are printed with %.4f / %.1f, and the device's
//      FMA contraction could change their last bits.
// The files are then written in input order.
//
// The search driver's heap holds maxaccepts + maxrejects + 8 = 28 candidates where the reference's holds 20 (:2180).
// That changes nothing: the heap's order (count, then length, then sequence number) is total, so the first 20 of the 28
// are the reference's 20, and the candidate loop examines at most maxaccepts + maxrejects - 1 = 19 of them.
#include "vsg_internal.h"
#include "hit_logic.h"
#include "workers.h"

#include <algorithm>
#include <cctype>
#include <chrono>
#include <cinttypes>
#include <cstdarg>
#include <climits>
#include <cstdio>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

using namespace vsg;

namespace {

constexpr int PARTS = 4;                       // parts of a query for uchime (realloc_arrays)
constexpr int MAXPARTS = 100;                  // the most parts of a query for --chimeras_denovo
constexpr int WINDOW = 32;                     // smoothing window of find_best_parents
constexpr int ACCEPTS = 4, REJECTS = 16;       // maxaccepts / maxrejects of the part searches
constexpr double CHIMERA_ID = 0.55;
constexpr int MAXCAND = PARTS * ACCEPTS;       // the most distinct candidates a uchime query can have
constexpr int MAXPARENTS = 20;                 // the most parents of find_best_parents_long ('A' to 'T')
constexpr int PARENT_THREADS = 256;
constexpr int LONG_THREADS = 128;

// the parts of a query of `len` nt (realloc_arrays): four for the uchime commands, --chimeras_parts (0: one per 100 nt)
// clamped to 2 .. 100 for --chimeras_denovo
int parts_of(const vsg_uchime_opts & o, int64_t len)
{
  if (o.command != VSG_CHIMERAS_DENOVO) { return PARTS; }
  int64_t const p = o.chimeras_parts == 0 ? (len + 99) / 100 : o.chimeras_parts;
  return static_cast<int>(std::min<int64_t>(MAXPARTS, std::max<int64_t>(2, p)));
}

// Status of chimera.cpp: what eval_parents decides for a query
enum Status : int { NO_PARENTS = 0, NO_ALIGNMENT = 1, LOW_SCORE = 2, SUSPICIOUS = 3, CHIMERIC = 4 };

// One query of a parents_kernel launch: its entry in the query set, its candidates [c0, c0 + nc) of the launch's
// candidate arrays, and its scratch (2 * nc * qlen + 3 * qlen bytes) at `scratch`.
struct ParentJob {
  int64_t qi;
  int64_t scratch;
  int32_t c0, nc;
};

// find_matches + find_best_parents (chimera.cpp:367-413, 627-750) for one query per CTA, a warp per candidate.
//   match[c][p]  = 1 where candidate c's CIGAR aligns query position p to a target symbol sharing a 4-bit bit with it;
//   smooth[c][p] = the match count over the 32-position window ending at p (p >= 31), from a warp prefix sum: the
//                  inclusive sum at p minus the one 32 positions earlier, which the same lane held one chunk before;
//   maxs[p]      = the largest smooth over the candidates not selected yet;
//   wins[c]      = the positions p (maxs[p] != 0) where candidate c reaches maxs[p].
// The candidate with the most wins (the first on a tie) is parent A.  Round two wipes the 32-window of every position
// where A reached the maximum from every candidate's matches and selects parent B the same way.
// out[b] = the two parents (candidate indices within the query), or -1 where none was found.
__global__ void __launch_bounds__(PARENT_THREADS) parents_kernel(DevSeqs q, DevSeqs t, const ParentJob * __restrict__ jobs,
                                                                 const uint32_t * __restrict__ cand, const char * __restrict__ cigars,
                                                                 const int64_t * __restrict__ cigar_off, uint8_t * __restrict__ scratch,
                                                                 int2 * __restrict__ out)
{
  __shared__ int wins[MAXCAND];
  __shared__ int best[2];
  ParentJob const J = jobs[blockIdx.x];
  int const qlen = q.len[J.qi];
  int const nc = J.nc;
  uint8_t const * const qs = q.sym + q.off[J.qi];
  uint8_t * const match = scratch + J.scratch;
  uint8_t * const smooth = match + static_cast<size_t>(nc) * qlen;
  uint8_t * const maxs = smooth + static_cast<size_t>(nc) * qlen;
  uint8_t * const cond = maxs + qlen;
  uint8_t * const wiped = cond + qlen;
  int const lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;

  for (int c = warp; c < nc; c += nwarps) {
    uint8_t * const m = match + static_cast<size_t>(c) * qlen;
    for (int i = lane; i < qlen; i += 32) { m[i] = 0; }
    __syncwarp();
    uint32_t const tg = cand[J.c0 + c];
    uint8_t const * const ts = t.sym + t.off[tg];
    char const * s = cigars + cigar_off[J.c0 + c];
    int qpos = 0, tpos = 0;
    while (*s != '\0') {   // every lane parses the same CIGAR; an M run is compared 32 positions at a time
      int run = 0;
      bool digits = false;
      while (*s >= '0' && *s <= '9') { run = run * 10 + (*s - '0'); ++s; digits = true; }
      if (!digits) { run = 1; }
      char const op = *s++;
      if (op == 'M') {
        for (int j = lane; j < run; j += 32) { m[qpos + j] = ((qs[qpos + j] & ts[tpos + j] & 15) != 0) ? 1 : 0; }
        qpos += run; tpos += run;
      } else if (op == 'I') {
        tpos += run;
      } else {
        qpos += run;
      }
    }
  }
  if (threadIdx.x < 2) { best[threadIdx.x] = -1; }
  __syncthreads();

  for (int f = 0; f < 2; f++) {
    int const b0 = best[0];
    if (f > 0) {
      for (int p = threadIdx.x; p < qlen; p += blockDim.x) {
        cond[p] = (p >= WINDOW - 1 && smooth[static_cast<size_t>(b0) * qlen + p] == maxs[p]) ? 1 : 0;
      }
      __syncthreads();
      for (int p = threadIdx.x; p < qlen; p += blockDim.x) {
        uint8_t w = 0;
        int const hi = min(p + WINDOW - 1, qlen - 1);
        for (int z = max(p, WINDOW - 1); z <= hi; z++) { w |= cond[z]; }
        wiped[p] = w;
      }
      __syncthreads();
      for (int c = 0; c < nc; c++) {
        for (int p = threadIdx.x; p < qlen; p += blockDim.x) {
          if (wiped[p] != 0) { match[static_cast<size_t>(c) * qlen + p] = 0; }
        }
      }
    }
    if (threadIdx.x < MAXCAND) { wins[threadIdx.x] = 0; }
    __syncthreads();
    for (int c = warp; c < nc; c += nwarps) {
      if (c == b0) { continue; }
      uint8_t const * const m = match + static_cast<size_t>(c) * qlen;
      uint8_t * const sm = smooth + static_cast<size_t>(c) * qlen;
      int carry = 0, prev = 0;
      for (int base = 0; base < qlen; base += 32) {
        int const p = base + lane;
        int v = p < qlen ? m[p] : 0;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          int const u = __shfl_up_sync(0xffffffffu, v, d);
          if (lane >= d) { v += u; }
        }
        int const cur = carry + v;   // matches in [0, p]
        if (p < qlen && p >= WINDOW - 1) { sm[p] = static_cast<uint8_t>(cur - prev); }
        prev = cur;
        carry = __shfl_sync(0xffffffffu, cur, 31);
      }
    }
    __syncthreads();
    for (int p = threadIdx.x; p < qlen; p += blockDim.x) {
      int mx = 0;
      if (p >= WINDOW - 1) {
        for (int c = 0; c < nc; c++) {
          if (c != b0) { mx = max(mx, static_cast<int>(smooth[static_cast<size_t>(c) * qlen + p])); }
        }
      }
      maxs[p] = static_cast<uint8_t>(mx);
    }
    __syncthreads();
    for (int p = WINDOW - 1 + threadIdx.x; p < qlen; p += blockDim.x) {
      int const mx = maxs[p];
      if (mx == 0) { continue; }
      for (int c = 0; c < nc; c++) {
        if (c != b0 && smooth[static_cast<size_t>(c) * qlen + p] == mx) { atomicAdd(&wins[c], 1); }
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int maxwins = 0, bi = -1;
      for (int c = 0; c < nc; c++) {
        if (wins[c] > maxwins) { maxwins = wins[c]; bi = c; }
      }
      best[f] = bi;
    }
    __syncthreads();
    if (best[f] < 0) { break; }
  }
  if (threadIdx.x == 0) { out[blockIdx.x] = make_int2(best[0], best[1]); }
}

// scan_matches (chimera.cpp:439-502) over m[0, len): the longest window whose score sum is >= 0, a match scoring pct and
// a mismatch pct - 100, and of those the first.  q holds len + 1 doubles: the prefix sums p, then their suffix maxima in
// place; p[i - 1] of the two-pointer walk is summed again in the same order, so every double is the reference's.  The
// additions are explicitly rounded so that no contraction can change a comparison.
__device__ bool scan_matches(const uint8_t * __restrict__ m, int len, double pct, double * __restrict__ q, int & best_start, int & best_len)
{
  double const sm = pct, sx = __dsub_rn(pct, 100.0);
  double p = 0.0;
  q[0] = 0.0;
  for (int i = 0; i < len; i++) { p = __dadd_rn(p, m[i] != 0 ? sm : sx); q[i + 1] = p; }
  for (int i = len - 1; i >= 0; i--) { double const a = q[i + 1], b = q[i]; q[i] = a < b ? b : a; }
  int bi = 0, bd = -1;
  double bc = -1.0, pim1 = 0.0;   // pim1 = p[i - 1]
  int i = 1, j = 1;
  while (j <= len) {
    double const c = __dsub_rn(q[j], pim1);
    if (c >= 0.0) {
      int const d = j - i + 1;
      if (d > bd) { bi = i; bd = d; bc = c; }
      j += 1;
    } else {
      pim1 = __dadd_rn(pim1, m[i - 1] != 0 ? sm : sx);
      i += 1;
    }
  }
  if (bc >= 0.0) { best_start = bi - 1; best_len = bd; return true; }
  return false;
}

// find_matches + find_best_parents_long (chimera.cpp:367-413, 505-624) for one query per CTA.
//   match[c][p] = 1 where candidate c's CIGAR aligns query position p to a target symbol sharing a 4-bit bit with it;
//   ins[c][p]   = 1 where the CIGAR inserts target symbols before query position p;
//   used[p]     = 1 where a parent found so far covers p.
// Each round, a thread scans the segments of its candidates' rows in order (a segment runs over unused positions and
// stops before an insert; the position that ends it is skipped) and keeps its first longest scan_matches window; the
// CTA then takes the longest, the lowest candidate on a tie, which is the reference's first strict maximum.  A window
// shorter than length_min ends the search.  The scratch at `scratch` holds min(nc, LONG_THREADS) * (qlen + 1) doubles (a
// scan_matches buffer for each thread that has a candidate), then
// 2 * nc * qlen + qlen bytes.  out[b * MAXPARENTS + f] = (candidate, start, length) of the f-th parent found, candidate
// -1 past the last.
__global__ void __launch_bounds__(LONG_THREADS, 1) parents_long_kernel(DevSeqs q, DevSeqs t, const ParentJob * __restrict__ jobs,
                                                                    const uint32_t * __restrict__ cand, const char * __restrict__ cigars,
                                                                    const int64_t * __restrict__ cigar_off, uint8_t * __restrict__ scratch,
                                                                    int parents_max, int length_min, double diff_pct, int4 * __restrict__ out)
{
  __shared__ unsigned long long best_key;
  __shared__ int best_start;
  ParentJob const J = jobs[blockIdx.x];
  int const qlen = q.len[J.qi];
  int const nc = J.nc;
  uint8_t const * const qs = q.sym + q.off[J.qi];
  double * const pq = reinterpret_cast<double *>(scratch + J.scratch) + static_cast<size_t>(threadIdx.x) * (qlen + 1);
  uint8_t * const match = scratch + J.scratch + static_cast<size_t>(min(nc, LONG_THREADS)) * (qlen + 1) * sizeof(double);
  uint8_t * const ins = match + static_cast<size_t>(nc) * qlen;
  uint8_t * const used = ins + static_cast<size_t>(nc) * qlen;
  int const lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;

  for (int c = warp; c < nc; c += nwarps) {
    uint8_t * const m = match + static_cast<size_t>(c) * qlen;
    uint8_t * const in = ins + static_cast<size_t>(c) * qlen;
    for (int i = lane; i < qlen; i += 32) { m[i] = 0; in[i] = 0; }
    __syncwarp();
    uint32_t const tg = cand[J.c0 + c];
    uint8_t const * const ts = t.sym + t.off[tg];
    char const * s = cigars + cigar_off[J.c0 + c];
    int qpos = 0, tpos = 0;
    while (*s != '\0') {
      int run = 0;
      bool digits = false;
      while (*s >= '0' && *s <= '9') { run = run * 10 + (*s - '0'); ++s; digits = true; }
      if (!digits) { run = 1; }
      char const op = *s++;
      if (op == 'M') {
        for (int j = lane; j < run; j += 32) { m[qpos + j] = ((qs[qpos + j] & ts[tpos + j] & 15) != 0) ? 1 : 0; }
        qpos += run; tpos += run;
      } else if (op == 'I') {
        // an insert after the last position lands, in the reference, on the next row's position 0, which always starts
        // a segment: it changes nothing, so it is dropped
        if (lane == 0 && qpos < qlen) { in[qpos] = 1; }
        tpos += run;
      } else {
        qpos += run;
      }
    }
  }
  for (int p = threadIdx.x; p < qlen; p += blockDim.x) { used[p] = 0; }
  __syncthreads();

  int found = 0;
  for (int f = 0; f < parents_max; f++) {
    if (threadIdx.x == 0) { best_key = 0; }
    __syncthreads();
    int blen = 0, bcand = -1, bstart = 0;
    for (int c = threadIdx.x; c < nc; c += blockDim.x) {
      uint8_t const * const m = match + static_cast<size_t>(c) * qlen;
      uint8_t const * const in = ins + static_cast<size_t>(c) * qlen;
      int j = 0;
      while (j < qlen) {
        int const start = j;
        int len = 0;
        while (j < qlen && used[j] == 0 && (len == 0 || in[j] == 0)) { ++len; ++j; }
        int ss = 0, sl = 0;
        if (len > blen && scan_matches(m + start, len, diff_pct, pq, ss, sl) && sl > blen) { bcand = c; bstart = start + ss; blen = sl; }
        ++j;
      }
    }
    // the longest window, then the lowest candidate (each thread holds one candidate's first longest window)
    unsigned long long const key = bcand < 0 ? 0ull : (static_cast<unsigned long long>(blen) << 32) | (0xffffffffu - static_cast<unsigned>(bcand));
    if (key != 0) { atomicMax(&best_key, key); }
    __syncthreads();
    unsigned long long const bk = best_key;
    if (bk != 0 && key == bk) { best_start = bstart; }
    __syncthreads();
    int const len = static_cast<int>(bk >> 32);
    if (bk == 0 || len < length_min) { break; }
    int const start = best_start;
    if (threadIdx.x == 0) { out[static_cast<size_t>(blockIdx.x) * MAXPARENTS + f] = make_int4(static_cast<int>(0xffffffffu - static_cast<unsigned>(bk)), start, len, 0); }
    for (int p = start + threadIdx.x; p < start + len; p += blockDim.x) { used[p] = 1; }
    found++;
    __syncthreads();
  }
  for (int f = found + threadIdx.x; f < MAXPARENTS; f += blockDim.x) { out[static_cast<size_t>(blockIdx.x) * MAXPARENTS + f] = make_int4(-1, 0, 0, 0); }
}

// ---- the host side of eval_parents ------------------------------------------------------------------------------------

struct Maps {
  unsigned char code[256];   // map_4bit: the IUPAC bits, 0 for a gap or anything else
  char upper[256];           // map_uppercase: letters upper-cased, anything else 'N'
  Maps()
  {
    for (int i = 0; i < 256; i++) { code[i] = 0; upper[i] = 'N'; }
    char const * const sym = "ACGTUMRSVWYHKDBN";
    unsigned char const val[] = {1, 2, 4, 8, 8, 3, 5, 6, 7, 9, 10, 11, 12, 13, 14, 15};
    for (int i = 0; sym[i] != '\0'; i++) {
      code[static_cast<unsigned char>(sym[i])] = val[i];
      code[static_cast<unsigned char>(sym[i] + 32)] = val[i];
    }
    for (int ch = 'A'; ch <= 'Z'; ch++) { upper[ch] = static_cast<char>(ch); upper[ch + 32] = static_cast<char>(ch); }
  }
};
const Maps & maps()
{
  static const Maps m;
  return m;
}
inline bool ambiguous(unsigned char c) { return !(c == 1 || c == 2 || c == 4 || c == 8); }

template <class Fn>
void for_each_run(const char * s, Fn && fn)
{
  while (*s != '\0') {
    int run = 0;
    bool digits = false;
    while (*s >= '0' && *s <= '9') { run = run * 10 + (*s - '0'); ++s; digits = true; }
    if (!digits) { run = 1; }
    fn(*s++, run);
  }
}

struct Parent {
  const char * seq;
  int64_t len;
  const std::string * head;
  const char * cigar;
};

struct Eval {
  int status = NO_PARENTS;
  double h = 0.0;
  std::string uchimeout, uchimealns;
};

struct EvalOpts {
  double dn, xn, mindiv, minh;
  int mindiffs;
  bool xsize, uchimeout5, want_out, want_alns;
  int alignwidth;
  bool perfect_model;   // --uchime2_denovo / --uchime3_denovo: chimeric only when the model matches the query perfectly
};

std::string fmt(const char * f, ...) __attribute__((format(printf, 1, 2)));
std::string fmt(const char * f, ...)
{
  char buf[512];
  va_list ap;
  va_start(ap, f);
  int const n = std::vsnprintf(buf, sizeof buf, f, ap);
  va_end(ap);
  return std::string(buf, static_cast<size_t>(std::max(0, std::min<int>(n, sizeof buf - 1))));
}

std::string strip(const std::string & h, bool xsize)
{
  std::string s;
  header_fprint_strip(s, h, xsize);
  return s;
}

// eval_parents (chimera.cpp:1245-1880) for a query with parents P[0], P[1]: the multiple alignment of the three, the
// diffs and votes, the best crossover, the status, and the --uchimeout row and --uchimealns block when asked for.
void eval_parents(const char * qseq, int qlen, const std::string & qhead, const Parent P[2], const EvalOpts & o, Eval & e)
{
  Maps const & M = maps();
  // fill_max_alignment_length: the longest insertion in front of each query position
  std::vector<int> maxi(static_cast<size_t>(qlen) + 1, 0);
  for (int f = 0; f < 2; f++) {
    int64_t pos = 0;
    for_each_run(P[f].cigar, [&](char op, int run) {
      if (op == 'I') { maxi[static_cast<size_t>(pos)] = std::max(maxi[static_cast<size_t>(pos)], run); } else { pos += run; }
    });
  }
  int alnlen = qlen;
  for (int v : maxi) { alnlen += v; }
  // fill_alignment_parents
  std::string paln[2];
  for (int f = 0; f < 2; f++) {
    std::string & a = paln[f];
    a.reserve(static_cast<size_t>(alnlen));
    bool inserted = false;
    int qpos = 0;
    int64_t tpos = 0;
    for_each_run(P[f].cigar, [&](char op, int run) {
      if (op == 'I') {
        for (int j = 0; j < maxi[static_cast<size_t>(qpos)]; j++) {
          a += j < run ? M.upper[static_cast<unsigned char>(P[f].seq[tpos++])] : '-';
        }
        inserted = true;
      } else {
        for (int j = 0; j < run; j++) {
          if (!inserted) { a.append(static_cast<size_t>(maxi[static_cast<size_t>(qpos)]), '-'); }
          a += op == 'M' ? M.upper[static_cast<unsigned char>(P[f].seq[tpos++])] : '-';
          ++qpos;
          inserted = false;
        }
      }
    });
    if (!inserted) { a.append(static_cast<size_t>(maxi[static_cast<size_t>(qpos)]), '-'); }
  }
  std::string qaln;
  qaln.reserve(static_cast<size_t>(alnlen));
  for (int i = 0; i < qlen; i++) {
    qaln.append(static_cast<size_t>(maxi[static_cast<size_t>(i)]), '-');
    qaln += M.upper[static_cast<unsigned char>(qseq[i])];
  }
  qaln.append(static_cast<size_t>(maxi[static_cast<size_t>(qlen)]), '-');

  // ignored columns, lower-cased parent symbols and diffs
  std::vector<char> ignore(static_cast<size_t>(alnlen), 0);
  std::string diffs(static_cast<size_t>(alnlen), ' ');
  auto code = [&](char ch) { return M.code[static_cast<unsigned char>(ch)]; };
  for (int i = 0; i < alnlen; i++) {
    unsigned char const qs = code(qaln[static_cast<size_t>(i)]), p1 = code(paln[0][static_cast<size_t>(i)]),
                        p2 = code(paln[1][static_cast<size_t>(i)]);
    if (qs == 0 || p1 == 0 || p2 == 0) {
      ignore[static_cast<size_t>(i)] = 1;
      if (i > 0) { ignore[static_cast<size_t>(i) - 1] = 1; }
      if (i < alnlen - 1) { ignore[static_cast<size_t>(i) + 1] = 1; }
    }
    if (ambiguous(qs) || ambiguous(p1) || ambiguous(p2)) { ignore[static_cast<size_t>(i)] = 1; }
    if (p1 != 0 && p1 != qs) { paln[0][static_cast<size_t>(i)] = static_cast<char>(std::tolower(paln[0][static_cast<size_t>(i)])); }
    if (p2 != 0 && p2 != qs) { paln[1][static_cast<size_t>(i)] = static_cast<char>(std::tolower(paln[1][static_cast<size_t>(i)])); }
    char d = ' ';
    if (qs != 0 && p1 != 0 && p2 != 0) {
      if (p1 == p2) { d = qs == p1 ? ' ' : 'N'; } else { d = qs == p1 ? 'A' : (qs == p2 ? 'B' : '?'); }
    }
    diffs[static_cast<size_t>(i)] = d;
  }

  // the best crossover
  int sumA = 0, sumB = 0, sumN = 0;
  for (int i = 0; i < alnlen; i++) {
    if (ignore[static_cast<size_t>(i)] != 0) { continue; }
    char const d = diffs[static_cast<size_t>(i)];
    if (d == 'A') { ++sumA; } else if (d == 'B') { ++sumB; } else if (d != ' ') { ++sumN; }
  }
  int left_n = 0, left_a = 0, left_y = 0, right_n = sumA, right_a = sumN, right_y = sumB;
  double best_h = -1;
  int best_i = -1;
  bool reverse = false;
  int bly = 0, bry = 0, bln = 0, brn = 0, bla = 0, bra = 0;
  for (int i = 0; i < alnlen; i++) {
    if (ignore[static_cast<size_t>(i)] != 0) { continue; }
    char const d = diffs[static_cast<size_t>(i)];
    if (d == ' ') { continue; }
    if (d == 'A') { ++left_y; --right_n; } else if (d == 'B') { ++left_n; --right_y; } else { ++left_a; --right_a; }
    if (left_y > left_n && right_y > right_n) {
      double const lh = left_y / ((o.xn * (left_n + o.dn)) + left_a);
      double const rh = right_y / ((o.xn * (right_n + o.dn)) + right_a);
      double const h = lh * rh;
      if (h > best_h) {
        reverse = false; best_h = h; best_i = i;
        bln = left_n; bly = left_y; bla = left_a; brn = right_n; bry = right_y; bra = right_a;
      }
    } else if (left_n > left_y && right_n > right_y) {
      double const lh = left_n / ((o.xn * (left_y + o.dn)) + left_a);
      double const rh = right_n / ((o.xn * (right_y + o.dn)) + right_a);
      double const h = lh * rh;
      if (h > best_h) {
        reverse = true; best_h = h; best_i = i;
        bln = left_y; bly = left_n; bla = left_a; brn = right_y; bry = right_n; bra = right_a;
      }
    }
  }
  e.h = best_h > 0 ? best_h : 0.0;
  e.status = NO_ALIGNMENT;
  if (!(best_h >= 0.0)) { return; }
  e.status = LOW_SCORE;
  if (reverse) {
    for (char & d : diffs) { if (d == 'A') { d = 'B'; } else if (d == 'B') { d = 'A'; } }
  }
  std::string model(static_cast<size_t>(alnlen), ' '), votes(static_cast<size_t>(alnlen), ' ');
  for (int i = 0; i < alnlen; i++) {
    char const m = i <= best_i ? 'A' : 'B';
    model[static_cast<size_t>(i)] = m;
    char v = ' ';
    if (ignore[static_cast<size_t>(i)] == 0) {
      char const d = diffs[static_cast<size_t>(i)];
      if (d == 'A' || d == 'B') { v = d == m ? '+' : '!'; } else if (d == 'N' || d == '?') { v = '0'; }
    }
    votes[static_cast<size_t>(i)] = v;
    if (v == '!') { diffs[static_cast<size_t>(i)] = static_cast<char>(std::tolower(diffs[static_cast<size_t>(i)])); }
  }
  for (int i = best_i + 1; i < alnlen; i++) {
    if (diffs[static_cast<size_t>(i)] == ' ' || diffs[static_cast<size_t>(i)] == 'A') { model[static_cast<size_t>(i)] = 'x'; } else { break; }
  }
  int const ia = reverse ? 1 : 0, ib = reverse ? 0 : 1;
  int mQA = 0, mQB = 0, mAB = 0, mQM = 0, cols = 0;
  for (int i = 0; i < alnlen; i++) {
    if (ignore[static_cast<size_t>(i)] != 0) { continue; }
    ++cols;
    unsigned char const qs = code(qaln[static_cast<size_t>(i)]), as = code(paln[ia][static_cast<size_t>(i)]),
                        bs = code(paln[ib][static_cast<size_t>(i)]);
    unsigned char const ms = i <= best_i ? as : bs;
    mQA += qs == as; mQB += qs == bs; mAB += as == bs; mQM += qs == ms;
  }
  double const QA = 100.0 * mQA / cols;
  double const QB = 100.0 * mQB / cols;
  double const AB = 100.0 * mAB / cols;
  double const QT = std::max(QA, QB);
  double const QM = 100.0 * mQM / cols;
  double const divdiff = QM - QT;
  double const divfrac = 100.0 * divdiff / QT;
  int const sumL = bln + bla + bly, sumR = brn + bra + bry;
  if (o.perfect_model) {
    if (mQM == cols && QT < 100.0) { e.status = CHIMERIC; }
  } else if (best_h >= o.minh) {
    e.status = SUSPICIOUS;
    if (divdiff >= o.mindiv && sumL >= o.mindiffs && sumR >= o.mindiffs) { e.status = CHIMERIC; }
  }
  Parent const & A = P[ia];
  Parent const & B = P[ib];
  if (o.want_alns && e.status == CHIMERIC) {
    std::string & s = e.uchimealns;
    s += '\n';
    s.append(72, '-');
    s += '\n';
    s += fmt("Query   (%5d nt) ", qlen) + strip(qhead, o.xsize);
    s += fmt("\nParentA (%5" PRIu64 " nt) ", static_cast<uint64_t>(A.len)) + strip(*A.head, o.xsize);
    s += fmt("\nParentB (%5" PRIu64 " nt) ", static_cast<uint64_t>(B.len)) + strip(*B.head, o.xsize);
    s += "\n\n";
    int const width = o.alignwidth > 0 ? o.alignwidth : alnlen;
    int qpos = 0, p1pos = 0, p2pos = 0, rest = alnlen;
    for (int i = 0; i < alnlen; i += width) {
      int const w = std::min(rest, width);
      int qnt = 0, p1nt = 0, p2nt = 0;
      for (int j = 0; j < w; j++) {
        qnt += qaln[static_cast<size_t>(i + j)] != '-';
        p1nt += paln[0][static_cast<size_t>(i + j)] != '-';
        p2nt += paln[1][static_cast<size_t>(i + j)] != '-';
      }
      auto line = [&](char tag, int pos, const std::string & a, int nt) {
        s += fmt("%c %5d ", tag, pos + 1);
        s.append(a, static_cast<size_t>(i), static_cast<size_t>(w));
        s += fmt(" %d\n", pos + nt);
      };
      if (!reverse) {
        line('A', p1pos, paln[0], p1nt); line('Q', qpos, qaln, qnt); line('B', p2pos, paln[1], p2nt);
      } else {
        line('A', p2pos, paln[1], p2nt); line('Q', qpos, qaln, qnt); line('B', p1pos, paln[0], p1nt);
      }
      s += "Diffs   "; s.append(diffs, static_cast<size_t>(i), static_cast<size_t>(w)); s += '\n';
      s += "Votes   "; s.append(votes, static_cast<size_t>(i), static_cast<size_t>(w)); s += '\n';
      s += "Model   "; s.append(model, static_cast<size_t>(i), static_cast<size_t>(w)); s += "\n\n";
      qpos += qnt; p1pos += p1nt; p2pos += p2nt;
      rest -= width;
    }
    s += fmt("Ids.  QA %.1f%%, QB %.1f%%, AB %.1f%%, QModel %.1f%%, Div. %+.1f%%\n", QA, QB, AB, QM, divfrac);
    s += fmt("Diffs Left %d: N %d, A %d, Y %d (%.1f%%); Right %d: N %d, A %d, Y %d (%.1f%%), Score %.4f\n", sumL, bln, bla, bly,
             100.0 * bly / sumL, sumR, brn, bra, bry, 100.0 * bry / sumR, best_h);
  }
  if (o.want_out) {
    std::string & s = e.uchimeout;
    s += fmt("%.4f\t", best_h) + strip(qhead, o.xsize) + '\t' + strip(*A.head, o.xsize) + '\t' + strip(*B.head, o.xsize) + '\t';
    if (!o.uchimeout5) { s += strip(QA >= QB ? *A.head : *B.head, o.xsize) + '\t'; }
    s += fmt("%.1f\t%.1f\t%.1f\t%.1f\t%.1f\t%d\t%d\t%d\t%d\t%d\t%d\t%.1f\t%c\n", QM, QA, QB, AB, QT, bly, bln, bla, bry, brn, bra, divdiff,
             e.status == CHIMERIC ? 'Y' : (e.status == LOW_SCORE ? 'N' : '?'));
  }
}

// eval_parents_long (chimera.cpp:995-1242) for a query whose parents P[0 .. np) cover it, sorted by start; the model
// gives positions [starts[f], starts[f] + lens[f]) to parent f.  Always chimeric, with score 99.9999 in the --tabbedout
// row (the uchimeout slot) and the --alnout block (the uchimealns slot) when asked for.
void eval_parents_long(const char * qseq, int qlen, const std::string & qhead, const Parent * P, const int * starts, const int * lens, int np,
                       const EvalOpts & o, Eval & e)
{
  Maps const & M = maps();
  e.status = CHIMERIC;
  std::vector<int> maxi(static_cast<size_t>(qlen) + 1, 0);
  for (int f = 0; f < np; f++) {
    int64_t pos = 0;
    for_each_run(P[f].cigar, [&](char op, int run) {
      if (op == 'I') { maxi[static_cast<size_t>(pos)] = std::max(maxi[static_cast<size_t>(pos)], run); } else { pos += run; }
    });
  }
  int alnlen = qlen;
  for (int v : maxi) { alnlen += v; }
  std::vector<std::string> paln(static_cast<size_t>(np));
  for (int f = 0; f < np; f++) {
    std::string & a = paln[static_cast<size_t>(f)];
    a.reserve(static_cast<size_t>(alnlen));
    bool inserted = false;
    int qpos = 0;
    int64_t tpos = 0;
    for_each_run(P[f].cigar, [&](char op, int run) {
      if (op == 'I') {
        for (int j = 0; j < maxi[static_cast<size_t>(qpos)]; j++) {
          a += j < run ? M.upper[static_cast<unsigned char>(P[f].seq[tpos++])] : '-';
        }
        inserted = true;
      } else {
        for (int j = 0; j < run; j++) {
          if (!inserted) { a.append(static_cast<size_t>(maxi[static_cast<size_t>(qpos)]), '-'); }
          a += op == 'M' ? M.upper[static_cast<unsigned char>(P[f].seq[tpos++])] : '-';
          ++qpos;
          inserted = false;
        }
      }
    });
    if (!inserted) { a.append(static_cast<size_t>(maxi[static_cast<size_t>(qpos)]), '-'); }
  }
  std::string qaln, model;
  qaln.reserve(static_cast<size_t>(alnlen));
  model.reserve(static_cast<size_t>(alnlen));
  int nth = 0;
  for (int i = 0; i < qlen; i++) {
    if (nth + 1 < np && i >= starts[nth] + lens[nth]) { ++nth; }
    qaln.append(static_cast<size_t>(maxi[static_cast<size_t>(i)]), '-');
    qaln += M.upper[static_cast<unsigned char>(qseq[i])];
    model.append(static_cast<size_t>(maxi[static_cast<size_t>(i)]) + 1, static_cast<char>('A' + nth));
  }
  qaln.append(static_cast<size_t>(maxi[static_cast<size_t>(qlen)]), '-');
  model.append(static_cast<size_t>(maxi[static_cast<size_t>(qlen)]), static_cast<char>('A' + nth));

  // lower-cased parent symbols, diffs (the one parent that matches the query, if exactly one does) and matches
  std::string diffs(static_cast<size_t>(alnlen), ' ');
  std::vector<int> mQP(static_cast<size_t>(np), 0);
  for (int i = 0; i < alnlen; i++) {
    unsigned char const qs = M.code[static_cast<unsigned char>(qaln[static_cast<size_t>(i)])];
    bool defined = qs != 0;
    int z = 0;
    char d = ' ';
    for (int f = 0; f < np; f++) {
      char & ch = paln[static_cast<size_t>(f)][static_cast<size_t>(i)];
      unsigned char const ps = M.code[static_cast<unsigned char>(ch)];
      defined = defined && ps != 0;
      if (ps == qs) { d = static_cast<char>('A' + f); ++z; ++mQP[static_cast<size_t>(f)]; }
      if (ps != 0 && ps != qs) { ch = static_cast<char>(std::tolower(ch)); }
    }
    diffs[static_cast<size_t>(i)] = defined && z == 1 ? d : ' ';
  }
  double QP[MAXPARENTS] = {};
  for (int f = 0; f < np; f++) { QP[f] = 100.0 * mQP[static_cast<size_t>(f)] / alnlen; }
  double const QT = *std::max_element(QP, QP + MAXPARENTS);
  double const QA = QP[0], QB = QP[1], QC = np > 2 ? QP[2] : 0.00, QM = 100.00;
  double const divfrac = 100.00 * (QM - QT) / QT;
  if (o.want_alns) {
    std::string & s = e.uchimealns;
    s += '\n';
    s.append(72, '-');
    s += '\n';
    s += fmt("Query   (%5d nt) ", qlen) + strip(qhead, o.xsize);
    for (int f = 0; f < np; f++) {
      s += fmt("\nParent%c (%5" PRIu64 " nt) ", 'A' + f, static_cast<uint64_t>(P[f].len)) + strip(*P[f].head, o.xsize);
    }
    s += "\n\n";
    int const width = o.alignwidth > 0 ? o.alignwidth : alnlen;
    int qpos = 0, rest = alnlen;
    std::vector<int> ppos(static_cast<size_t>(np), 0), pnt(static_cast<size_t>(np));
    for (int i = 0; i < alnlen; i += width) {
      int const w = std::min(rest, width);
      int qnt = 0;
      std::fill(pnt.begin(), pnt.end(), 0);
      for (int j = 0; j < w; j++) {
        qnt += qaln[static_cast<size_t>(i + j)] != '-';
        for (int f = 0; f < np; f++) { pnt[static_cast<size_t>(f)] += paln[static_cast<size_t>(f)][static_cast<size_t>(i + j)] != '-'; }
      }
      s += fmt("Q %5d ", qpos + 1); s.append(qaln, static_cast<size_t>(i), static_cast<size_t>(w)); s += fmt(" %d\n", qpos + qnt);
      for (int f = 0; f < np; f++) {
        s += fmt("%c %5d ", 'A' + f, ppos[static_cast<size_t>(f)] + 1);
        s.append(paln[static_cast<size_t>(f)], static_cast<size_t>(i), static_cast<size_t>(w));
        s += fmt(" %d\n", ppos[static_cast<size_t>(f)] + pnt[static_cast<size_t>(f)]);
      }
      s += "Diffs   "; s.append(diffs, static_cast<size_t>(i), static_cast<size_t>(w)); s += '\n';
      s += "Model   "; s.append(model, static_cast<size_t>(i), static_cast<size_t>(w)); s += "\n\n";
      rest -= width;
      qpos += qnt;
      for (int f = 0; f < np; f++) { ppos[static_cast<size_t>(f)] += pnt[static_cast<size_t>(f)]; }
    }
    s += fmt("Ids.  QA %.2f%%, QB %.2f%%, QC %.2f%%, QT %.2f%%, QModel %.2f%%, Div. %+.2f%%\n", QA, QB, QC, QT, QM, divfrac);
  }
  if (o.want_out) {
    std::string & s = e.uchimeout;
    s += fmt("%.4f\t", 99.9999) + strip(qhead, o.xsize) + '\t' + strip(*P[0].head, o.xsize) + '\t' + strip(*P[1].head, o.xsize) + '\t';
    s += np > 2 ? strip(*P[2].head, o.xsize) : std::string("*");
    s += fmt("\t%.2f\t%.2f\t%.2f\t%.2f\t%.2f\t%d\t%d\t%d\t%d\t%d\t%d\t%.2f\t%c\n", QM, QA, QB, QC, QT, 0, 0, 0, 0, 0, 0, 0.00, 'Y');
  }
}

// fasta_print_general for the sequence files: the FastaFormat's header, then ";uchime_ref=<score>" with --fasta_score
void print_fasta(std::string & out, const FastaFormat & f, const std::string & head, const char * seq, int64_t len, int64_t abundance,
                 const char * score, double h)
{
  std::string one;
  fasta_print_general(one, f, head, nullptr, 0, abundance, 0, -1);
  if (score != nullptr) {
    one.pop_back();
    if (one.back() != ';') { one += ';'; }
    one += fmt("%s=%.4f\n", score, h);
  }
  out += one;
  if (f.fasta_width < 1) { out.append(seq, static_cast<size_t>(len)); out += '\n'; return; }
  for (int64_t i = 0; i < len; i += f.fasta_width) {
    out.append(seq + i, static_cast<size_t>(std::min<int64_t>(f.fasta_width, len - i)));
    out += '\n';
  }
}


int check_opts(const char * caller, const char * db_path, const vsg_uchime_opts & o, const vsg_uchime_outputs & out)
{
  auto bad = [&](const std::string & m) { Error::set(std::string(caller) + ": " + m); return VSG_EINVAL; };
  if (o.command < VSG_UCHIME_REF || o.command > VSG_CHIMERAS_DENOVO) {
    return bad("command must be VSG_UCHIME_REF, _DENOVO, _2_DENOVO, _3_DENOVO or VSG_CHIMERAS_DENOVO");
  }
  if (o.command == VSG_CHIMERAS_DENOVO) {
    if (o.chimeras_parts != 0 && (o.chimeras_parts < 2 || o.chimeras_parts > MAXPARTS)) { return bad("--chimeras_parts must be in the range 2 to 100"); }
    if (o.chimeras_parents_max < 2 || o.chimeras_parents_max > MAXPARENTS) { return bad("--chimeras_parents_max must be in the range 2 to 20"); }
    if (o.chimeras_length_min < 1) { return bad("--chimeras_length_min must be at least 1"); }
    if (!(o.chimeras_diff_pct >= 0.0 && o.chimeras_diff_pct <= 50.0)) { return bad("--chimeras_diff_pct must be in the range 0.0 to 50.0"); }
    if (out.borderline != nullptr) { return bad("--borderline is not an output of --chimeras_denovo"); }
  } else if (o.chimeras_parts != 0 || o.chimeras_parents_max != 3 || o.chimeras_length_min != 10 || o.chimeras_diff_pct != 0.0) {
    return bad("the chimeras_* options belong to --chimeras_denovo only");
  }
  if (o.command == VSG_UCHIME_REF && db_path == nullptr) { return bad("--uchime_ref needs a database (--db)"); }
  if (o.command != VSG_UCHIME_REF && db_path != nullptr) { return bad("a database (--db) is read by --uchime_ref only"); }
  if (out.chimeras == nullptr && out.nonchimeras == nullptr && out.borderline == nullptr && out.uchimeout == nullptr &&
      out.uchimealns == nullptr) {
    return bad("no output file requested (--chimeras, --nonchimeras, --borderline, --uchimeout or --uchimealns)");
  }
  if (o.strand_both != 0) { return bad("only --strand plus is allowed with uchime_ref"); }
  if (o.qmask < VSG_DBMASK_NONE || o.qmask > VSG_DBMASK_DUST || o.dbmask < VSG_DBMASK_NONE || o.dbmask > VSG_DBMASK_DUST) {
    return bad("qmask / dbmask must be VSG_DBMASK_NONE, _SOFT or _DUST");
  }
  if (o.hardmask != 0 && (o.qmask == VSG_DBMASK_DUST || (o.command == VSG_UCHIME_REF && o.dbmask == VSG_DBMASK_DUST))) {
    return bad("--hardmask with --qmask dust or --dbmask dust is not offered (the device DUST upper-cases first)");
  }
  return VSG_OK;
}

double seconds(std::chrono::steady_clock::time_point t0)
{
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

// sequences as printed, indexed like a device set
struct Text {
  const char * cat;
  const int64_t * off;
  const int32_t * len;
  const std::string * head;
};

// The last steps of chimera_process_query for a list of queries: the whole query against each of its candidates (one
// vsg_align_pairs call with CIGARs), parents_kernel (parents_long_kernel for --chimeras_denovo), and eval_parents
// (eval_parents_long) on host threads.  Query qs[k] is entry qs[k] of qset (text qt), its candidates are
// cand[cfirst[k] .. cfirst[k + 1]), entries of tset (text tt).
class Finisher {
 public:
  Finisher(vsg_ctx * c, const char * caller, const vsg_uchime_opts & o, const EvalOpts & eo)
      : c_(c), caller_(caller), o_(o), eo_(eo), long_(o.command == VSG_CHIMERAS_DENOVO)
  {
    nthreads_ = static_cast<int>(std::max(1u, std::min(16u, std::thread::hardware_concurrency())));
  }
  int run(const vsg_seqset * qset, const Text & qt, const vsg_seqset * tset, const Text & tt, const std::vector<int64_t> & qs,
          const std::vector<int32_t> & cfirst, const std::vector<uint32_t> & cand, std::vector<Eval> & ev, vsg_uchime_stats & st)
  {
    int rc = VSG_OK;
    size_t const nb = qs.size(), npairs = cand.size();
    ev.assign(nb, Eval{});
    st.candidates += static_cast<int64_t>(npairs);
    if (npairs == 0) { return VSG_OK; }
    auto tp = std::chrono::steady_clock::now();
    std::vector<uint32_t> pq(npairs);
    for (size_t k = 0; k < nb; k++) {
      for (int32_t z = cfirst[k]; z < cfirst[k + 1]; z++) { pq[static_cast<size_t>(z)] = static_cast<uint32_t>(qs[k]); }
    }
    int64_t cap = 1;
    for (size_t k = 0; k < npairs; k++) { cap += qset->h_len[pq[k]] + tset->h_len[cand[k]] + 1; }
    std::vector<char> cig(static_cast<size_t>(cap));
    std::vector<int64_t> cigoff(npairs + 1, 0);
    {
      std::vector<int16_t> score(npairs);
      std::vector<uint16_t> aligned(npairs), matches(npairs), mismatches(npairs), gaps(npairs);
      if ((rc = vsg_align_pairs(c_, qset, tset, static_cast<int64_t>(npairs), pq.data(), cand.data(), score.data(), aligned.data(),
                                matches.data(), mismatches.data(), gaps.data(), nullptr, cig.data(), cap, cigoff.data())) != VSG_OK) { return rc; }
      for (size_t k = 0; k < npairs; k++) {
        if (score[k] == VSG_SCORE_SENTINEL) {
          Error::set(std::string(caller_) + ": the 16-bit aligner defers the alignment of " + qt.head[pq[k]] + " with " + tt.head[cand[k]] +
                     ": its CIGAR cannot come from the fallback callback");
          return VSG_EINVAL;
        }
      }
    }
    st.align_s += seconds(tp); tp = std::chrono::steady_clock::now();
    // parent selection, in launches whose scratch stays under SCRATCH_CAP
    std::vector<int2> par(nb, make_int2(-1, -1));
    std::vector<int4> lpar(long_ ? nb * MAXPARENTS : 0, make_int4(-1, 0, 0, 0));
    size_t const per_job = long_ ? MAXPARENTS * sizeof(int4) : sizeof(int2);
    {
      std::vector<ParentJob> jobs;
      std::vector<size_t> job_q;
      size_t used = 0;
      auto flush = [&]() -> int {
        if (jobs.empty()) { return VSG_OK; }
        int r;
        if ((r = d_jobs_.reserve(jobs.size() * sizeof(ParentJob))) != VSG_OK || (r = d_out_.reserve(jobs.size() * per_job)) != VSG_OK ||
            (r = d_scratch_.reserve(std::max<size_t>(used, 1))) != VSG_OK) { return r; }
        VSG_CUDA_OK(cudaMemcpyAsync(d_jobs_.p, jobs.data(), jobs.size() * sizeof(ParentJob), cudaMemcpyHostToDevice, c_->stream));
        if (long_) {
          parents_long_kernel<<<static_cast<unsigned>(jobs.size()), LONG_THREADS, 0, c_->stream>>>(
              qset->d, tset->d, static_cast<const ParentJob *>(d_jobs_.p), static_cast<const uint32_t *>(d_cand_.p),
              static_cast<const char *>(d_cig_.p), static_cast<const int64_t *>(d_cigoff_.p), static_cast<uint8_t *>(d_scratch_.p),
              o_.chimeras_parents_max, o_.chimeras_length_min, o_.chimeras_diff_pct, static_cast<int4 *>(d_out_.p));
        } else {
          parents_kernel<<<static_cast<unsigned>(jobs.size()), PARENT_THREADS, 0, c_->stream>>>(
              qset->d, tset->d, static_cast<const ParentJob *>(d_jobs_.p), static_cast<const uint32_t *>(d_cand_.p),
              static_cast<const char *>(d_cig_.p), static_cast<const int64_t *>(d_cigoff_.p), static_cast<uint8_t *>(d_scratch_.p),
              static_cast<int2 *>(d_out_.p));
        }
        count_launch();
        VSG_CUDA_OK(cudaGetLastError());
        if (long_) {
          std::vector<int4> h(jobs.size() * MAXPARENTS);
          VSG_CUDA_OK(cudaMemcpyAsync(h.data(), d_out_.p, h.size() * sizeof(int4), cudaMemcpyDeviceToHost, c_->stream));
          VSG_CUDA_OK(cudaStreamSynchronize(c_->stream));
          for (size_t j = 0; j < jobs.size(); j++) {
            std::copy(h.begin() + static_cast<std::ptrdiff_t>(j * MAXPARENTS), h.begin() + static_cast<std::ptrdiff_t>((j + 1) * MAXPARENTS),
                      lpar.begin() + static_cast<std::ptrdiff_t>(job_q[j] * MAXPARENTS));
          }
        } else {
          std::vector<int2> h(jobs.size());
          VSG_CUDA_OK(cudaMemcpyAsync(h.data(), d_out_.p, h.size() * sizeof(int2), cudaMemcpyDeviceToHost, c_->stream));
          VSG_CUDA_OK(cudaStreamSynchronize(c_->stream));
          for (size_t j = 0; j < jobs.size(); j++) { par[job_q[j]] = h[j]; }
        }
        jobs.clear(); job_q.clear(); used = 0;
        return VSG_OK;
      };
      if ((rc = d_cand_.reserve(npairs * sizeof(uint32_t))) != VSG_OK || (rc = d_cig_.reserve(cig.size())) != VSG_OK ||
          (rc = d_cigoff_.reserve(cigoff.size() * sizeof(int64_t))) != VSG_OK) { return rc; }
      VSG_CUDA_OK(cudaMemcpyAsync(d_cand_.p, cand.data(), npairs * sizeof(uint32_t), cudaMemcpyHostToDevice, c_->stream));
      VSG_CUDA_OK(cudaMemcpyAsync(d_cig_.p, cig.data(), cig.size(), cudaMemcpyHostToDevice, c_->stream));
      VSG_CUDA_OK(cudaMemcpyAsync(d_cigoff_.p, cigoff.data(), cigoff.size() * sizeof(int64_t), cudaMemcpyHostToDevice, c_->stream));
      for (size_t k = 0; k < nb; k++) {
        int const nc = cfirst[k + 1] - cfirst[k];
        if (nc < (long_ ? 1 : 2)) { continue; }   // two parents are needed; find_best_parents_long may take both from one candidate
        size_t const qlen = static_cast<size_t>(qset->h_len[static_cast<size_t>(qs[k])]);
        if (nc > (long_ ? ACCEPTS * parts_of(o_, static_cast<int64_t>(qlen)) : MAXCAND)) {
          Error::set(std::string(caller_) + ": more candidates than the parts of a query can accept");
          return VSG_EINVAL;
        }
        size_t const need = long_ ? static_cast<size_t>(std::min(nc, LONG_THREADS)) * (qlen + 1) * sizeof(double) + (2 * static_cast<size_t>(nc) + 1) * qlen
                                  : (2 * static_cast<size_t>(nc) + 3) * qlen;
        if (!jobs.empty() && used + need > SCRATCH_CAP && (rc = flush()) != VSG_OK) { return rc; }
        jobs.push_back(ParentJob{qs[k], static_cast<int64_t>(used), cfirst[k], nc});
        job_q.push_back(k);
        used += (need + 15) & ~static_cast<size_t>(15);
      }
      if ((rc = flush()) != VSG_OK) { return rc; }
    }
    st.parents_s += seconds(tp); tp = std::chrono::steady_clock::now();
    int const nt = static_cast<int>(std::min<int64_t>(nthreads_, std::max<int64_t>(1, static_cast<int64_t>(nb) / 64)));
    rc = run_parallel(nt, [&](int w) -> int {
      for (size_t k = static_cast<size_t>(w); k < nb; k += static_cast<size_t>(nt)) {
        if (long_) {
          finish_long(qt, tt, qs[k], cfirst[k], cand, cig, cigoff, lpar.data() + k * MAXPARENTS, ev[k]);
          continue;
        }
        int2 const p = par[k];
        if (p.x < 0 || p.y < 0) { continue; }
        size_t const q = static_cast<size_t>(qs[k]);
        Parent P[2];
        int const pp[2] = {p.x, p.y};
        for (int f = 0; f < 2; f++) {
          size_t const z = static_cast<size_t>(cfirst[k] + pp[f]);
          uint32_t const tg = cand[z];
          P[f] = Parent{tt.cat + tt.off[tg], tt.len[tg], &tt.head[tg], cig.data() + cigoff[z]};
        }
        eval_parents(qt.cat + qt.off[q], qt.len[q], qt.head[q], P, eo_, ev[k]);
      }
      return VSG_OK;
    });
    st.eval_s += seconds(tp);
    return rc;
  }

 private:
  // the parents found for a query (in the order found), sorted by start; eval_parents_long when there are two or more
  // and they cover the query
  void finish_long(const Text & qt, const Text & tt, int64_t qi, int32_t c0, const std::vector<uint32_t> & cand, const std::vector<char> & cig,
                   const std::vector<int64_t> & cigoff, const int4 * found, Eval & e) const
  {
    int4 pp[MAXPARENTS];
    int np = 0, covered = 0;
    for (int f = 0; f < MAXPARENTS && found[f].x >= 0; f++) { pp[np++] = found[f]; covered += found[f].z; }
    size_t const q = static_cast<size_t>(qi);
    if (np < 2 || covered != qt.len[q]) { return; }
    std::sort(pp, pp + np, [](const int4 & a, const int4 & b) { return a.y < b.y; });
    Parent P[MAXPARENTS];
    int starts[MAXPARENTS], lens[MAXPARENTS];
    for (int f = 0; f < np; f++) {
      size_t const z = static_cast<size_t>(c0 + pp[f].x);
      uint32_t const tg = cand[z];
      P[f] = Parent{tt.cat + tt.off[tg], tt.len[tg], &tt.head[tg], cig.data() + cigoff[z]};
      starts[f] = pp[f].y; lens[f] = pp[f].z;
    }
    eval_parents_long(qt.cat + qt.off[q], qt.len[q], qt.head[q], P, starts, lens, np, eo_, e);
  }

  static constexpr size_t SCRATCH_CAP = static_cast<size_t>(256) << 20;
  vsg_ctx * c_;
  const char * caller_;
  const vsg_uchime_opts & o_;
  EvalOpts eo_;
  bool long_;
  int nthreads_ = 1;
  DevBuf d_jobs_, d_cand_, d_cig_, d_cigoff_, d_scratch_, d_out_;
};

// The output files of chimera_thread_core's process_query, in query order
class Writer {
 public:
  Writer(const char * caller, const vsg_uchime_opts & o, const vsg_uchime_outputs & out)
      : caller_(caller), o_(o), ff_{nullptr, o.xsize != 0, o.sizeout != 0, o.fasta_width},
        score_(o.fasta_score == 0 ? nullptr : (o.command == VSG_UCHIME_REF ? "uchime_ref" : "uchime_denovo")),
        paths_{out.chimeras, out.nonchimeras, out.borderline, out.uchimeout, out.uchimealns}
  {
  }
  ~Writer() { close(); }
  int open()
  {
    for (int k = 0; k < 5; k++) {
      if (paths_[k] == nullptr) { continue; }
      if ((fh_[k] = files.open(paths_[k])) == nullptr) {
        Error::set(std::string(caller_) + ": unable to open " + paths_[k] + " for writing");
        return VSG_EINVAL;
      }
    }
    return VSG_OK;
  }
  void add(const std::string & head, const char * seq, int64_t len, int64_t size, const Eval & e, vsg_uchime_stats & st)
  {
    st.queries++;
    st.queries_abundance += size;
    if (e.status == CHIMERIC) {
      st.chimeras++; st.chimeras_abundance += size;
      if (fh_[0] != nullptr) { print_fasta(s_[0], ff_, head, seq, len, size, score_, e.h); }
    } else if (e.status == SUSPICIOUS) {
      st.borderline++; st.borderline_abundance += size;
      if (fh_[2] != nullptr) { print_fasta(s_[2], ff_, head, seq, len, size, score_, e.h); }
    } else {
      st.nonchimeras++; st.nonchimeras_abundance += size;
      if (fh_[1] != nullptr) { print_fasta(s_[1], ff_, head, seq, len, size, score_, e.h); }
    }
    if (fh_[3] != nullptr) {
      if (e.status < LOW_SCORE && o_.command != VSG_CHIMERAS_DENOVO) {   // --tabbedout has rows for chimeras only
        s_[3] += fmt("%.4f\t", e.h) + strip(head, o_.xsize != 0);
        s_[3] += o_.uchimeout5 != 0 ? "\t*\t*\t*\t*\t*\t*\t*\t0\t0\t0\t0\t0\t0\t*\tN\n" : "\t*\t*\t*\t*\t*\t*\t*\t*\t0\t0\t0\t0\t0\t0\t*\tN\n";
      } else {
        s_[3] += e.uchimeout;
      }
    }
    if (fh_[4] != nullptr) { s_[4] += e.uchimealns; }
  }
  int flush()
  {
    for (int k = 0; k < 5; k++) {
      if (fh_[k] != nullptr && !s_[k].empty() && std::fwrite(s_[k].data(), 1, s_[k].size(), fh_[k]) != s_[k].size()) {
        Error::set(std::string(caller_) + ": unable to write to " + paths_[k]);
        return VSG_EINVAL;
      }
      s_[k].clear();
    }
    return VSG_OK;
  }
  bool close()
  {
    bool ok = true;
    for (auto & f : fh_) { if (f != nullptr) { ok = std::fclose(f) == 0 && ok; f = nullptr; } }
    return ok;
  }
  OutFiles files;

 private:
  const char * caller_;
  const vsg_uchime_opts & o_;
  FastaFormat ff_;
  const char * score_;
  const char * paths_[5];
  std::FILE * fh_[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  std::string s_[5];
};

// the `parts` pieces of a query (partition_query) as [offset, length) views of its text; none for a query shorter than
// its part count
void pieces_of(int64_t off, int len, int parts, std::vector<int64_t> & poff, std::vector<int32_t> & plen)
{
  if (len < parts) { return; }
  int rest = len;
  for (int p = 0; p < parts; p++) {
    int const l = (rest + (parts - p - 1)) / (parts - p);
    poff.push_back(off); plen.push_back(l);
    off += l; rest -= l;
  }
}

// --uchime_ref over batches of queries (chimera.cpp:2488-2522 and the worker loop with one thread)
int uchime_ref(vsg_ctx * ctx, const char * caller, const char * input_path, const char * db_path, const vsg_uchime_opts & o,
               const EvalOpts & eo, Writer & wr, vsg_uchime_stats & st)
{
  auto const t0 = std::chrono::steady_clock::now();
  // the queries: FASTA only (fasta_open), every record kept, case as read (chrmap_no_change), never DUST-masked
  {
    std::FILE * f = std::fopen(input_path, "rb");
    if (f == nullptr) { Error::set(std::string(caller) + ": cannot open " + input_path); return VSG_EINVAL; }
    int const first = std::fgetc(f);
    std::fclose(f);
    if (first == '@') { Error::set(std::string(caller) + ": --uchime_ref reads FASTA queries, not FASTQ (" + input_path + ")"); return VSG_EINVAL; }
  }
  FastxFile qf;
  int rc = read_fastx_file(caller, input_path, o.notrunclabels != 0, 0, INT64_MAX, qf);
  if (rc != VSG_OK) { return rc; }
  int64_t const nq = static_cast<int64_t>(qf.head.size());
  std::vector<int64_t> qsize(static_cast<size_t>(nq));
  for (int64_t i = 0; i < nq; i++) {
    std::string err;
    if (!abundance_of(qf.head[static_cast<size_t>(i)], qsize[static_cast<size_t>(i)], err)) {
      Error::set(std::string(caller) + ": " + err + " (" + qf.head[static_cast<size_t>(i)] + ")");
      return VSG_EINVAL;
    }
  }
  // the database and its index (chimera.cpp:2488-2511)
  SearchDb db;
  vsg_index * ixraw = nullptr;
  if (vsg_udb_detect(db_path) == 1) {
    vsg_udb * uraw = nullptr;
    if ((rc = vsg_udb_open(db_path, &uraw)) != VSG_OK) { return rc; }
    std::unique_ptr<vsg_udb, void (*)(vsg_udb *)> udb(uraw, vsg_udb_close);
    int64_t const n = static_cast<int64_t>(udb->len.size());
    db.file.cat = udb->cat;
    db.file.off = udb->off;
    db.file.len = udb->len;
    db.file.head.resize(static_cast<size_t>(n));
    for (int64_t i = 0; i < n; i++) { db.file.head[static_cast<size_t>(i)] = vsg_udb_header(udb.get(), i); }
    if ((rc = search_db_labels(caller, o.self != 0, db)) != VSG_OK) { return rc; }
    vsg_seqset * setraw = nullptr;
    if ((rc = vsg_udb_load(ctx, udb.get(), &setraw, &ixraw, nullptr)) != VSG_OK) { return rc; }
    db.set.reset(setraw);
  } else {
    if ((rc = search_db_read(ctx, caller, db_path, o.notrunclabels != 0, o.minseqlength, o.maxseqlength, o.dbmask, o.hardmask != 0,
                             o.dbmask == VSG_DBMASK_DUST, o.self != 0, db)) != VSG_OK) { return rc; }
    if ((rc = vsg_index_create(ctx, db.set.get(), 8, o.dbmask != VSG_DBMASK_NONE ? 1 : 0, &ixraw)) != VSG_OK) { return rc; }
  }
  std::unique_ptr<vsg_index, void (*)(vsg_index *)> ix(ixraw, vsg_index_destroy);
  st.db_sequences = static_cast<int64_t>(db.heads.size());
  std::vector<int64_t> qlabel;
  if (o.self != 0) {
    qlabel.resize(static_cast<size_t>(nq));
    for (int64_t i = 0; i < nq; i++) {
      auto const it = db.label_ids.find(qf.head[static_cast<size_t>(i)]);
      qlabel[static_cast<size_t>(i)] = it == db.label_ids.end() ? -1 : it->second;
    }
  }
  st.parse_s += seconds(t0);
  if ((rc = wr.open()) != VSG_OK) { return rc; }

  // the detection parameters of the part searches
  vsg_search_opts so;
  vsg_search_opts_default(&so);
  so.id = CHIMERA_ID;
  so.weak_id = CHIMERA_ID;
  so.maxaccepts = ACCEPTS;
  so.maxrejects = REJECTS;
  so.wordlength = index_wordlength(ix.get());
  so.mask_lower = o.qmask != VSG_DBMASK_NONE ? 1 : 0;
  so.self = o.self;
  so.selfid = o.selfid;
  so.target_sizes = db.size.data();
  if (o.self != 0) { so.target_labels = db.label_id.data(); }

  Finisher fin(ctx, caller, o, eo);
  Text const tt{db.file.cat.data(), db.file.off.data(), db.file.len.data(), db.file.head.data()};
  int64_t const B = o.batch_queries < 1 ? 8192 : o.batch_queries;
  std::vector<vsg_search_result> rows;
  std::vector<int64_t> first;
  for (int64_t b0 = 0; b0 < nq; b0 += B) {
    int64_t const nb = std::min(B, nq - b0);
    auto tp = std::chrono::steady_clock::now();
    std::vector<int64_t> poff, psize, plabel;
    std::vector<int32_t> plen;
    std::vector<int64_t> pfirst(static_cast<size_t>(nb) + 1, 0);
    for (int64_t i = 0; i < nb; i++) {
      size_t const q = static_cast<size_t>(b0 + i);
      pieces_of(qf.off[q], qf.len[q], PARTS, poff, plen);
      while (psize.size() < plen.size()) { psize.push_back(qsize[q]); if (o.self != 0) { plabel.push_back(qlabel[q]); } }
      pfirst[static_cast<size_t>(i) + 1] = static_cast<int64_t>(plen.size());
    }
    int64_t const np = static_cast<int64_t>(plen.size());
    SeqsetPtr pieces, qset;
    vsg_seqset * raw = nullptr;
    if ((rc = vsg_seqset_create(ctx, qf.cat.data(), poff.data(), plen.data(), np, 1, &raw)) != VSG_OK) { return rc; }
    pieces.reset(raw);
    if ((rc = vsg_seqset_create(ctx, qf.cat.data(), qf.off.data() + b0, qf.len.data() + b0, nb, 1, &raw)) != VSG_OK) { return rc; }
    qset.reset(raw);
    vsg_search_opts po = so;
    po.query_sizes = psize.data();
    if (o.self != 0) { po.query_labels = plabel.data(); }
    rows.clear(); first.assign(static_cast<size_t>(np) + 1, 0);
    if (np > 0) {
      int64_t work[4] = {0, 0, 0, 0};
      if ((rc = search_hits_host(ctx, ix.get(), db.set.get(), pieces.get(), 0, np, &po, 0, rows, first, work)) != VSG_OK) { return rc; }
      st.part_pairs += work[2];
    }
    st.search_s += seconds(tp);
    // the candidates: the accepted hits of the parts in order, without duplicates
    std::vector<int32_t> cfirst(static_cast<size_t>(nb) + 1, 0);
    std::vector<uint32_t> cand;
    std::vector<int64_t> qs(static_cast<size_t>(nb));
    for (int64_t i = 0; i < nb; i++) {
      qs[static_cast<size_t>(i)] = i;
      size_t const c0 = cand.size();
      for (int64_t p = pfirst[static_cast<size_t>(i)]; p < pfirst[static_cast<size_t>(i) + 1]; p++) {
        for (int64_t r = first[static_cast<size_t>(p)]; r < first[static_cast<size_t>(p) + 1]; r++) {
          if (rows[static_cast<size_t>(r)].accepted == 0) { continue; }
          uint32_t const tg = static_cast<uint32_t>(rows[static_cast<size_t>(r)].target);
          if (std::find(cand.begin() + static_cast<std::ptrdiff_t>(c0), cand.end(), tg) == cand.end()) { cand.push_back(tg); }
        }
      }
      cfirst[static_cast<size_t>(i) + 1] = static_cast<int32_t>(cand.size());
    }
    Text const qt{qf.cat.data(), qf.off.data() + b0, qf.len.data() + b0, qf.head.data() + b0};
    std::vector<Eval> ev;
    if ((rc = fin.run(qset.get(), qt, db.set.get(), tt, qs, cfirst, cand, ev, st)) != VSG_OK) { return rc; }
    tp = std::chrono::steady_clock::now();
    for (int64_t i = 0; i < nb; i++) {
      size_t const q = static_cast<size_t>(b0 + i);
      wr.add(qf.head[q], qf.cat.data() + qf.off[q], qf.len[q], qsize[q], ev[static_cast<size_t>(i)], st);
    }
    if ((rc = wr.flush()) != VSG_OK) { return rc; }
    st.write_s += seconds(tp);
  }
  return VSG_OK;
}

// ---- de novo ----------------------------------------------------------------------------------------------------------

constexpr int KMER = 8;                                     // the word length of the de novo index
constexpr int KMER_WORDS = (1 << (2 * KMER)) / 32;          // a 4^8-bit set in 32-bit words
constexpr int KMER_THREADS = 256;

// the 2-bit code of a symbol in a k-mer, or -1 where unique_count (core/unique.cpp) breaks the window: an ambiguous
// symbol, or a lower-case one under --qmask soft / dust
__device__ inline int kmer_code(unsigned char ch, bool mask_lower)
{
  if (mask_lower && ch >= 'a' && ch <= 'z') { return -1; }
  switch (ch | 0x20) {
    case 'a': return 0;
    case 'c': return 1;
    case 'g': return 2;
    case 't': case 'u': return 3;
    default: return -1;
  }
}

// the k-mer that ends at s[p] (p >= KMER - 1), or -1
__device__ inline int kmer_at(const char * s, int p, bool mask_lower)
{
  int v = 0;
  for (int z = p - KMER + 1; z <= p; z++) {
    int const c = kmer_code(static_cast<unsigned char>(s[z]), mask_lower);
    if (c < 0) { return -1; }
    v = (v << 2) | c;
  }
  return v;
}

// the k-mer set of every member of a band, one CTA per member: bits[m] is a 4^8-bit set
__global__ void __launch_bounds__(KMER_THREADS) member_kmers_kernel(const char * __restrict__ txt, const int64_t * __restrict__ off,
                                                                    const int32_t * __restrict__ len, bool mask_lower, uint32_t * __restrict__ bits)
{
  char const * const s = txt + off[blockIdx.x];
  int const L = len[blockIdx.x];
  uint32_t * const b = bits + static_cast<size_t>(blockIdx.x) * KMER_WORDS;
  for (int w = threadIdx.x; w < KMER_WORDS; w += blockDim.x) { b[w] = 0; }
  __syncthreads();
  for (int p = KMER - 1 + threadIdx.x; p < L; p += blockDim.x) {
    int const v = kmer_at(s, p, mask_lower);
    if (v >= 0) { atomicOr(&b[v >> 5], 1u << (v & 31)); }
  }
}

// The shared k-mer counts of the parts of a band with its earlier members, one CTA per part: the part's distinct k-mers
// (a set in shared memory; each new one is listed at kl[klo[p] ..]), then, a warp per member m < member[p], how many of
// them are in m's set.  counts[row[p] + m] = that count; nk[p] = the part's distinct k-mers.
__global__ void __launch_bounds__(KMER_THREADS) part_counts_kernel(const char * __restrict__ txt, const int64_t * __restrict__ poff,
                                                                   const int32_t * __restrict__ plen, const int32_t * __restrict__ member,
                                                                   const int64_t * __restrict__ row, const int64_t * __restrict__ klo, bool mask_lower,
                                                                   const uint32_t * __restrict__ bits, uint32_t * __restrict__ kl,
                                                                   uint32_t * __restrict__ counts, int32_t * __restrict__ nk)
{
  __shared__ uint32_t seen[KMER_WORDS];
  __shared__ int listed;
  int const p = blockIdx.x;
  char const * const s = txt + poff[p];
  int const L = plen[p];
  uint32_t * const mine = kl + klo[p];
  for (int w = threadIdx.x; w < KMER_WORDS; w += blockDim.x) { seen[w] = 0; }
  if (threadIdx.x == 0) { listed = 0; }
  __syncthreads();
  for (int x = KMER - 1 + threadIdx.x; x < L; x += blockDim.x) {
    int const v = kmer_at(s, x, mask_lower);
    if (v < 0) { continue; }
    uint32_t const bit = 1u << (v & 31);
    if ((atomicOr(&seen[v >> 5], bit) & bit) == 0) { mine[atomicAdd(&listed, 1)] = static_cast<uint32_t>(v); }
  }
  __syncthreads();
  int const n = listed;
  if (threadIdx.x == 0) { nk[p] = n; }
  int const lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (int m = warp; m < member[p]; m += nwarps) {
    uint32_t const * const b = bits + static_cast<size_t>(m) * KMER_WORDS;
    int c = 0;
    for (int x = lane; x < n; x += 32) { uint32_t const v = mine[x]; c += static_cast<int>((b[v >> 5] >> (v & 31)) & 1u); }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) { c += __shfl_xor_sync(0xffffffffu, c, d); }
    if (lane == 0) { counts[row[p] + m] = static_cast<uint32_t>(c); }
  }
}

// The k-mers the parts of a band share with each earlier member of the band, counted on the device (member_kmers_kernel,
// part_counts_kernel).  The band's text is the whole sorted input, uploaded once.
class BandKmers {
 public:
  int upload(vsg_ctx * c, const std::vector<char> & cat)
  {
    int rc;
    if ((rc = txt_.reserve(cat.size())) != VSG_OK) { return rc; }
    VSG_CUDA_OK(cudaMemcpyAsync(txt_.p, cat.data(), cat.size(), cudaMemcpyHostToDevice, c->stream));
    return VSG_OK;
  }
  // members [moff, mlen) of the band; parts [poff, plen) of member pmember (0-based in the band).  On return
  // counts[row[p] + m] holds part p's shared k-mers with member m < pmember[p], and nk[p] its distinct k-mers.
  int run(vsg_ctx * c, bool mask_lower, const std::vector<int64_t> & moff, const std::vector<int32_t> & mlen, const std::vector<int64_t> & poff,
          const std::vector<int32_t> & plen, const std::vector<int32_t> & pmember, std::vector<int64_t> & row, std::vector<uint32_t> & counts,
          std::vector<int32_t> & nk)
  {
    size_t const nb = moff.size(), np = poff.size();
    row.assign(np + 1, 0);
    std::vector<int64_t> klo(np + 1, 0);
    for (size_t p = 0; p < np; p++) { row[p + 1] = row[p] + pmember[p]; klo[p + 1] = klo[p] + plen[p]; }
    counts.assign(static_cast<size_t>(row[np]), 0);
    nk.assign(np, 0);
    if (np == 0) { return VSG_OK; }
    int rc;
    if ((rc = moff_.reserve(nb * sizeof(int64_t))) != VSG_OK || (rc = mlen_.reserve(nb * sizeof(int32_t))) != VSG_OK ||
        (rc = bits_.reserve(nb * KMER_WORDS * sizeof(uint32_t))) != VSG_OK || (rc = poff_.reserve(np * sizeof(int64_t))) != VSG_OK ||
        (rc = plen_.reserve(np * sizeof(int32_t))) != VSG_OK || (rc = pmem_.reserve(np * sizeof(int32_t))) != VSG_OK ||
        (rc = row_.reserve(np * sizeof(int64_t))) != VSG_OK || (rc = klo_.reserve(np * sizeof(int64_t))) != VSG_OK ||
        (rc = kl_.reserve(std::max<size_t>(1, static_cast<size_t>(klo[np])) * sizeof(uint32_t))) != VSG_OK ||
        (rc = counts_.reserve(std::max<size_t>(1, counts.size()) * sizeof(uint32_t))) != VSG_OK ||
        (rc = nk_.reserve(np * sizeof(int32_t))) != VSG_OK) { return rc; }
    VSG_CUDA_OK(cudaMemcpyAsync(moff_.p, moff.data(), nb * sizeof(int64_t), cudaMemcpyHostToDevice, c->stream));
    VSG_CUDA_OK(cudaMemcpyAsync(mlen_.p, mlen.data(), nb * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    VSG_CUDA_OK(cudaMemcpyAsync(poff_.p, poff.data(), np * sizeof(int64_t), cudaMemcpyHostToDevice, c->stream));
    VSG_CUDA_OK(cudaMemcpyAsync(plen_.p, plen.data(), np * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    VSG_CUDA_OK(cudaMemcpyAsync(pmem_.p, pmember.data(), np * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    VSG_CUDA_OK(cudaMemcpyAsync(row_.p, row.data(), np * sizeof(int64_t), cudaMemcpyHostToDevice, c->stream));
    VSG_CUDA_OK(cudaMemcpyAsync(klo_.p, klo.data(), np * sizeof(int64_t), cudaMemcpyHostToDevice, c->stream));
    member_kmers_kernel<<<static_cast<unsigned>(nb), KMER_THREADS, 0, c->stream>>>(static_cast<const char *>(txt_.p), static_cast<const int64_t *>(moff_.p),
                                                                                  static_cast<const int32_t *>(mlen_.p), mask_lower,
                                                                                  static_cast<uint32_t *>(bits_.p));
    count_launch();
    VSG_CUDA_OK(cudaGetLastError());
    part_counts_kernel<<<static_cast<unsigned>(np), KMER_THREADS, 0, c->stream>>>(
        static_cast<const char *>(txt_.p), static_cast<const int64_t *>(poff_.p), static_cast<const int32_t *>(plen_.p),
        static_cast<const int32_t *>(pmem_.p), static_cast<const int64_t *>(row_.p), static_cast<const int64_t *>(klo_.p), mask_lower,
        static_cast<const uint32_t *>(bits_.p), static_cast<uint32_t *>(kl_.p), static_cast<uint32_t *>(counts_.p), static_cast<int32_t *>(nk_.p));
    count_launch();
    VSG_CUDA_OK(cudaGetLastError());
    if (!counts.empty()) {
      VSG_CUDA_OK(cudaMemcpyAsync(counts.data(), counts_.p, counts.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    }
    VSG_CUDA_OK(cudaMemcpyAsync(nk.data(), nk_.p, np * sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
    VSG_CUDA_OK(cudaStreamSynchronize(c->stream));
    return VSG_OK;
  }

 ~BandKmers()
  {
    for (DevBuf * b : {&txt_, &moff_, &mlen_, &bits_, &poff_, &plen_, &pmem_, &row_, &klo_, &kl_, &counts_, &nk_}) { b->release(); }
  }

 private:
  DevBuf txt_, moff_, mlen_, bits_, poff_, plen_, pmem_, row_, klo_, kl_, counts_, nk_;
};

// one entry of a part's candidate heap: target, shared k-mers, target length; whether search_acceptable_unaligned passes
// and, for a static entry that passes, the aligned hit and whether search_acceptable_aligned accepts it
struct Entry {
  uint32_t t, count;
  int32_t len;
  bool ok, accepted, aligned;
  Hit hit;
};

// search_onequery's candidate loop with align_delayed (searchcore.cpp:740-957) over a heap already in pop order: the
// accepted entries, best first by hit_compare_byid (search_joinhits)
void replay(const std::vector<Entry> & L, std::vector<const Hit *> & acc)
{
  acc.clear();
  int accepts = 0, rejects = 0, finalized = 0, delayed = 0, n = 0;
  int const nl = static_cast<int>(L.size());
  auto process = [&](int from, int to) {
    for (int x = from; x < to; x++) {
      if (rejects < REJECTS && accepts < ACCEPTS) {
        Entry const & e = L[static_cast<size_t>(x)];
        if (!e.ok || !e.accepted) { rejects++; } else { accepts++; acc.push_back(&e.hit); }
      }
    }
  };
  while (finalized + delayed < ACCEPTS + REJECTS - 1 && rejects < REJECTS && accepts < ACCEPTS && n < nl) {
    if (L[static_cast<size_t>(n)].ok) { delayed++; }
    n++;
    if (delayed == MAXDELAYED) { process(finalized, n); finalized = n; delayed = 0; }
  }
  if (delayed > 0) { process(finalized, n); }
  std::stable_sort(acc.begin(), acc.end(), [](const Hit * a, const Hit * b) { return hit_less(*a, *b); });
}

// the candidates of a query from its parts' heaps: the accepted hits of each part in order, without duplicates
void candidates_of(const std::vector<std::vector<Entry>> & heaps, std::vector<uint32_t> & cand)
{
  cand.clear();
  std::vector<const Hit *> acc;
  for (auto const & L : heaps) {
    replay(L, acc);
    for (const Hit * h : acc) {
      uint32_t const t = static_cast<uint32_t>(h->target);
      if (std::find(cand.begin(), cand.end(), t) == cand.end()) { cand.push_back(t); }
    }
  }
}

// --uchime_denovo / --uchime2_denovo / --uchime3_denovo / --chimeras_denovo (chimera.cpp:2526-2559 and the single
// worker): the input read as db.read keeps it, DUST-masked (or hardmasked), sorted by abundance, then cut into bands.
// For the uchime commands a band holds sequences none of which can be a parent of another (a sequence i passes the size
// test of a later j only when abundance_ratio_cmp(a_j, 1/abskew, a_i) <= 0); for --chimeras_denovo it is band_cap
// consecutive reads.  Per band:
//   1. speculative pass: the members' pieces are ranked against the non-chimeras indexed before the band (heap of 20);
//      the k-mers each piece shares with every earlier member are counted on the device (BandKmers), and for
//      --chimeras_denovo the members that reach minwordmatches are merged into the heaps as if all were non-chimeric.
//      Every entry that passes search_acceptable_unaligned is aligned in one call, the candidate loop is replayed on
//      the host, and the candidates of every member are finished together (Finisher);
//   2. serial pass, in order: the non-chimeric members before j are in the reference's index when j is searched.  j's
//      heaps are rebuilt from the static entries and those members only (for the uchime commands the size test rejects
//      them before alignment); an entry the speculative heap did not hold is aligned, the loop is replayed, and a
//      changed candidate list is finished again for j alone (recomputed);
//   3. the band's non-chimeras are appended to the device index.
int uchime_denovo(vsg_ctx * ctx, const char * caller, const char * input_path, const vsg_uchime_opts & o, const EvalOpts & eo,
                  Writer & wr, vsg_uchime_stats & st)
{
  auto const t0 = std::chrono::steady_clock::now();
  FastxFile f;
  int rc = read_fastx_file(caller, input_path, o.notrunclabels != 0, o.minseqlength, o.maxseqlength, f);
  if (rc != VSG_OK) { return rc; }
  size_t const n = f.head.size();
  if (n > 0x7fffffffULL) { Error::set(std::string(caller) + ": too many sequences"); return VSG_EINVAL; }
  std::vector<int64_t> fsize(n);
  for (size_t i = 0; i < n; i++) {
    std::string err;
    if (!abundance_of(f.head[i], fsize[i], err)) { Error::set(std::string(caller) + ": " + err + " (" + f.head[i] + ")"); return VSG_EINVAL; }
  }
  // sortbyabundance (db.cpp:471-486): abundance descending, then label, then input order
  std::vector<size_t> perm(n);
  for (size_t i = 0; i < n; i++) { perm[i] = i; }
  std::sort(perm.begin(), perm.end(), [&](size_t a, size_t b) {
    if (fsize[a] != fsize[b]) { return fsize[a] > fsize[b]; }
    int const c = std::strcmp(f.head[a].c_str(), f.head[b].c_str());
    if (c != 0) { return c < 0; }
    return a < b;
  });
  std::vector<char> cat;
  std::vector<int64_t> off(n), size(n);
  std::vector<int32_t> len(n);
  std::vector<std::string> head(n);
  for (size_t i = 0; i < n; i++) {
    size_t const s = perm[i];
    off[i] = static_cast<int64_t>(cat.size());
    len[i] = f.len[s];
    cat.insert(cat.end(), f.cat.begin() + f.off[s], f.cat.begin() + f.off[s] + f.len[s]);
    head[i] = std::move(f.head[s]);
    size[i] = fsize[s];
  }
  cat.push_back('\0');
  f = FastxFile{};
  if (o.qmask == VSG_DBMASK_SOFT && o.hardmask != 0) { hardmask(cat); }
  SeqsetPtr set;
  vsg_seqset * raw = nullptr;
  if ((rc = vsg_seqset_create(ctx, cat.data(), off.data(), len.data(), static_cast<int64_t>(n), 1, &raw)) != VSG_OK) { return rc; }
  set.reset(raw);
  if (o.qmask == VSG_DBMASK_DUST && (rc = dust_case(ctx, set.get(), cat)) != VSG_OK) { return rc; }
  // --self: label identities
  std::vector<int64_t> label(n);
  {
    std::unordered_map<std::string, int64_t> ids;
    for (size_t i = 0; i < n; i++) { label[i] = ids.emplace(head[i], static_cast<int64_t>(i)).first->second; }
  }
  bool const mask_lower = o.qmask != VSG_DBMASK_NONE;
  int const k = KMER;
  CIndex * cixraw = nullptr;
  if ((rc = cindex_create(ctx, set.get(), k, mask_lower ? 1 : 0, &cixraw)) != VSG_OK) { return rc; }
  std::unique_ptr<CIndex, void (*)(CIndex *)> cix(cixraw, cindex_destroy);
  st.parse_s += seconds(t0);
  if ((rc = wr.open()) != VSG_OK) { return rc; }

  // the detection parameters of de novo mode (chimera_detection_parameters): self, selfid and --maxsizeratio 1/abskew
  vsg_search_opts so;
  vsg_search_opts_default(&so);
  so.id = CHIMERA_ID;
  so.weak_id = CHIMERA_ID;
  so.maxaccepts = ACCEPTS;
  so.maxrejects = REJECTS;
  so.wordlength = k;
  so.self = 1;
  so.selfid = 1;
  so.maxsizeratio = 1.0 / o.abskew;
  int const minwordmatches = minwordmatches_defaults[k];
  auto unaligned_ok = [&](size_t j, int64_t poff, int plen, uint32_t t) {
    bool selfid_fails = plen == len[t];
    if (selfid_fails) {
      Maps const & M = maps();
      for (int z = 0; z < plen && selfid_fails; z++) {
        selfid_fails = M.code[static_cast<unsigned char>(cat[static_cast<size_t>(poff + z)])] ==
                       M.code[static_cast<unsigned char>(cat[static_cast<size_t>(off[t] + z)])];
      }
    }
    return acceptable_unaligned(so, plen, len[t], size[j], size[t], label[j] == label[t], selfid_fails ? 4u : 0u);
  };

  Finisher fin(ctx, caller, o, eo);
  Text const txt{cat.data(), off.data(), len.data(), head.data()};
  int64_t const cap = o.band_cap < 1 ? 1024 : o.band_cap;
  double const ratio = 1.0 / o.abskew;
  bool const inband = o.command == VSG_CHIMERAS_DENOVO;   // earlier members of a band may be parents of later ones
  const std::vector<uint32_t> & dense = cindex_seqnos(cix.get());
  auto const heap_order = [](const Entry & x, const Entry & y) {   // the ranker's order
    if (x.count != y.count) { return x.count > y.count; }
    if (x.len != y.len) { return x.len < y.len; }
    return x.t < y.t;
  };
  BandKmers bk;
  if ((rc = bk.upload(ctx, cat)) != VSG_OK) { return rc; }
  std::vector<uint32_t> hs, hc, counts;
  std::vector<int32_t> hn, nk;
  std::vector<int64_t> row;
  PairResults a;
  for (size_t b0 = 0; b0 < n;) {
    auto tp = std::chrono::steady_clock::now();
    size_t b1 = b0 + 1;
    if (inband) {
      b1 = std::min(n, b0 + static_cast<size_t>(cap));
    } else {
      while (b1 < n && static_cast<int64_t>(b1 - b0) < cap && size_ratio_sign(size[b1], ratio, size[b0]) > 0) { b1++; }
    }
    size_t const nb = b1 - b0;
    st.bands++;
    // 1. the speculative pass
    std::vector<int64_t> poff, moff(nb);
    std::vector<int32_t> plen, pmember, mlen(nb);
    std::vector<size_t> pfirst(nb + 1, 0), powner;
    for (size_t i = 0; i < nb; i++) {
      pieces_of(off[b0 + i], len[b0 + i], parts_of(o, len[b0 + i]), poff, plen);
      while (powner.size() < plen.size()) { powner.push_back(b0 + i); pmember.push_back(static_cast<int32_t>(i)); }
      pfirst[i + 1] = plen.size();
      moff[i] = off[b0 + i]; mlen[i] = len[b0 + i];
    }
    size_t const np = plen.size();
    // per part: the static entries (ranked against the index), the earlier members that share enough k-mers with it,
    // and the speculative heap (the static entries, and for --chimeras_denovo every such member, cut to 20)
    std::vector<std::vector<Entry>> stat(np), mem(np), heaps(np);
    SeqsetPtr pset;
    // aligns the entries es[x] of parts ep[x] with their targets
    auto align_entries = [&](const std::vector<size_t> & ep, const std::vector<Entry *> & es) -> int {
      if (es.empty()) { return VSG_OK; }
      std::vector<uint32_t> pq(ep.size()), pt(ep.size());
      for (size_t x = 0; x < ep.size(); x++) { pq[x] = static_cast<uint32_t>(ep[x]); pt[x] = es[x]->t; }
      a.resize(pq.size());
      int r;
      if ((r = align_into(ctx, pset.get(), set.get(), pq.size(), pq.data(), pt.data(), a, 0)) != VSG_OK) { return r; }
      st.part_pairs += static_cast<int64_t>(pq.size());
      for (size_t x = 0; x < pq.size(); x++) {
        Entry & e = *es[x];
        size_t const p = ep[x];
        std::memset(&e.hit, 0, sizeof(Hit));
        e.hit.target = static_cast<int>(e.t);
        if ((r = fill_hit(e.hit, a, x, plen[p], e.len, 2, *ctx, static_cast<int64_t>(powner[p]), 0, caller)) != VSG_OK) { return r; }
        e.accepted = acceptable_aligned(e.hit, CHIMERA_ID, CHIMERA_ID, so, plen[p], e.len, size[powner[p]], size[e.t]);
        e.aligned = true;
      }
      return VSG_OK;
    };
    if (np > 0) {
      if ((rc = vsg_seqset_create(ctx, cat.data(), poff.data(), plen.data(), static_cast<int64_t>(np), 1, &raw)) != VSG_OK) { return rc; }
      pset.reset(raw);
      hs.resize(np * 20); hc.resize(np * 20); hn.resize(np);
      RankTop rt;
      if ((rc = cindex_rank_enqueue(ctx, cix.get(), pset.get(), 0, static_cast<int64_t>(np), minwordmatches, 20, rt)) != VSG_OK ||
          (rc = rank_download(ctx, rt, static_cast<int64_t>(np), 20, hs.data(), hc.data(), hn.data(), caller)) != VSG_OK) { return rc; }
      for (size_t p = 0; p < np; p++) {
        for (int z = 0; z < hn[p]; z++) {
          uint32_t const t = dense[hs[p * 20 + static_cast<size_t>(z)]];
          Entry e{};
          e.t = t; e.count = hc[p * 20 + static_cast<size_t>(z)]; e.len = len[t];
          e.ok = unaligned_ok(powner[p], poff[p], plen[p], t);
          stat[p].push_back(e);
        }
      }
      if (nb > 1) {
        if ((rc = bk.run(ctx, mask_lower, moff, mlen, poff, plen, pmember, row, counts, nk)) != VSG_OK) { return rc; }
        for (size_t p = 0; p < np; p++) {
          unsigned const minmatches = std::min<unsigned>(static_cast<unsigned>(minwordmatches), static_cast<unsigned>(nk[p]));
          for (int32_t m = 0; m < pmember[p]; m++) {
            unsigned const shared = counts[static_cast<size_t>(row[p] + m)];
            if (shared < minmatches) { continue; }
            Entry e{};
            e.t = static_cast<uint32_t>(b0 + static_cast<size_t>(m)); e.count = shared; e.len = len[e.t];
            e.ok = unaligned_ok(powner[p], poff[p], plen[p], e.t);
            if (e.ok && !inband) {   // the abundance band's size test rejects every member for a later one
              Error::set(std::string(caller) + ": internal error: a member of an abundance band passes the size test of a later one");
              return VSG_EINVAL;
            }
            mem[p].push_back(e);
          }
        }
      }
      std::vector<size_t> ep;
      std::vector<Entry *> es;
      for (size_t p = 0; p < np; p++) {
        heaps[p] = stat[p];
        if (inband && !mem[p].empty()) {
          heaps[p].insert(heaps[p].end(), mem[p].begin(), mem[p].end());
          std::stable_sort(heaps[p].begin(), heaps[p].end(), heap_order);
          if (heaps[p].size() > 20) { heaps[p].resize(20); }
        }
      }
      for (size_t p = 0; p < np; p++) {
        for (Entry & e : heaps[p]) { if (e.ok) { ep.push_back(p); es.push_back(&e); } }
      }
      if ((rc = align_entries(ep, es)) != VSG_OK) { return rc; }
    }
    st.search_s += seconds(tp);
    std::vector<int32_t> cfirst(nb + 1, 0);
    std::vector<uint32_t> cand, c1;
    std::vector<int64_t> qs(nb);
    std::vector<std::vector<uint32_t>> spec(nb);
    for (size_t i = 0; i < nb; i++) {
      qs[i] = static_cast<int64_t>(b0 + i);
      std::vector<std::vector<Entry>> hp(heaps.begin() + static_cast<std::ptrdiff_t>(pfirst[i]), heaps.begin() + static_cast<std::ptrdiff_t>(pfirst[i + 1]));
      candidates_of(hp, spec[i]);
      cand.insert(cand.end(), spec[i].begin(), spec[i].end());
      cfirst[i + 1] = static_cast<int32_t>(cand.size());
    }
    std::vector<Eval> ev;
    if ((rc = fin.run(set.get(), txt, set.get(), txt, qs, cfirst, cand, ev, st)) != VSG_OK) { return rc; }
    // 2. the serial pass: each member's heaps rebuilt from the static entries and the members before it that really are
    //    non-chimeric; an entry the speculative heap did not hold is aligned now, and a changed candidate list is
    //    finished again
    tp = std::chrono::steady_clock::now();
    std::vector<char> nonchim(nb, 0);
    std::vector<uint32_t> appended;
    for (size_t i = 0; i < nb; i++) {
      size_t const j = b0 + i;
      bool any = false;
      for (size_t p = pfirst[i]; p < pfirst[i + 1] && !any; p++) { any = !mem[p].empty(); }
      if (any) {
        std::vector<std::vector<Entry>> hp;
        std::vector<size_t> ep;
        std::vector<Entry *> es;
        for (size_t p = pfirst[i]; p < pfirst[i + 1]; p++) {
          std::vector<Entry> L = stat[p];
          for (Entry const & e : mem[p]) { if (nonchim[e.t - b0] != 0) { L.push_back(e); } }
          std::stable_sort(L.begin(), L.end(), heap_order);
          if (L.size() > 20) { L.resize(20); }
          hp.push_back(std::move(L));
        }
        for (size_t x = 0; x < hp.size(); x++) {
          size_t const p = pfirst[i] + x;
          for (Entry & e : hp[x]) {
            if (!e.ok) { continue; }
            auto const it = std::find_if(heaps[p].begin(), heaps[p].end(), [&](const Entry & h) { return h.t == e.t; });
            if (it != heaps[p].end()) { e = *it; } else { ep.push_back(p); es.push_back(&e); }
          }
        }
        if ((rc = align_entries(ep, es)) != VSG_OK) { return rc; }
        candidates_of(hp, c1);
        if (c1 != spec[i]) {
          st.recomputed++;
          std::vector<int64_t> q1{static_cast<int64_t>(j)};
          std::vector<int32_t> f1{0, static_cast<int32_t>(c1.size())};
          std::vector<Eval> e1;
          if ((rc = fin.run(set.get(), txt, set.get(), txt, q1, f1, c1, e1, st)) != VSG_OK) { return rc; }
          ev[i] = std::move(e1[0]);
        }
      }
      if (ev[i].status < SUSPICIOUS) { nonchim[i] = 1; appended.push_back(static_cast<uint32_t>(j)); }
      wr.add(head[j], cat.data() + off[j], len[j], size[j], ev[i], st);
    }
    st.serial_s += seconds(tp);
    tp = std::chrono::steady_clock::now();
    if ((rc = wr.flush()) != VSG_OK) { return rc; }
    st.write_s += seconds(tp);
    // 3. the band's non-chimeras join the index
    if (!appended.empty() && (rc = cindex_append(ctx, cix.get(), appended.data(), static_cast<int>(appended.size()))) != VSG_OK) { return rc; }
    b0 = b1;
  }
  return VSG_OK;
}

}  // namespace

extern "C" void vsg_uchime_opts_default(int command, vsg_uchime_opts * o)
{
  if (o == nullptr) { return; }
  *o = vsg_uchime_opts{};
  o->command = command;
  o->abskew = command == VSG_UCHIME_3_DENOVO ? 16.0 : (command == VSG_CHIMERAS_DENOVO ? 1.0 : 2.0);
  o->dn = 1.4;
  o->xn = 8.0;
  o->mindiv = 0.8;
  o->minh = 0.28;
  o->mindiffs = 3;
  o->qmask = VSG_DBMASK_DUST;
  o->dbmask = VSG_DBMASK_DUST;
  o->fasta_width = 80;
  o->alignwidth = command == VSG_CHIMERAS_DENOVO ? 60 : 80;
  o->minseqlength = 1;
  o->maxseqlength = 50000;
  o->batch_queries = 8192;
  o->band_cap = 1024;
  o->chimeras_parts = 0;
  o->chimeras_parents_max = 3;
  o->chimeras_length_min = 10;
  o->chimeras_diff_pct = 0.0;
}

extern "C" int vsg_uchime_command(vsg_ctx * ctx, const char * input_path, const char * db_path, const vsg_uchime_opts * opts,
                                  const vsg_uchime_outputs * outputs, vsg_uchime_stats * stats)
{
  char const * const caller = "vsg_uchime_command";
  if (ctx == nullptr || input_path == nullptr || opts == nullptr || outputs == nullptr) { Error::set("vsg_uchime_command: null argument"); return VSG_EINVAL; }
  vsg_uchime_opts const & o = *opts;
  int rc = check_opts(caller, db_path, o, *outputs);
  if (rc != VSG_OK) { return rc; }
  VSG_CUDA_OK(cudaSetDevice(ctx->device));
  auto const t_wall = std::chrono::steady_clock::now();
  vsg_uchime_stats st{};
  EvalOpts const eo{o.dn, o.xn, o.mindiv, o.minh, o.mindiffs, o.xsize != 0, o.uchimeout5 != 0, outputs->uchimeout != nullptr,
                    outputs->uchimealns != nullptr, o.alignwidth, o.command == VSG_UCHIME_2_DENOVO || o.command == VSG_UCHIME_3_DENOVO};
  Writer wr(caller, o, *outputs);
  rc = o.command == VSG_UCHIME_REF ? uchime_ref(ctx, caller, input_path, db_path, o, eo, wr, st)
                                   : uchime_denovo(ctx, caller, input_path, o, eo, wr, st);
  bool const closed = wr.close();
  if (rc != VSG_OK) { return rc; }
  if (!closed) { Error::set(std::string(caller) + ": unable to write the output files"); return VSG_EINVAL; }
  wr.files.ok = true;
  st.wall_s = seconds(t_wall);
  if (stats != nullptr) { *stats = st; }
  return VSG_OK;
}
