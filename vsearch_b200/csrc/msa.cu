// msa.cu — cluster consensus: the column layout, the symbol profile and the consensus row of every cluster of a
// clustering, for --msaout, --consout and --profile.
//
// Replaces the computation of msa() (reference core/msa.cpp), which cluster() calls cluster by cluster
// (core/cluster.cpp:1473-1539); the printing is vsg_cluster_msa_write's (cluster_cmd.cu).  In order, per chunk of
// clusters on the device:
//   find_max_insertions_per_position   msa_insertions_kernel   atomicMax of every D run at its centroid position
//   find_total_alignment_length         cub::DeviceScan         column offsets of the insertion blocks (64-bit)
//   update_profile over every row       msa_histogram_kernel    symbol counters; gaps are never scattered
//   compute_and_print_consensus         msa_consensus_kernel    gap = cluster weight - symbols, censoring, argmax
// Every count is an exact integer sum, so the results do not depend on the order of the atomics.
#include "vsg_internal.h"

#include <cub/cub.cuh>
#include <thrust/iterator/transform_iterator.h>

#include <algorithm>
#include <chrono>
#include <cinttypes>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

using namespace vsg;

namespace {

constexpr int MSA_THREADS = 256;
constexpr int MSA_TILE = 1024;               // columns of a shared-memory tile: 5 u64 counters each, 40 KiB
constexpr int64_t MSA_PRIVATE_MIN = 64;      // rows from which a cluster is counted in shared memory
constexpr int64_t MSA_JOB_SYMBOLS = 1 << 16; // symbols a histogram CTA aims to cover

// A run of a row's CIGAR that puts row symbols into columns: t0 = first row symbol, q0 = centroid position, run > 0:
// an M run (symbol t0 + k in the centroid column of position q0 + k), run < 0: a D run of -run symbols (into the
// insertion block before position q0).  I runs put gaps and are not stored.  member: the chunk's row number.
struct MsaSeg {
  int32_t t0, q0, run, member;
};

// One CTA of the histogram: the segments of rows [m0, m1).  shared != 0: the rows are one cluster's, and only their
// symbols in columns [col0, col0 + ncols) are counted, in shared memory, then flushed with one atomic per counter.
struct MsaJob {
  int64_t col0;
  int32_t ncols, m0, m1, shared;
};

struct MsaDev {
  DevSeqs set;
  const MsaSeg * seg;
  const int32_t * seg_first;   // per row, + 1
  const uint32_t * mseq;       // the row's sequence in the set
  const uint8_t * mstrand;     // 1: the row is the sequence's reverse complement
  const uint64_t * mweight;
  const int32_t * mcluster;    // chunk-local cluster
  const int64_t * ibase;       // per cluster + 1: its first entry of ins / start (len(centroid) + 1 entries each)
  int32_t * ins;               // nins + 1: the insertion block widths, then -1
  int64_t * start;             // nins + 1: exclusive sum of ins + 1
  int64_t * colfirst;          // per cluster + 1: the cluster's first column
  const uint64_t * cweight;    // per cluster: the weight of its rows
  uint64_t * prof;             // 6 per column
  char * cons;                 // 1 per column
  int64_t nseg, nins, ncols;
  int32_t nc;
};

// Column layout: entry i of cluster c (0 <= i - ibase[c] <= len(centroid)) is the insertion block before centroid
// position i - ibase[c] followed by that position's column; the last entry has no centroid column.  The scan counts
// every entry as ins + 1, so cluster c's entries are shifted by c columns: block i begins at start[i] - c, and the
// centroid column of position p is start[ibase[c] + p + 1] - c - 1.
__device__ __forceinline__ int64_t block_col(const MsaDev & d, int64_t i, int c) { return d.start[i] - c; }

__global__ void __launch_bounds__(MSA_THREADS) msa_insertions_kernel(MsaDev d)
{
  for (int64_t s = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; s < d.nseg; s += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    MsaSeg const g = d.seg[s];
    if (g.run < 0) { atomicMax(&d.ins[d.ibase[d.mcluster[g.member]] + g.q0], -g.run); }
  }
}

struct PlusOne {
  __host__ __device__ int64_t operator()(int32_t x) const { return static_cast<int64_t>(x) + 1; }
};

__global__ void msa_colfirst_kernel(MsaDev d)
{
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c <= d.nc; c += gridDim.x * blockDim.x) {
    d.colfirst[c] = block_col(d, d.ibase[c], c);
  }
}

// update_profile's counters: A, C, G, T / U, then every other code (IUPAC, N) as N; a minus-strand row reads the
// sequence backwards and complemented (the bit reversal of the 4-bit code)
__device__ __forceinline__ int symbol_class(const uint8_t * p, int len, bool minus, int t)
{
  int code = minus ? p[len - 1 - t] & 15 : p[t] & 15;
  if (minus) { code = ((code & 1) << 3) | ((code & 2) << 1) | ((code & 4) >> 1) | ((code & 8) >> 3); }
  switch (code) {
    case 1: return 0;
    case 2: return 1;
    case 4: return 2;
    case 8: return 3;
    default: return 4;
  }
}

__global__ void __launch_bounds__(MSA_THREADS) msa_histogram_kernel(MsaDev d, const MsaJob * __restrict__ jobs)
{
  extern __shared__ unsigned long long tile[];
  MsaJob const j = jobs[blockIdx.x];
  bool const priv = j.shared != 0;
  if (priv) {
    for (int i = threadIdx.x; i < j.ncols * 5; i += blockDim.x) { tile[i] = 0; }
    __syncthreads();
  }
  int const lane = threadIdx.x & 31;
  int const nw = blockDim.x >> 5;
  int const s1 = d.seg_first[j.m1];
  for (int s = d.seg_first[j.m0] + static_cast<int>(threadIdx.x >> 5); s < s1; s += nw) {
    MsaSeg const g = d.seg[s];
    int const c = d.mcluster[g.member];
    int64_t const ib = d.ibase[c] + g.q0;
    uint32_t const seq = d.mseq[g.member];
    bool const minus = d.mstrand[g.member] != 0;
    unsigned long long const w = d.mweight[g.member];
    uint8_t const * const p = d.set.sym + d.set.off[seq];
    int const len = d.set.len[seq];
    bool const del = g.run < 0;
    int const n = del ? -g.run : g.run;
    int lo = 0, hi = n;
    if (priv) {
      // the part of the run inside the tile: a D run's columns are consecutive, an M run's increase with k
      int64_t const a = j.col0, b = j.col0 + j.ncols;
      if (del) {
        int64_t const c0 = block_col(d, ib, c);
        lo = static_cast<int>(a - c0 < 0 ? 0 : (a - c0 > n ? n : a - c0));
        hi = static_cast<int>(b - c0 < 0 ? 0 : (b - c0 > n ? n : b - c0));
      } else {
        auto first_at = [&](int64_t x) {   // the first k with column(k) >= x
          int l = 0, h = n;
          while (l < h) {
            int const m = (l + h) >> 1;
            if (block_col(d, ib + m + 1, c) - 1 < x) { l = m + 1; } else { h = m; }
          }
          return l;
        };
        lo = first_at(a);
        hi = first_at(b);
      }
    }
    int64_t const c0 = del ? block_col(d, ib, c) : 0;
    for (int k = lo + lane; k < hi; k += 32) {
      int64_t const col = del ? c0 + k : block_col(d, ib + k + 1, c) - 1;
      int const cls = symbol_class(p, len, minus, g.t0 + k);
      if (priv) {
        atomicAdd(&tile[(col - j.col0) * 5 + cls], w);
      } else {
        atomicAdd(reinterpret_cast<unsigned long long *>(&d.prof[col * 6 + cls]), w);
      }
    }
  }
  if (priv) {
    __syncthreads();
    for (int i = threadIdx.x; i < j.ncols * 5; i += blockDim.x) {
      unsigned long long const v = tile[i];
      if (v != 0) { atomicAdd(reinterpret_cast<unsigned long long *>(&d.prof[(j.col0 + i / 5) * 6 + i % 5]), v); }
    }
  }
}

// compute_and_print_consensus: the first ins[0] and last ins[len] columns censored ('+'); elsewhere the best of A, C,
// G, T under a strict '>' (A wins a tie), else N when there are N, printed when its count reaches the gaps, else '-'
__global__ void __launch_bounds__(MSA_THREADS) msa_consensus_kernel(MsaDev d)
{
  for (int64_t col = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; col < d.ncols;
       col += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    int lo = 0, hi = d.nc;   // the last cluster whose first column is <= col
    while (hi - lo > 1) {
      int const m = (lo + hi) >> 1;
      if (d.colfirst[m] <= col) { lo = m; } else { hi = m; }
    }
    int64_t const k = col - d.colfirst[lo];
    int64_t const width = d.colfirst[lo + 1] - d.colfirst[lo];
    int const left = d.ins[d.ibase[lo]];
    int const right = d.ins[d.ibase[lo + 1] - 1];
    uint64_t * const q = d.prof + col * 6;
    uint64_t const gap = d.cweight[lo] - (q[0] + q[1] + q[2] + q[3] + q[4]);
    q[5] = gap;
    char sym = '+';
    if (k >= left && k < width - right) {
      char best = '-';
      uint64_t count = 0;
      for (int i = 0; i < 4; i++) {
        if (q[i] > count) { count = q[i]; best = "ACGT"[i]; }
      }
      if (count == 0 && q[4] > 0) { count = q[4]; best = 'N'; }
      sym = count >= gap ? best : '-';
    }
    d.cons[col] = sym;
  }
}

int grid_for(int64_t work)
{
  return static_cast<int>(std::max<int64_t>(1, std::min<int64_t>((work + MSA_THREADS - 1) / MSA_THREADS, 1 << 16)));
}

// device buffers of one call, released on every return
struct MsaBufs {
  DevBuf seg, seg_first, mseq, mstrand, mweight, mcluster, ibase, ins, start, colfirst, cweight, prof, cons, jobs, tmp;
  ~MsaBufs()
  {
    for (DevBuf * b : {&seg, &seg_first, &mseq, &mstrand, &mweight, &mcluster, &ibase, &ins, &start, &colfirst, &cweight, &prof,
                       &cons, &jobs, &tmp}) {
      b->release();
    }
  }
};

template <typename T>
int upload(vsg_ctx * ctx, DevBuf & b, const std::vector<T> & v)
{
  if (b.reserve(std::max<size_t>(v.size(), 1) * sizeof(T)) != VSG_OK) { return VSG_ECUDA; }
  if (!v.empty()) { VSG_CUDA_OK(cudaMemcpyAsync(b.p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, ctx->stream)); }
  return VSG_OK;
}

// parse one CIGAR into segments; false unless it spans the centroid (M + I) and the row (M + D)
bool parse_cigar(const char * cigar, int32_t member, int64_t centroid_len, int64_t row_len, std::vector<MsaSeg> & out)
{
  int64_t q = 0, t = 0;
  for (char const * p = cigar; *p != '\0';) {
    int64_t run = 1;
    if (*p >= '0' && *p <= '9') {
      run = 0;
      while (*p >= '0' && *p <= '9') { run = run * 10 + (*p++ - '0'); if (run > 0x7fffffff) { return false; } }
    }
    char const op = *p++;
    if (op == 'M') {
      out.push_back(MsaSeg{static_cast<int32_t>(t), static_cast<int32_t>(q), static_cast<int32_t>(run), member});
      q += run;
      t += run;
    } else if (op == 'D') {
      if (q > centroid_len) { return false; }
      out.push_back(MsaSeg{static_cast<int32_t>(t), static_cast<int32_t>(q), static_cast<int32_t>(-run), member});
      t += run;
    } else if (op == 'I') {
      q += run;
    } else {
      return false;
    }
    if (q > centroid_len || t > row_len) { return false; }
  }
  return q == centroid_len && t == row_len;
}

}  // namespace

extern "C" int vsg_cluster_msa(vsg_ctx * ctx, const vsg_seqset * set, int64_t n, const vsg_cluster_result * results,
                               const uint64_t * weights, const char * cigar_buf, const int64_t * cigar_off, int32_t * insertions,
                               int64_t * col_first, uint64_t * profile, char * consensus, int64_t cap, int64_t * ncolumns)
{
  if (ctx == nullptr || set == nullptr || ncolumns == nullptr || n < 0 ||
      (n > 0 && (results == nullptr || weights == nullptr || cigar_buf == nullptr || cigar_off == nullptr ||
                 insertions == nullptr || col_first == nullptr))) {
    Error::set("vsg_cluster_msa: null argument");
    return VSG_EINVAL;
  }
  if (n != set->d.n) { Error::set("vsg_cluster_msa: n is not the number of sequences of the set"); return VSG_EINVAL; }
  if (n > 0x7fffffff) { Error::set("vsg_cluster_msa: too many sequences"); return VSG_EINVAL; }
  static const bool trace = std::getenv("VSG_TRACE") != nullptr;
  auto const t0 = std::chrono::steady_clock::now();

  // the clusters: rows by cluster in processing order, the centroid (the S record) first
  int64_t nclusters = 0;
  for (int64_t i = 0; i < n; i++) {
    vsg_cluster_result const & r = results[i];
    bool const ok = r.cluster >= 0 && r.cluster <= i &&
                    (r.centroid < 0 ? true : r.centroid < i && results[r.centroid].centroid < 0 && results[r.centroid].cluster == r.cluster);
    if (!ok || weights[i] == 0) {
      Error::set("vsg_cluster_msa: result " + std::to_string(i) + (ok ? " has weight 0" : " is not a cluster assignment"));
      return VSG_EINVAL;
    }
    nclusters = std::max<int64_t>(nclusters, r.cluster + 1);
  }
  std::vector<int64_t> rfirst(static_cast<size_t>(nclusters) + 1, 0), centroid(static_cast<size_t>(nclusters), -1);
  for (int64_t i = 0; i < n; i++) {
    rfirst[static_cast<size_t>(results[i].cluster) + 1]++;
    if (results[i].centroid < 0) {
      if (centroid[static_cast<size_t>(results[i].cluster)] >= 0) { Error::set("vsg_cluster_msa: a cluster with two centroids"); return VSG_EINVAL; }
      centroid[static_cast<size_t>(results[i].cluster)] = i;
    }
  }
  for (int64_t c = 0; c < nclusters; c++) {
    if (centroid[static_cast<size_t>(c)] < 0) { Error::set("vsg_cluster_msa: cluster " + std::to_string(c) + " has no centroid"); return VSG_EINVAL; }
    rfirst[static_cast<size_t>(c) + 1] += rfirst[static_cast<size_t>(c)];
  }
  std::vector<int64_t> rows(static_cast<size_t>(n));
  {
    std::vector<int64_t> fill(rfirst.begin(), rfirst.end() - 1);
    for (int64_t i = 0; i < n; i++) { rows[static_cast<size_t>(fill[static_cast<size_t>(results[i].cluster)]++)] = i; }
  }
  // every row's segments, rows in cluster order; the centroid is one M run
  std::vector<int64_t> ifirst(static_cast<size_t>(nclusters) + 1, 0), sfirst(static_cast<size_t>(n) + 1, 0);
  std::vector<MsaSeg> segs;
  for (int64_t c = 0; c < nclusters; c++) {
    int64_t const cl = set->h_len[static_cast<size_t>(centroid[static_cast<size_t>(c)])];
    ifirst[static_cast<size_t>(c) + 1] = ifirst[static_cast<size_t>(c)] + cl + 1;
    for (int64_t k = rfirst[static_cast<size_t>(c)]; k < rfirst[static_cast<size_t>(c) + 1]; k++) {
      int64_t const i = rows[static_cast<size_t>(k)];
      if (results[i].centroid < 0) {
        if (cl > 0) { segs.push_back(MsaSeg{0, 0, static_cast<int32_t>(cl), static_cast<int32_t>(k)}); }
      } else if (!parse_cigar(cigar_buf + cigar_off[i], static_cast<int32_t>(k), cl, set->h_len[static_cast<size_t>(i)], segs)) {
        Error::set("vsg_cluster_msa: the CIGAR of record " + std::to_string(i) + " does not align it with its centroid");
        return VSG_EINVAL;
      }
      sfirst[static_cast<size_t>(k) + 1] = static_cast<int64_t>(segs.size());
    }
  }
  if (static_cast<int64_t>(segs.size()) > 0x7fffffff) { Error::set("vsg_cluster_msa: too many CIGAR runs"); return VSG_EINVAL; }
  std::vector<uint64_t> cweight(static_cast<size_t>(nclusters), 0);
  for (int64_t i = 0; i < n; i++) { cweight[static_cast<size_t>(results[i].cluster)] += weights[i]; }

  // chunks of whole clusters under a quarter of the direction-bit budget (at most 1 GiB); a cluster that needs more
  // goes alone.  The first pass sizes the layout, the second (with the exact column counts) adds the profile.
  size_t const budget = std::min<size_t>(ctx->dir_budget / 4, static_cast<size_t>(1) << 30);
  auto cluster_bytes = [&](int64_t c, int64_t cols) {
    int64_t const nr = rfirst[static_cast<size_t>(c) + 1] - rfirst[static_cast<size_t>(c)];
    int64_t const ns = sfirst[static_cast<size_t>(rfirst[static_cast<size_t>(c) + 1])] - sfirst[static_cast<size_t>(rfirst[static_cast<size_t>(c)])];
    return static_cast<size_t>((ifirst[static_cast<size_t>(c) + 1] - ifirst[static_cast<size_t>(c)]) * 12 + ns * 16 + nr * 29 + 32 + cols * 49 +
                               (cols / MSA_TILE + 1) * (nr / 32 + 1) * 24);
  };
  auto chunks_of = [&](const std::vector<int64_t> * cols) {
    std::vector<int64_t> cut{0};
    size_t used = 0;
    for (int64_t c = 0; c < nclusters; c++) {
      size_t const b = cluster_bytes(c, cols != nullptr ? (*cols)[static_cast<size_t>(c) + 1] - (*cols)[static_cast<size_t>(c)] : 0);
      if (c > cut.back() && used + b > budget) { cut.push_back(c); used = 0; }
      used += b;
    }
    if (nclusters > 0) { cut.push_back(nclusters); }
    return cut;
  };

  MsaBufs B;
  MsaDev d{};
  d.set = set->d;
  int rc = VSG_OK;
  cudaEvent_t ev0 = ctx->ev[0], ev1 = ctx->ev[1];
  float kernel_ms = 0.f;
  // uploads clusters [c0, c1), lays out their columns on the device
  auto prepare = [&](int64_t c0, int64_t c1) -> int {
    int64_t const r0 = rfirst[static_cast<size_t>(c0)], r1 = rfirst[static_cast<size_t>(c1)];
    int64_t const s0 = sfirst[static_cast<size_t>(r0)], s1 = sfirst[static_cast<size_t>(r1)];
    std::vector<MsaSeg> seg(segs.begin() + s0, segs.begin() + s1);
    for (MsaSeg & g : seg) { g.member -= static_cast<int32_t>(r0); }
    std::vector<int32_t> sf(static_cast<size_t>(r1 - r0) + 1), mcl(static_cast<size_t>(r1 - r0));
    std::vector<uint32_t> mseq(static_cast<size_t>(r1 - r0));
    std::vector<uint8_t> mstrand(static_cast<size_t>(r1 - r0));
    std::vector<uint64_t> mw(static_cast<size_t>(r1 - r0));
    for (int64_t k = r0; k <= r1; k++) { sf[static_cast<size_t>(k - r0)] = static_cast<int32_t>(sfirst[static_cast<size_t>(k)] - s0); }
    for (int64_t k = r0; k < r1; k++) {
      int64_t const i = rows[static_cast<size_t>(k)];
      mseq[static_cast<size_t>(k - r0)] = static_cast<uint32_t>(i);
      mstrand[static_cast<size_t>(k - r0)] = results[i].centroid >= 0 && results[i].strand != 0 ? 1 : 0;
      mw[static_cast<size_t>(k - r0)] = weights[i];
      mcl[static_cast<size_t>(k - r0)] = results[i].cluster - static_cast<int32_t>(c0);
    }
    std::vector<int64_t> ib(static_cast<size_t>(c1 - c0) + 1);
    for (int64_t c = c0; c <= c1; c++) { ib[static_cast<size_t>(c - c0)] = ifirst[static_cast<size_t>(c)] - ifirst[static_cast<size_t>(c0)]; }
    std::vector<uint64_t> cw(cweight.begin() + c0, cweight.begin() + c1);
    d.nseg = s1 - s0;
    d.nins = ib.back();
    d.nc = static_cast<int32_t>(c1 - c0);
    int e;
    if ((e = upload(ctx, B.seg, seg)) != VSG_OK || (e = upload(ctx, B.seg_first, sf)) != VSG_OK || (e = upload(ctx, B.mseq, mseq)) != VSG_OK ||
        (e = upload(ctx, B.mstrand, mstrand)) != VSG_OK || (e = upload(ctx, B.mweight, mw)) != VSG_OK ||
        (e = upload(ctx, B.mcluster, mcl)) != VSG_OK || (e = upload(ctx, B.ibase, ib)) != VSG_OK || (e = upload(ctx, B.cweight, cw)) != VSG_OK) {
      return e;
    }
    if (B.ins.reserve(static_cast<size_t>(d.nins + 1) * 4) != VSG_OK || B.start.reserve(static_cast<size_t>(d.nins + 1) * 8) != VSG_OK ||
        B.colfirst.reserve(static_cast<size_t>(d.nc + 1) * 8) != VSG_OK) {
      return VSG_ECUDA;
    }
    d.seg = static_cast<const MsaSeg *>(B.seg.p);
    d.seg_first = static_cast<const int32_t *>(B.seg_first.p);
    d.mseq = static_cast<const uint32_t *>(B.mseq.p);
    d.mstrand = static_cast<const uint8_t *>(B.mstrand.p);
    d.mweight = static_cast<const uint64_t *>(B.mweight.p);
    d.mcluster = static_cast<const int32_t *>(B.mcluster.p);
    d.ibase = static_cast<const int64_t *>(B.ibase.p);
    d.cweight = static_cast<const uint64_t *>(B.cweight.p);
    d.ins = static_cast<int32_t *>(B.ins.p);
    d.start = static_cast<int64_t *>(B.start.p);
    d.colfirst = static_cast<int64_t *>(B.colfirst.p);
    VSG_CUDA_OK(cudaEventRecord(ev0, ctx->stream));
    VSG_CUDA_OK(cudaMemsetAsync(d.ins, 0, static_cast<size_t>(d.nins) * 4, ctx->stream));
    VSG_CUDA_OK(cudaMemsetAsync(d.ins + d.nins, 0xff, 4, ctx->stream));   // -1: the scan's last entry adds 0
    msa_insertions_kernel<<<grid_for(d.nseg), MSA_THREADS, 0, ctx->stream>>>(d);
    count_launch();
    auto const widths = thrust::make_transform_iterator(static_cast<const int32_t *>(d.ins), PlusOne{});
    size_t tmp = 0;
    VSG_CUDA_OK(cub::DeviceScan::ExclusiveSum(nullptr, tmp, widths, d.start, d.nins + 1, ctx->stream));
    if (B.tmp.reserve(std::max<size_t>(tmp, 1)) != VSG_OK) { return VSG_ECUDA; }
    VSG_CUDA_OK(cub::DeviceScan::ExclusiveSum(B.tmp.p, tmp, widths, d.start, d.nins + 1, ctx->stream));
    msa_colfirst_kernel<<<grid_for(d.nc + 1), MSA_THREADS, 0, ctx->stream>>>(d);
    count_launch(2);
    VSG_CUDA_OK(cudaEventRecord(ev1, ctx->stream));
    VSG_CUDA_OK(cudaGetLastError());
    return VSG_OK;
  };
  auto add_time = [&]() -> int {
    VSG_CUDA_OK(cudaEventSynchronize(ev1));
    float ms = 0.f;
    VSG_CUDA_OK(cudaEventElapsedTime(&ms, ev0, ev1));
    kernel_ms += ms;
    return VSG_OK;
  };

  // pass 1: the insertion widths and the column offsets of every cluster
  std::vector<int64_t> const cut1 = chunks_of(nullptr);
  std::vector<int64_t> cols(static_cast<size_t>(nclusters) + 1, 0);
  std::vector<int64_t> lf;
  for (size_t h = 0; h + 1 < cut1.size(); h++) {
    int64_t const c0 = cut1[h], c1 = cut1[h + 1];
    if ((rc = prepare(c0, c1)) != VSG_OK) { return rc; }
    lf.resize(static_cast<size_t>(c1 - c0) + 1);
    VSG_CUDA_OK(cudaMemcpyAsync(insertions + ifirst[static_cast<size_t>(c0)], d.ins, static_cast<size_t>(d.nins) * 4, cudaMemcpyDeviceToHost, ctx->stream));
    VSG_CUDA_OK(cudaMemcpyAsync(lf.data(), d.colfirst, lf.size() * 8, cudaMemcpyDeviceToHost, ctx->stream));
    VSG_CUDA_OK(cudaStreamSynchronize(ctx->stream));
    if ((rc = add_time()) != VSG_OK) { return rc; }
    for (int64_t c = c0; c <= c1; c++) { cols[static_cast<size_t>(c)] = cols[static_cast<size_t>(c0)] + lf[static_cast<size_t>(c - c0)]; }
  }
  for (int64_t c = 0; c <= nclusters; c++) { col_first[c] = cols[static_cast<size_t>(c)]; }
  int64_t const total = cols.back();
  *ncolumns = total;
  if (total > cap) {
    Error::set("vsg_cluster_msa: the profile needs " + std::to_string(total) + " columns, cap is " + std::to_string(cap));
    return VSG_ECAP;
  }
  if (total > 0 && (profile == nullptr || consensus == nullptr)) { Error::set("vsg_cluster_msa: null argument"); return VSG_EINVAL; }

  // pass 2: the profile and the consensus, chunk by chunk
  std::vector<int64_t> const cut2 = chunks_of(&cols);
  bool const reuse = cut1.size() == 2 && cut2 == cut1;
  std::vector<MsaJob> jobs;
  for (size_t h = 0; h + 1 < cut2.size(); h++) {
    int64_t const c0 = cut2[h], c1 = cut2[h + 1];
    if (!reuse && (rc = prepare(c0, c1)) != VSG_OK) { return rc; }
    int64_t const colbase = cols[static_cast<size_t>(c0)];
    d.ncols = cols[static_cast<size_t>(c1)] - colbase;
    // jobs: a large cluster as column tiles by row slices counted in shared memory, small ones packed together and
    // counted with global atomics
    jobs.clear();
    int64_t const rbase = rfirst[static_cast<size_t>(c0)];
    int64_t open = -1, open_sym = 0;
    auto close_open = [&](int64_t r_end) {
      if (open >= 0) { jobs.push_back(MsaJob{0, 0, static_cast<int32_t>(open - rbase), static_cast<int32_t>(r_end - rbase), 0}); }
      open = -1;
      open_sym = 0;
    };
    for (int64_t c = c0; c < c1; c++) {
      int64_t const r0 = rfirst[static_cast<size_t>(c)], r1 = rfirst[static_cast<size_t>(c) + 1];
      int64_t const width = cols[static_cast<size_t>(c) + 1] - cols[static_cast<size_t>(c)];
      if (r1 - r0 < MSA_PRIVATE_MIN) {
        if (open < 0) { open = r0; }
        open_sym += (r1 - r0) * width;
        if (open_sym >= MSA_JOB_SYMBOLS) { close_open(r1); }
        continue;
      }
      close_open(r0);
      int64_t const slice = std::max<int64_t>(32, MSA_JOB_SYMBOLS / std::max<int64_t>(1, std::min<int64_t>(width, MSA_TILE)));
      for (int64_t a = 0; a < width; a += MSA_TILE) {
        for (int64_t r = r0; r < r1; r += slice) {
          jobs.push_back(MsaJob{cols[static_cast<size_t>(c)] - colbase + a, static_cast<int32_t>(std::min<int64_t>(MSA_TILE, width - a)),
                                static_cast<int32_t>(r - rbase), static_cast<int32_t>(std::min(r1, r + slice) - rbase), 1});
        }
      }
    }
    close_open(rfirst[static_cast<size_t>(c1)]);
    if ((rc = upload(ctx, B.jobs, jobs)) != VSG_OK) { return rc; }
    if (B.prof.reserve(static_cast<size_t>(std::max<int64_t>(d.ncols, 1)) * 48) != VSG_OK ||
        B.cons.reserve(static_cast<size_t>(std::max<int64_t>(d.ncols, 1))) != VSG_OK) {
      return VSG_ECUDA;
    }
    d.prof = static_cast<uint64_t *>(B.prof.p);
    d.cons = static_cast<char *>(B.cons.p);
    VSG_CUDA_OK(cudaEventRecord(ev0, ctx->stream));
    VSG_CUDA_OK(cudaMemsetAsync(d.prof, 0, static_cast<size_t>(d.ncols) * 48, ctx->stream));
    if (!jobs.empty()) {
      msa_histogram_kernel<<<static_cast<unsigned>(jobs.size()), MSA_THREADS, MSA_TILE * 5 * sizeof(unsigned long long), ctx->stream>>>(
          d, static_cast<const MsaJob *>(B.jobs.p));
      count_launch();
    }
    if (d.ncols > 0) {
      msa_consensus_kernel<<<grid_for(d.ncols), MSA_THREADS, 0, ctx->stream>>>(d);
      count_launch();
    }
    VSG_CUDA_OK(cudaEventRecord(ev1, ctx->stream));
    VSG_CUDA_OK(cudaGetLastError());
    VSG_CUDA_OK(cudaMemcpyAsync(profile + colbase * 6, d.prof, static_cast<size_t>(d.ncols) * 48, cudaMemcpyDeviceToHost, ctx->stream));
    VSG_CUDA_OK(cudaMemcpyAsync(consensus + colbase, d.cons, static_cast<size_t>(d.ncols), cudaMemcpyDeviceToHost, ctx->stream));
    VSG_CUDA_OK(cudaStreamSynchronize(ctx->stream));
    if ((rc = add_time()) != VSG_OK) { return rc; }
  }
  if (trace) {
    std::fprintf(stderr, "[vsg] cluster_msa: %" PRId64 " rows, %" PRId64 " clusters, %" PRId64 " columns, %zu + %zu chunks, kernels %.3f ms, call %.3f ms\n",
                 n, nclusters, total, cut1.size() - 1, reuse ? size_t{0} : cut2.size() - 1, static_cast<double>(kernel_ms),
                 std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count());
  }
  return VSG_OK;
}
