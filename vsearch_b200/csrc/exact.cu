// exact.cu — exact-match search: the device index of full-length sequence hashes and vsg_search_exact.
//
// Replaces, for --search_exact, Dbhash (core/dbhash.cpp) and search_exact_onequery / add_hit (commands/search_exact.cpp:
// 136-209):
//   Dbhash::add_all      CityHash64 of every normalized database sequence into an open-addressing table
//                                       -> hash_kernel over the set, (hash, seqno) keys sorted with CUB
//   Dbhash::search_first / search_next  probe, then compare length and seqcmp
//                                       -> binary search of each query strand's hash, then one warp per candidate
//                                          comparing length and 4-bit codes
//   add_hit                             struct hit of a 100 % match, then the two accept functions (hit_logic.h)
// The hash covers the 4-bit codes (bits 0-3 of a device symbol) and the length, so equal hashes mean what seqcmp
// means: case and U / T never matter, N only equals N.  Every candidate is verified, so the hash only has to spread.
#include "vsg_internal.h"
#include "hit_logic.h"

#include <cub/cub.cuh>

#include <algorithm>
#include <cstdlib>
#include <string>
#include <vector>

using namespace vsg;

struct vsg_exact_index {
  const vsg_seqset * db = nullptr;
  int device = 0;
  int bits = 64;
  int64_t n = 0;
  DevBuf keys, seqnos;   // the database's hashes ascending, and their sequence numbers (ascending among equal hashes)
};

namespace {

// VSG_EXACT_HASH_BITS (1..64, unset = 64): only the low bits of every hash are kept, so tests can force collisions
// through the verify path
int hash_bits()
{
  char const * const e = std::getenv("VSG_EXACT_HASH_BITS");
  if (e == nullptr || *e == '\0') { return 64; }
  int const b = std::atoi(e);
  return b < 1 ? 1 : (b > 64 ? 64 : b);
}

__device__ __forceinline__ uint64_t mix64(uint64_t z)   // the SplitMix64 finaliser
{
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ULL;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebULL;
  return z ^ (z >> 31);
}

// one symbol's share of a hash: position-dependent, summed over the sequence (so lanes can hash disjoint chunks)
__device__ __forceinline__ uint64_t term(int64_t pos, int code)
{
  return mix64((static_cast<uint64_t>(pos) << 4 | static_cast<uint64_t>(code)) + 0x9e3779b97f4a7c15ULL);
}

// the complement of a 4-bit IUPAC code is its bit reversal; a byte without a code (0) becomes N, as revcomp_kernel does
__device__ __forceinline__ int complement4(int c)
{
  return c == 0 ? 15 : ((c & 1) << 3) | ((c & 2) << 1) | ((c & 4) >> 1) | ((c & 8) >> 3);
}

__device__ __forceinline__ void add_symbol(uint8_t s, int64_t i, int len, uint64_t & plus, uint64_t & minus, bool both)
{
  int const c = s & 15;
  plus += term(i, c);
  if (both) { minus += term(len - 1 - i, complement4(c)); }
}

// One warp per sequence s0 + w: the hash of its codes (plus[w]) and, with minus != nullptr, of its reverse complement
// (minus[w]) from the same reads.  Device offsets are not aligned: the bytes before the first and after the last
// 16-byte boundary are read one by one, the chunks in between as aligned 16-byte loads.
__global__ void hash_kernel(DevSeqs s, int64_t s0, int64_t n, uint64_t keep, uint64_t * __restrict__ plus_out,
                            uint64_t * __restrict__ minus_out)
{
  int64_t const w = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  int const lane = threadIdx.x & 31;
  if (w >= n) { return; }
  int64_t const off = s.off[s0 + w];
  int const len = s.len[s0 + w];
  bool const both = minus_out != nullptr;
  uint8_t const * const p = s.sym + off;
  uint64_t plus = 0, minus = 0;
  int64_t const align = (16 - (reinterpret_cast<uintptr_t>(p) & 15)) & 15;
  int64_t const head = align < len ? align : len;
  int64_t const body = ((len - head) / 16) * 16;
  if (lane < head) { add_symbol(p[lane], lane, len, plus, minus, both); }
  int64_t const tail = len - head - body;
  if (lane >= 16 && lane - 16 < tail) {
    int64_t const i = head + body + (lane - 16);
    add_symbol(p[i], i, len, plus, minus, both);
  }
  uint4 const * const chunks = reinterpret_cast<uint4 const *>(p + head);
  for (int64_t k = lane; k < body / 16; k += 32) {
    uint4 const v = chunks[k];
    uint32_t const words[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 16; j++) {
      add_symbol(static_cast<uint8_t>(words[j >> 2] >> (8 * (j & 3))), head + 16 * k + j, len, plus, minus, both);
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    plus += __shfl_xor_sync(0xffffffffu, plus, d);
    minus += __shfl_xor_sync(0xffffffffu, minus, d);
  }
  if (lane == 0) {
    uint64_t const l = mix64(static_cast<uint64_t>(len) + 0x632be59bd9b4e019ULL);
    plus_out[w] = mix64(plus ^ l) & keep;
    if (both) { minus_out[w] = mix64(minus ^ l) & keep; }
  }
}

// query strand j (= query * strands + strand): the range of database keys equal to its hash
__global__ void lookup_kernel(const uint64_t * __restrict__ keys, int64_t nkeys, const uint64_t * __restrict__ qhash, int64_t nj,
                              int strands, int64_t * __restrict__ lo, int64_t * __restrict__ count)
{
  int64_t const j = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (j >= nj) { return; }
  // qhash holds the plus hashes of all queries, then the minus hashes
  int64_t const nq = nj / strands;
  uint64_t const h = qhash[(j % strands) * nq + j / strands];
  int64_t a = 0, b = nkeys;
  while (a < b) { int64_t const m = (a + b) >> 1; if (keys[m] < h) { a = m + 1; } else { b = m; } }
  int64_t e = a, f = nkeys;
  while (e < f) { int64_t const m = (e + f) >> 1; if (keys[m] <= h) { e = m + 1; } else { f = m; } }
  lo[j] = a;
  count[j] = e - a;
}

// One warp per candidate k: its query strand (the last j with first[j] <= k), its target, and whether the two are
// equal: the same length and the same codes, read through the complement for the minus strand.  row[k] packs
// (query strand, target); flag[k] says whether it is a match.
__global__ void verify_kernel(DevSeqs q, int64_t q0, DevSeqs t, const uint32_t * __restrict__ seqnos, const int64_t * __restrict__ lo,
                              const int64_t * __restrict__ first, int64_t nj, int strands, int64_t ncand,
                              uint64_t * __restrict__ row, uint8_t * __restrict__ flag)
{
  int64_t const k = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  int const lane = threadIdx.x & 31;
  if (k >= ncand) { return; }
  int64_t a = 0, b = nj;   // first index with first[.] > k, minus one
  while (a < b) { int64_t const m = (a + b) >> 1; if (first[m] <= k) { a = m + 1; } else { b = m; } }
  int64_t const j = a - 1;
  uint32_t const target = seqnos[lo[j] + (k - first[j])];
  int64_t const query = j / strands;
  int const strand = static_cast<int>(j % strands);
  int const len = q.len[q0 + query];
  bool same = len == t.len[target];
  if (same) {
    uint8_t const * const qs = q.sym + q.off[q0 + query];
    uint8_t const * const ts = t.sym + t.off[target];
    for (int base = 0; base < len && same; base += 32) {
      int const i = base + lane;
      bool ok = true;
      if (i < len) {
        int const c = strand == 0 ? (qs[i] & 15) : complement4(qs[len - 1 - i] & 15);
        ok = c == (ts[i] & 15);
      }
      same = __all_sync(0xffffffffu, ok);
    }
  }
  if (lane == 0) {
    row[k] = (static_cast<uint64_t>(j) << 32) | target;
    flag[k] = same ? 1 : 0;
  }
}

int launch_hash(vsg_ctx * c, const vsg_seqset * s, int64_t s0, int64_t n, int bits, uint64_t * plus, uint64_t * minus)
{
  if (n == 0) { return VSG_OK; }
  uint64_t const keep = bits >= 64 ? ~0ULL : ((1ULL << bits) - 1);
  int64_t const blocks = (n * 32 + 255) / 256;
  hash_kernel<<<static_cast<unsigned>(blocks), 256, 0, c->stream>>>(s->d, s0, n, keep, plus, minus);
  count_launch();
  VSG_CUDA_OK(cudaGetLastError());
  return VSG_OK;
}

}  // namespace

extern "C" int vsg_exact_index_create(vsg_ctx * c, const vsg_seqset * db, vsg_exact_index ** out)
{
  if (c == nullptr || db == nullptr || out == nullptr) { Error::set("vsg_exact_index_create: null argument"); return VSG_EINVAL; }
  *out = nullptr;
  if (db->device != c->device) { Error::set("vsg_exact_index_create: the set lives on another device than the context"); return VSG_EINVAL; }
  if (db->d.n > 0xffffffffLL) { Error::set("vsg_exact_index_create: more than 2^32 sequences"); return VSG_EINVAL; }
  VSG_CUDA_OK(cudaSetDevice(c->device));
  std::unique_ptr<vsg_exact_index> ix(new vsg_exact_index());
  ix->db = db;
  ix->device = c->device;
  ix->bits = hash_bits();
  int64_t const n = db->d.n;
  ix->n = n;
  int rc = VSG_OK;
  if ((rc = ix->keys.reserve(sizeof(uint64_t) * std::max<int64_t>(n, 1))) != VSG_OK ||
      (rc = ix->seqnos.reserve(sizeof(uint32_t) * std::max<int64_t>(n, 1))) != VSG_OK) { return rc; }
  if (n > 0) {
    DevBuf raw, order;
    if ((rc = raw.reserve(sizeof(uint64_t) * n)) != VSG_OK || (rc = order.reserve(sizeof(uint32_t) * n)) != VSG_OK) {
      raw.release(); order.release();
      return rc;
    }
    std::vector<uint32_t> iota(static_cast<size_t>(n));
    for (int64_t i = 0; i < n; i++) { iota[static_cast<size_t>(i)] = static_cast<uint32_t>(i); }
    rc = launch_hash(c, db, 0, n, ix->bits, static_cast<uint64_t *>(raw.p), nullptr);
    size_t tmp = 0;
    cudaError_t e = cudaSuccess;
    if (rc == VSG_OK) {
      e = cudaMemcpyAsync(order.p, iota.data(), sizeof(uint32_t) * n, cudaMemcpyHostToDevice, c->stream);
      // LSD radix sort is stable: equal hashes keep ascending sequence numbers
      if (e == cudaSuccess) {
        e = cub::DeviceRadixSort::SortPairs(nullptr, tmp, static_cast<uint64_t *>(raw.p), static_cast<uint64_t *>(ix->keys.p),
                                            static_cast<uint32_t *>(order.p), static_cast<uint32_t *>(ix->seqnos.p), n, 0,
                                            ix->bits, c->stream);
      }
      if (e == cudaSuccess && (rc = c->cub_tmp.reserve(tmp)) == VSG_OK) {
        e = cub::DeviceRadixSort::SortPairs(c->cub_tmp.p, tmp, static_cast<uint64_t *>(raw.p), static_cast<uint64_t *>(ix->keys.p),
                                            static_cast<uint32_t *>(order.p), static_cast<uint32_t *>(ix->seqnos.p), n, 0,
                                            ix->bits, c->stream);
        count_launch();
      }
      if (e == cudaSuccess) { e = cudaStreamSynchronize(c->stream); }   // iota must outlive its copy
    }
    raw.release();
    order.release();
    if (rc != VSG_OK) { return rc; }
    VSG_CUDA_OK(e);
  }
  *out = ix.release();
  return VSG_OK;
}

extern "C" void vsg_exact_index_destroy(vsg_exact_index * ix)
{
  if (ix == nullptr) { return; }
  cudaSetDevice(ix->device);
  ix->keys.release();
  ix->seqnos.release();
  delete ix;
}

int vsg::search_exact_host(vsg_ctx * c, const vsg_exact_index * ix, const vsg_seqset * queries, int64_t q0, int64_t nq,
                           const vsg_search_opts * opts, int64_t maxhits, std::vector<vsg_search_result> & rows,
                           std::vector<int64_t> & first)
{
  if (c == nullptr || ix == nullptr || queries == nullptr || opts == nullptr || maxhits < 0) {
    Error::set("vsg_search_exact: bad argument");
    return VSG_EINVAL;
  }
  if (q0 < 0 || nq < 0 || q0 > queries->d.n || nq > queries->d.n - q0) { Error::set("vsg_search_exact: query range out of bounds"); return VSG_EINVAL; }
  if (queries->device != c->device || ix->device != c->device) {
    Error::set("vsg_search_exact: sequence set / index lives on another device than the context");
    return VSG_EINVAL;
  }
  if (nq > 0x7fffffffLL) { Error::set("vsg_search_exact: more than 2^31 queries in one call"); return VSG_EINVAL; }
  VSG_CUDA_OK(cudaSetDevice(c->device));
  int const strands = opts->strand_both != 0 ? 2 : 1;
  int64_t const nj = nq * strands;
  std::vector<uint64_t> found;
  if (nq > 0 && ix->n > 0) {
    DevBuf qhash, lo, cnt, firstd, rowd, flag, sel, nsel;
    struct Release {
      std::vector<DevBuf *> b;
      ~Release() { for (DevBuf * x : b) { x->release(); } }
    } release{{&qhash, &lo, &cnt, &firstd, &rowd, &flag, &sel, &nsel}};
    int rc = VSG_OK;
    if ((rc = qhash.reserve(sizeof(uint64_t) * nj)) != VSG_OK || (rc = lo.reserve(sizeof(int64_t) * nj)) != VSG_OK ||
        (rc = cnt.reserve(sizeof(int64_t) * nj)) != VSG_OK || (rc = firstd.reserve(sizeof(int64_t) * (nj + 1))) != VSG_OK ||
        (rc = nsel.reserve(sizeof(int64_t))) != VSG_OK) { return rc; }
    uint64_t * const qh = static_cast<uint64_t *>(qhash.p);
    if ((rc = launch_hash(c, queries, q0, nq, ix->bits, qh, strands == 2 ? qh + nq : nullptr)) != VSG_OK) { return rc; }
    lookup_kernel<<<static_cast<unsigned>((nj + 255) / 256), 256, 0, c->stream>>>(
        static_cast<const uint64_t *>(ix->keys.p), ix->n, qh, nj, strands, static_cast<int64_t *>(lo.p), static_cast<int64_t *>(cnt.p));
    count_launch();
    // first[j] = the candidates of the strands before j; first[nj] = all of them
    int64_t * const fd = static_cast<int64_t *>(firstd.p);
    VSG_CUDA_OK(cudaMemsetAsync(fd, 0, sizeof(int64_t), c->stream));
    size_t tmp = 0;
    VSG_CUDA_OK(cub::DeviceScan::InclusiveSum(nullptr, tmp, static_cast<int64_t *>(cnt.p), fd + 1, nj, c->stream));
    if ((rc = c->cub_tmp.reserve(tmp)) != VSG_OK) { return rc; }
    VSG_CUDA_OK(cub::DeviceScan::InclusiveSum(c->cub_tmp.p, tmp, static_cast<int64_t *>(cnt.p), fd + 1, nj, c->stream));
    count_launch();
    int64_t ncand = 0;
    VSG_CUDA_OK(cudaMemcpyAsync(&ncand, fd + nj, sizeof(int64_t), cudaMemcpyDeviceToHost, c->stream));
    VSG_CUDA_OK(cudaStreamSynchronize(c->stream));
    if (ncand > 0) {
      if ((rc = rowd.reserve(sizeof(uint64_t) * ncand)) != VSG_OK || (rc = flag.reserve(ncand)) != VSG_OK ||
          (rc = sel.reserve(sizeof(uint64_t) * ncand)) != VSG_OK) { return rc; }
      verify_kernel<<<static_cast<unsigned>((ncand * 32 + 255) / 256), 256, 0, c->stream>>>(
          queries->d, q0, ix->db->d, static_cast<const uint32_t *>(ix->seqnos.p), static_cast<const int64_t *>(lo.p), fd, nj,
          strands, ncand, static_cast<uint64_t *>(rowd.p), static_cast<uint8_t *>(flag.p));
      count_launch();
      VSG_CUDA_OK(cudaGetLastError());
      tmp = 0;
      VSG_CUDA_OK(cub::DeviceSelect::Flagged(nullptr, tmp, static_cast<uint64_t *>(rowd.p), static_cast<uint8_t *>(flag.p),
                                             static_cast<uint64_t *>(sel.p), static_cast<int64_t *>(nsel.p), ncand, c->stream));
      if ((rc = c->cub_tmp.reserve(tmp)) != VSG_OK) { return rc; }
      VSG_CUDA_OK(cub::DeviceSelect::Flagged(c->cub_tmp.p, tmp, static_cast<uint64_t *>(rowd.p), static_cast<uint8_t *>(flag.p),
                                             static_cast<uint64_t *>(sel.p), static_cast<int64_t *>(nsel.p), ncand, c->stream));
      count_launch();
      int64_t nfound = 0;
      VSG_CUDA_OK(cudaMemcpyAsync(&nfound, nsel.p, sizeof(int64_t), cudaMemcpyDeviceToHost, c->stream));
      VSG_CUDA_OK(cudaStreamSynchronize(c->stream));
      found.resize(static_cast<size_t>(nfound));
      VSG_CUDA_OK(cudaMemcpyAsync(found.data(), sel.p, sizeof(uint64_t) * nfound, cudaMemcpyDeviceToHost, c->stream));
      VSG_CUDA_OK(cudaStreamSynchronize(c->stream));
    }
  }

  // add_hit for every match, search_joinhits over both strands.  The found rows come by query strand, each strand's
  // targets ascending.  --search_exact runs with opt_id forced to 1.0 and --id not among its options, so weak_id is
  // -1 (cli.cc's fix-up against the default opt_id): every hit that passes the filters is accepted.
  vsg_search_opts o = *opts;
  o.unoise = 0;
  int64_t const nwmatch = c->scoring.v[0];
  first.assign(static_cast<size_t>(nq) + 1, 0);
  rows.clear();
  std::vector<Hit> hits;
  size_t at = 0;
  for (int64_t q = 0; q < nq; q++) {
    hits.clear();
    int const qlen = queries->h_len[static_cast<size_t>(q0 + q)];
    int64_t const qsize = o.query_sizes != nullptr ? o.query_sizes[q] : 1;
    // idprefix / idsuffix pass for a query at least that long, selfid never does: the target is identical
    unsigned const content = (qlen < o.idprefix || qlen < o.idsuffix || o.selfid != 0) ? 1u : 0u;
    for (; at < found.size() && static_cast<int64_t>(found[at] >> 32) / strands == q; at++) {
      int const target = static_cast<int>(found[at] & 0xffffffffu);
      int const strand = static_cast<int>((found[at] >> 32) % strands);
      int64_t const tsize = o.target_sizes != nullptr ? o.target_sizes[target] : 1;
      bool const same_label = o.self != 0 && o.query_labels != nullptr && o.target_labels != nullptr &&
                              o.query_labels[q] == o.target_labels[target];
      int const dlen = ix->db->h_len[static_cast<size_t>(target)];
      if (!acceptable_unaligned(o, qlen, dlen, qsize, tsize, same_label, content)) { continue; }
      Hit h{};
      h.target = target;
      h.strand = strand;
      h.nwscore = static_cast<int>(static_cast<int64_t>(qlen) * nwmatch);
      h.nwalignmentlength = qlen;
      h.matches = qlen;
      h.internal_alignmentlength = qlen;
      h.id = h.id0 = h.id1 = h.id2 = h.id3 = h.id4 = 100.0;
      h.shortest = h.longest = qlen;
      h.aligned = true;
      acceptable_aligned(h, 1.0, -1.0, o, qlen, dlen, qsize, tsize);
      if (h.accepted || h.weak) { hits.push_back(h); }
    }
    // the plus strand's hits come first, so a palindrome's two hits on one target keep plus before minus
    std::stable_sort(hits.begin(), hits.end(), hit_less);
    size_t const n = maxhits > 0 ? std::min<size_t>(hits.size(), static_cast<size_t>(maxhits)) : hits.size();
    for (size_t k = 0; k < n; k++) {
      Hit const & h = hits[k];
      vsg_search_result r{};
      r.target = h.target; r.matches = h.matches; r.mismatches = 0; r.gaps = 0; r.alignment_length = qlen;
      r.query_length = qlen; r.target_length = qlen; r.accepted = h.accepted ? 1 : 0; r.strand = h.strand;
      r.nwscore = h.nwscore; r.id = h.id; r.internal_alignment_length = qlen; r.internal_gaps = 0;
      rows.push_back(r);
    }
    first[static_cast<size_t>(q) + 1] = static_cast<int64_t>(rows.size());
  }
  return VSG_OK;
}

extern "C" int vsg_search_exact(vsg_ctx * c, const vsg_exact_index * ix, const vsg_seqset * queries, int64_t q0, int64_t nq,
                                const vsg_search_opts * opts, int64_t maxhits, vsg_search_result * hits, int64_t cap,
                                int64_t * first, int64_t * nhits)
{
  if (first == nullptr || nhits == nullptr || cap < 0 || (cap > 0 && hits == nullptr)) { Error::set("vsg_search_exact: bad argument"); return VSG_EINVAL; }
  *nhits = 0;
  std::vector<vsg_search_result> rows;
  std::vector<int64_t> f;
  int const rc = search_exact_host(c, ix, queries, q0, nq, opts, maxhits, rows, f);
  if (rc != VSG_OK) { return rc; }
  return hits_out(rows, f, "vsg_search_exact", hits, cap, first, nhits);
}
