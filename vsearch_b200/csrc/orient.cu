// orient.cu — read orientation against the static k-mer index (sm_90a).
//
// Replaces, for whole batches of reads at once, the body of the read loop of orient() (reference
// commands/orient.cpp:224-312):
//   unique_count(..., opt_qmask)   (core/unique.cpp:155-353)     the distinct k-mers of the read
//   rc_kmer                        (commands/orient.cpp:90-113)  the reverse complement of a k-mer
//   Dbindex::getmatchcount         (core/dbindex.hpp)            the number of database sequences holding a k-mer
//   the 8x vote per k-mer and the 4x decision per read
//
// One path for every read length.  The reads of a call are cut into launches whose windows fit a share of the
// context's memory budget, and each launch runs
//   1. orient_keys_kernel: one 64-bit key (read << 2k | k-mer) per window, all ones for a window with a masked symbol;
//   2. a CUB radix sort of the keys over the bits a valid key can have, so the masked windows sort last;
//   3. orient_vote_kernel: one thread per key.  A key that differs from its predecessor is a distinct k-mer of its read:
//      two lookups in the index's word-count table (index_word_counts) and the vote, summed per read over the warp
//      (match_any on the read: the keys are sorted, so a read's keys are neighbours) with one atomic per read and warp;
//   4. orient_finish_kernel: the decision per read.
#include "vsg_internal.h"
#include "rank_steps.cuh"

#include <cub/cub.cuh>

#include <algorithm>
#include <string>
#include <vector>

namespace vsg {

namespace {

constexpr uint64_t KEY_MASKED = ~0ull;
constexpr int KEY_THREADS = 256;
constexpr int VOTE_THREADS = 256;
constexpr uint32_t HITS_FACTOR = 8, MIN_FACTOR = 4;   // orient.cpp:237, 269

// rc_kmer: the complement of every 2-bit symbol, in reverse order.  __brev reverses the symbols and swaps the two bits
// of each; the swap undoes the latter, the shift drops the symbols above k.
__device__ __forceinline__ uint32_t rc_kmer(uint32_t w, int k)
{
  uint32_t x = __brev(~w);
  x = ((x >> 1) & 0x55555555u) | ((x & 0x55555555u) << 1);
  return x >> (32 - 2 * k);
}

// 1. read qi of the launch (sequence q0 + qi) writes its windows' keys at keys[woff[qi] ...]
__global__ void __launch_bounds__(KEY_THREADS)
orient_keys_kernel(DevSeqs qs, int64_t q0, int nq, int k, int mask_lower, const int64_t * __restrict__ woff,
                   uint64_t * __restrict__ keys)
{
  for (int qi = blockIdx.x; qi < nq; qi += gridDim.x) {
    const uint8_t * __restrict__ s = qs.sym + qs.off[q0 + qi];
    int64_t const base = woff[qi];
    int const nwin = static_cast<int>(woff[qi + 1] - base);
    for (int p = threadIdx.x; p < nwin; p += blockDim.x) {
      uint32_t v;
      keys[base + p] = kmer_at(s, p + k - 1, k, mask_lower, v) ? (static_cast<uint64_t>(qi) << (2 * k)) | v : KEY_MASKED;
    }
  }
}

// 3. the vote of every distinct (read, k-mer) key of the sorted keys[0, n)
__global__ void __launch_bounds__(VOTE_THREADS)
orient_vote_kernel(const uint64_t * __restrict__ keys, int64_t n, int k, const uint32_t * __restrict__ words,
                   uint32_t * __restrict__ fwd, uint32_t * __restrict__ rev)
{
  int64_t const i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  uint64_t const key = i < n ? keys[i] : KEY_MASKED;
  uint32_t q = 0xffffffffu;   // the read of a distinct k-mer; no read for masked keys and repeats
  bool f = false, r = false;
  if (key != KEY_MASKED && (i == 0 || keys[i - 1] != key)) {
    uint32_t const w = static_cast<uint32_t>(key) & ((1u << (2 * k)) - 1u);
    uint32_t const hf = words[w], hr = words[rc_kmer(w, k)];
    q = static_cast<uint32_t>(key >> (2 * k));
    f = hf > HITS_FACTOR * hr;
    r = !f && hr > HITS_FACTOR * hf;
  }
  unsigned const same = __match_any_sync(0xffffffffu, q);
  unsigned const bf = __ballot_sync(0xffffffffu, f), br = __ballot_sync(0xffffffffu, r);
  if (q != 0xffffffffu && static_cast<int>(threadIdx.x & 31) == __ffs(same) - 1) {
    int const nf = __popc(bf & same), nr = __popc(br & same);
    if (nf > 0) { atomicAdd(fwd + q, static_cast<uint32_t>(nf)); }
    if (nr > 0) { atomicAdd(rev + q, static_cast<uint32_t>(nr)); }
  }
}

// 4. the decision (orient.cpp:265-312), in the reference's unsigned arithmetic
__global__ void orient_finish_kernel(int nq, const uint32_t * __restrict__ fwd, const uint32_t * __restrict__ rev,
                                     vsg_orient_result * __restrict__ out)
{
  int const i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nq) { return; }
  uint32_t const f = fwd[i], r = rev[i];
  vsg_orient_result o;
  o.strand = (f >= 1u && f >= MIN_FACTOR * r) ? 0 : (r >= 1u && r >= MIN_FACTOR * f) ? 1 : 2;
  o.count_fwd = f;
  o.count_rev = r;
  out[i] = o;
}

int bits_for(int64_t m)   // the bits that hold 0 .. m
{
  int b = 1;
  while ((static_cast<int64_t>(1) << b) <= m) { b++; }
  return b;
}

}  // namespace

}  // namespace vsg

using namespace vsg;

extern "C" int vsg_orient(vsg_ctx * c, const vsg_index * ix, const vsg_seqset * queries, int64_t q0, int64_t nq,
                          int query_mask_lower, vsg_orient_result * out)
{
  if (c == nullptr || ix == nullptr || queries == nullptr || (out == nullptr && nq > 0)) {
    Error::set("vsg_orient: null argument");
    return VSG_EINVAL;
  }
  if (q0 < 0 || nq < 0 || q0 > queries->d.n || nq > queries->d.n - q0) { Error::set("vsg_orient: query range out of bounds"); return VSG_EINVAL; }
  if (queries->device != c->device || index_db(ix)->device != c->device) {
    Error::set("vsg_orient: sequence set / index lives on another device than the context");
    return VSG_EINVAL;
  }
  if (nq == 0) { return VSG_OK; }
  VSG_CUDA_OK(cudaSetDevice(c->device));
  int const k = index_wordlength(ix);
  const uint32_t * d_words = nullptr;
  int rc = index_word_counts(c, ix, &d_words);
  if (rc != VSG_OK) { return rc; }
  int sms = 132;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device);
  // Launches of consecutive reads whose keys (two 8-byte buffers per window for the sort) fit a quarter of the context's
  // direction-bit budget (a share of the device's free memory, vsg_ctx_create), capped at 1 GiB.  A read longer than
  // that goes alone.
  size_t const budget = std::min<size_t>(c->dir_budget / 4, static_cast<size_t>(1) << 30);
  size_t const max_windows = std::max<size_t>(budget / (2 * sizeof(uint64_t)), 1);
  std::vector<int64_t> woff;
  for (int64_t a = 0; a < nq;) {
    woff.assign(1, 0);
    int64_t b = a;
    while (b < nq) {
      int64_t const win = std::max(0, queries->h_len[static_cast<size_t>(q0 + b)] - k + 1);
      if (b > a && (static_cast<size_t>(woff.back() + win) > max_windows || b - a >= (1 << 20))) { break; }
      woff.push_back(woff.back() + win);
      b++;
    }
    int const m = static_cast<int>(b - a);
    int64_t const n = woff.back();   // < 2^31: one read's windows, or at most max_windows
    // rank_tmp: [woff m+1][keys0 n][keys1 n][fwd m][rev m][results m]
    auto up16 = [](size_t x) { return (x + 15) & ~static_cast<size_t>(15); };
    size_t const woff_b = sizeof(int64_t) * (static_cast<size_t>(m) + 1);
    size_t const keys_b = sizeof(uint64_t) * (static_cast<size_t>(n) + 1);
    size_t const cnt_b = sizeof(uint32_t) * static_cast<size_t>(m);
    size_t const res_b = sizeof(vsg_orient_result) * static_cast<size_t>(m);
    if ((rc = c->rank_tmp.reserve(up16(woff_b) + 2 * up16(keys_b) + 2 * up16(cnt_b) + up16(res_b))) != VSG_OK) { return rc; }
    unsigned char * p = static_cast<unsigned char *>(c->rank_tmp.p);
    int64_t * const d_woff = reinterpret_cast<int64_t *>(p); p += up16(woff_b);
    uint64_t * const d_keys0 = reinterpret_cast<uint64_t *>(p); p += up16(keys_b);
    uint64_t * const d_keys1 = reinterpret_cast<uint64_t *>(p); p += up16(keys_b);
    uint32_t * const d_fwd = reinterpret_cast<uint32_t *>(p); p += up16(cnt_b);
    uint32_t * const d_rev = reinterpret_cast<uint32_t *>(p); p += up16(cnt_b);
    vsg_orient_result * const d_res = reinterpret_cast<vsg_orient_result *>(p);
    int const end_bit = 2 * k + bits_for(m);   // a valid key is below m << 2k; the masked key has every bit set
    cub::DoubleBuffer<uint64_t> sorted(d_keys0, d_keys1);
    size_t tb = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, tb, sorted, static_cast<int>(n), 0, end_bit, c->stream);
    if ((rc = c->cub_tmp.reserve(tb + 16)) != VSG_OK) { return rc; }
    VSG_CUDA_OK(cudaMemcpyAsync(d_woff, woff.data(), woff_b, cudaMemcpyHostToDevice, c->stream));
    VSG_CUDA_OK(cudaMemsetAsync(d_fwd, 0, 2 * up16(cnt_b), c->stream));
    VSG_CUDA_OK(cudaEventRecord(c->ev[4], c->stream));
    if (n > 0) {
      orient_keys_kernel<<<std::min(m, sms * 8), KEY_THREADS, 0, c->stream>>>(queries->d, q0 + a, m, k, query_mask_lower != 0 ? 1 : 0,
                                                                             d_woff, d_keys0);
      count_launch();
      VSG_CUDA_OK(cub::DeviceRadixSort::SortKeys(c->cub_tmp.p, tb, sorted, static_cast<int>(n), 0, end_bit, c->stream));
      count_launch();
      orient_vote_kernel<<<static_cast<unsigned>((n + VOTE_THREADS - 1) / VOTE_THREADS), VOTE_THREADS, 0, c->stream>>>(
          sorted.Current(), n, k, d_words, d_fwd, d_rev);
      count_launch();
    }
    orient_finish_kernel<<<(m + 255) / 256, 256, 0, c->stream>>>(m, d_fwd, d_rev, d_res);
    count_launch();
    VSG_CUDA_OK(cudaEventRecord(c->ev[5], c->stream));
    VSG_CUDA_OK(cudaMemcpyAsync(out + a, d_res, res_b, cudaMemcpyDeviceToHost, c->stream));
    VSG_CUDA_OK(cudaStreamSynchronize(c->stream));
    VSG_CUDA_OK(cudaGetLastError());
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, c->ev[4], c->ev[5]) == cudaSuccess) { c->prof_rank_ms += ms; }   // vsg_profile.rank_ms
    a = b;
  }
  return VSG_OK;
}
