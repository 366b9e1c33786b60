// makeudb.cu — making UDB databases (SURVEY.md §8 f3, the writing half of udb.cu): the reference's word index built on
// the device, and the file makeudb_usearch writes.
//
// Replaces
//   makeudb_usearch              (reference commands/makeudb_usearch.cpp:105-273)   upper-case, mask, index, write
//   Dbindex::prepare / add_*     (core/dbindex.cpp:121-255)                          kmercount[4^k] and, per word, the
//                                                                                     ascending numbers of the
//                                                                                     sequences holding it
//   unique_count                 (core/unique.cpp:155-353)                           a word counts once per sequence
// The reference runs DUST and both index passes on one core ("does not support multithreading").
//
// The index is built in RANGES OF WORDS, not of sequences: the sequences stay on the device (as vsg_udb_load keeps
// them), and a range's part of the file's index is complete on its own, so ranges go to the host in word order and
// nothing the size of 4^k is needed on the device.
//   1. window_kernel<HIST>: one warp per sequence; every valid window (no masked symbol) adds 1 to the bin of its word,
//      2^20 bins at most (k <= 10: one word per bin), with one atomic per distinct bin of a warp step (match_any);
//   2. the host cuts the bins into ranges of consecutive words whose windows fit the scratch (two 8-byte keys per
//      window in a quarter of the context's direction-bit budget, at most 1 GiB).  A bin too large for it is binned
//      again at a finer width; a single word too large for it takes step 4;
//   3. per range: window_kernel<EMIT> writes one key ((word - first word of the range) << seqbits | sequence number)
//      per valid window of the range, compacted with one atomic per warp step; a CUB radix sort over the bits a key can
//      have, DeviceSelect::Unique (a word counts once per sequence, and its sequence numbers come out ascending), a
//      split into sequence numbers and words, DeviceRunLengthEncode of the words (the per-word counts).  The sequence
//      numbers are the range's stretch of kmerindex, the runs fill its words in kmercount;
//   4. a word with more windows than a range can hold: window_kernel<FLAG> marks the sequences holding it in a byte per
//      sequence, and DeviceSelect::Flagged over the sequence numbers lists them in order.
// Every range scans all windows once more; at the default budget that is a few scans of HBM-resident symbols per GiB of
// keys, and the sorts dominate the device time.
#include "vsg_internal.h"
#include "rank_steps.cuh"

#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

namespace vsg {

namespace {

constexpr int WIN_WARPS = 8;
constexpr int HIST_BINS_LOG2 = 20;
enum { WIN_HIST = 0, WIN_EMIT = 1, WIN_FLAG = 2 };

// The valid windows of every sequence whose word lies in [w_lo, w_lo + (nbins << shift)): HIST adds them to
// hist[(word - w_lo) >> shift], EMIT appends their keys at keys[*nkeys ...], FLAG (nbins << shift == 1) sets flags[seq].
template <int MODE>
__global__ void __launch_bounds__(WIN_WARPS * 32)
window_kernel(DevSeqs s, int k, int mask_lower, uint32_t w_lo, uint64_t width, int shift, int sbits,
              unsigned long long * __restrict__ hist, uint64_t * __restrict__ keys, unsigned long long * __restrict__ nkeys,
              uint8_t * __restrict__ flags)
{
  int const lane = threadIdx.x & 31;
  int64_t const nwarps = static_cast<int64_t>(gridDim.x) * WIN_WARPS;
  for (int64_t q = static_cast<int64_t>(blockIdx.x) * WIN_WARPS + (threadIdx.x >> 5); q < s.n; q += nwarps) {
    const uint8_t * __restrict__ sym = s.sym + s.off[q];
    int const nwin = s.len[q] - k + 1;
    bool seen = false;   // FLAG: this lane met the word
    for (int p0 = 0; p0 < nwin; p0 += 32) {
      int const p = p0 + lane;
      uint32_t w = 0;
      bool ok = p < nwin && kmer_at(sym, p + k - 1, k, mask_lower, w);
      ok = ok && w >= w_lo && static_cast<uint64_t>(w - w_lo) < width;
      if (MODE == WIN_HIST) {
        uint32_t const bin = ok ? (w - w_lo) >> shift : 0xffffffffu;
        unsigned const same = __match_any_sync(0xffffffffu, bin);
        if (ok && lane == __ffs(same) - 1) { atomicAdd(hist + bin, static_cast<unsigned long long>(__popc(same))); }
      } else if (MODE == WIN_EMIT) {
        unsigned const b = __ballot_sync(0xffffffffu, ok);
        unsigned long long base = 0;
        if (lane == 0 && b != 0) { base = atomicAdd(nkeys, static_cast<unsigned long long>(__popc(b))); }
        base = __shfl_sync(0xffffffffu, base, 0);
        if (ok) {
          keys[base + __popc(b & ((1u << lane) - 1u))] = (static_cast<uint64_t>(w - w_lo) << sbits) | static_cast<uint64_t>(q);
        }
      } else {
        seen |= ok;
      }
    }
    if (MODE == WIN_FLAG && __any_sync(0xffffffffu, seen) && lane == 0) { flags[q] = 1; }
  }
}

// the unique keys of a range: sequence numbers and words
__global__ void split_kernel(const uint64_t * __restrict__ keys, int n, int sbits, uint32_t w_lo, uint32_t * __restrict__ seqno,
                             uint32_t * __restrict__ word)
{
  int const i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) { return; }
  uint64_t const key = keys[i];
  seqno[i] = static_cast<uint32_t>(key & ((static_cast<uint64_t>(1) << sbits) - 1u));
  word[i] = w_lo + static_cast<uint32_t>(key >> sbits);
}

int bits_for(uint64_t m)   // the bits that hold 0 .. m
{
  int b = 1;
  while (b < 64 && (static_cast<uint64_t>(1) << b) <= m) { b++; }
  return b;
}

size_t up16(size_t x) { return (x + 15) & ~static_cast<size_t>(15); }

// The word index of the sequences of `s` at word length k into kmercount (4^k, zeroed) and kmerindex.
struct IndexBuilder {
  vsg_ctx * c;
  DevSeqs s;
  int k, mask_lower, sbits, grid;
  size_t cap;   // keys per range
  std::vector<uint32_t> & kmercount;
  std::vector<uint32_t> & kmerindex;
  DevBuf keys, small, flags;   // small: histogram / counters

  template <int MODE>
  void launch(uint32_t w_lo, uint64_t width, int shift, unsigned long long * hist, uint64_t * kp, unsigned long long * nk,
              uint8_t * fl)
  {
    window_kernel<MODE><<<grid, WIN_WARPS * 32, 0, c->stream>>>(s, k, mask_lower, w_lo, width, shift, sbits, hist, kp, nk, fl);
    count_launch();
  }

  // the valid windows of [w_lo, w_lo + width) in bins of 2^shift words
  int histogram(uint32_t w_lo, uint64_t width, int & shift, std::vector<uint64_t> & h)
  {
    shift = 0;
    while ((width >> shift) > (static_cast<uint64_t>(1) << HIST_BINS_LOG2)) { shift++; }
    size_t const nbins = static_cast<size_t>(width >> shift);
    int rc = small.reserve(sizeof(unsigned long long) * (nbins + 2));
    if (rc != VSG_OK) { return rc; }
    auto * const d = static_cast<unsigned long long *>(small.p);
    VSG_CUDA_OK(cudaMemsetAsync(d, 0, sizeof(unsigned long long) * nbins, c->stream));
    launch<WIN_HIST>(w_lo, width, shift, d, nullptr, nullptr, nullptr);
    h.resize(nbins);
    VSG_CUDA_OK(cudaMemcpyAsync(h.data(), d, sizeof(uint64_t) * nbins, cudaMemcpyDeviceToHost, c->stream));
    VSG_CUDA_OK(cudaStreamSynchronize(c->stream));
    VSG_CUDA_OK(cudaGetLastError());
    return VSG_OK;
  }

  // steps 3: the words [w_lo, w_hi), which have n valid windows (0 < n <= cap)
  int range(uint32_t w_lo, uint32_t w_hi, uint64_t n)
  {
    int const wbits = bits_for(w_hi - w_lo - 1);
    int const end_bit = sbits + wbits;
    int const ni = static_cast<int>(n);
    size_t const half = up16(sizeof(uint64_t) * n);
    int rc = keys.reserve(2 * half);
    if (rc != VSG_OK) { return rc; }
    if ((rc = small.reserve(64)) != VSG_OK) { return rc; }
    auto * const a = static_cast<uint64_t *>(keys.p);
    auto * const b = reinterpret_cast<uint64_t *>(static_cast<char *>(keys.p) + half);
    auto * const cnt = static_cast<unsigned long long *>(small.p);   // [0] keys written, [1] unique keys, [2] runs
    auto * const sel = reinterpret_cast<int *>(cnt + 1);
    auto * const runs = reinterpret_cast<int *>(cnt + 2);
    VSG_CUDA_OK(cudaMemsetAsync(cnt, 0, 3 * sizeof(unsigned long long), c->stream));
    launch<WIN_EMIT>(w_lo, w_hi - w_lo, 0, nullptr, a, cnt, nullptr);
    cub::DoubleBuffer<uint64_t> db(a, b);
    size_t t_sort = 0, t_uniq = 0, t_rle = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, t_sort, db, ni, 0, end_bit, c->stream);
    cub::DeviceSelect::Unique(nullptr, t_uniq, a, b, sel, ni, c->stream);
    cub::DeviceRunLengthEncode::Encode(nullptr, t_rle, reinterpret_cast<uint32_t *>(a), reinterpret_cast<uint32_t *>(b),
                                       reinterpret_cast<uint32_t *>(b), runs, ni, c->stream);
    if ((rc = c->cub_tmp.reserve(std::max(t_sort, std::max(t_uniq, t_rle)) + 16)) != VSG_OK) { return rc; }
    VSG_CUDA_OK(cub::DeviceRadixSort::SortKeys(c->cub_tmp.p, t_sort, db, ni, 0, end_bit, c->stream));
    uint64_t * const x = db.Current();
    uint64_t * const y = db.Alternate();
    VSG_CUDA_OK(cub::DeviceSelect::Unique(c->cub_tmp.p, t_uniq, x, y, sel, ni, c->stream));
    count_launch(2);
    int u = 0;
    VSG_CUDA_OK(cudaMemcpyAsync(&u, sel, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    VSG_CUDA_OK(cudaStreamSynchronize(c->stream));
    // x: seqno[u] then word[u] (u32, x holds 2n of them); y: the runs' words and counts
    auto * const seqno = reinterpret_cast<uint32_t *>(x);
    auto * const word = seqno + n;
    auto * const rword = reinterpret_cast<uint32_t *>(y);
    auto * const rcount = rword + n;
    split_kernel<<<(u + 255) / 256, 256, 0, c->stream>>>(y, u, sbits, w_lo, seqno, word);
    count_launch();
    VSG_CUDA_OK(cub::DeviceRunLengthEncode::Encode(c->cub_tmp.p, t_rle, word, rword, rcount, runs, u, c->stream));
    count_launch();
    int nr = 0;
    VSG_CUDA_OK(cudaMemcpyAsync(&nr, runs, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    VSG_CUDA_OK(cudaStreamSynchronize(c->stream));
    std::vector<uint32_t> hw(static_cast<size_t>(nr)), hc(static_cast<size_t>(nr));
    size_t const pos = kmerindex.size();
    kmerindex.resize(pos + static_cast<size_t>(u));
    VSG_CUDA_OK(cudaMemcpyAsync(kmerindex.data() + pos, seqno, sizeof(uint32_t) * u, cudaMemcpyDeviceToHost, c->stream));
    VSG_CUDA_OK(cudaMemcpyAsync(hw.data(), rword, sizeof(uint32_t) * nr, cudaMemcpyDeviceToHost, c->stream));
    VSG_CUDA_OK(cudaMemcpyAsync(hc.data(), rcount, sizeof(uint32_t) * nr, cudaMemcpyDeviceToHost, c->stream));
    VSG_CUDA_OK(cudaStreamSynchronize(c->stream));
    VSG_CUDA_OK(cudaGetLastError());
    for (int i = 0; i < nr; i++) { kmercount[hw[static_cast<size_t>(i)]] = hc[static_cast<size_t>(i)]; }
    return VSG_OK;
  }

  // step 4: the one word w
  int single(uint32_t w)
  {
    size_t const nseq = static_cast<size_t>(s.n);
    int rc = flags.reserve(up16(nseq) + sizeof(uint32_t) * nseq);
    if (rc != VSG_OK) { return rc; }
    if ((rc = small.reserve(64)) != VSG_OK) { return rc; }
    auto * const fl = static_cast<uint8_t *>(flags.p);
    auto * const out = reinterpret_cast<uint32_t *>(static_cast<char *>(flags.p) + up16(nseq));
    auto * const sel = static_cast<int *>(small.p);
    VSG_CUDA_OK(cudaMemsetAsync(fl, 0, nseq, c->stream));
    launch<WIN_FLAG>(w, 1, 0, nullptr, nullptr, nullptr, fl);
    thrust::counting_iterator<uint32_t> seqnos(0);
    size_t tb = 0;
    cub::DeviceSelect::Flagged(nullptr, tb, seqnos, fl, out, sel, static_cast<int>(nseq), c->stream);
    if ((rc = c->cub_tmp.reserve(tb + 16)) != VSG_OK) { return rc; }
    VSG_CUDA_OK(cub::DeviceSelect::Flagged(c->cub_tmp.p, tb, seqnos, fl, out, sel, static_cast<int>(nseq), c->stream));
    count_launch();
    int u = 0;
    VSG_CUDA_OK(cudaMemcpyAsync(&u, sel, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    VSG_CUDA_OK(cudaStreamSynchronize(c->stream));
    size_t const pos = kmerindex.size();
    kmerindex.resize(pos + static_cast<size_t>(u));
    VSG_CUDA_OK(cudaMemcpyAsync(kmerindex.data() + pos, out, sizeof(uint32_t) * u, cudaMemcpyDeviceToHost, c->stream));
    VSG_CUDA_OK(cudaStreamSynchronize(c->stream));
    VSG_CUDA_OK(cudaGetLastError());
    kmercount[w] = static_cast<uint32_t>(u);
    return VSG_OK;
  }

  // steps 1, 2: the words [w_lo, w_lo + width) in order
  int build(uint32_t w_lo, uint64_t width, bool top)
  {
    std::vector<uint64_t> h;
    int shift = 0;
    int rc = histogram(w_lo, width, shift, h);
    if (rc != VSG_OK) { return rc; }
    if (top) {   // an upper bound on the index's size (a word repeated in a sequence counts once there)
      uint64_t total = 0;
      for (uint64_t v : h) { total += v; }
      kmerindex.reserve(static_cast<size_t>(total));
    }
    uint64_t const bw = static_cast<uint64_t>(1) << shift;
    uint64_t g_lo = w_lo, acc = 0;
    auto flush = [&](uint64_t hi) { int r = acc > 0 ? range(static_cast<uint32_t>(g_lo), static_cast<uint32_t>(hi), acc) : VSG_OK; acc = 0; return r; };
    for (size_t i = 0; i < h.size(); i++) {
      uint64_t const b_lo = w_lo + i * bw;
      if (h[i] > cap) {
        if ((rc = flush(b_lo)) != VSG_OK) { return rc; }
        rc = (bw == 1) ? single(static_cast<uint32_t>(b_lo)) : build(static_cast<uint32_t>(b_lo), bw, false);
        if (rc != VSG_OK) { return rc; }
        g_lo = b_lo + bw;
      } else {
        if (acc + h[i] > cap) {
          if ((rc = flush(b_lo)) != VSG_OK) { return rc; }
          g_lo = b_lo;
        }
        acc += h[i];
      }
    }
    return flush(w_lo + width);
  }
};

// db.read(..., upcase = 1): chrmap_upcase (utils/maps.cpp) — letters to upper case, any other byte to 'N'
struct Upcase {
  char map[256];
  Upcase()
  {
    for (int i = 0; i < 256; i++) { map[i] = 'N'; }
    for (int i = 'A'; i <= 'Z'; i++) { map[i] = static_cast<char>(i); map[i + 32] = static_cast<char>(i); }
  }
};

int check_opts(const vsg_makeudb_opts * o, const char * caller)
{
  if (o->wordlength < 3 || o->wordlength > 15) {
    Error::set(std::string(caller) + ": wordlength " + std::to_string(o->wordlength) + " is outside 3..15");
    return VSG_EINVAL;
  }
  if (o->dbmask != VSG_DBMASK_NONE && o->dbmask != VSG_DBMASK_SOFT && o->dbmask != VSG_DBMASK_DUST) {
    Error::set(std::string(caller) + ": unknown dbmask " + std::to_string(o->dbmask) + " (none 0, soft 1, dust 2)");
    return VSG_EINVAL;
  }
  return VSG_OK;
}

}  // namespace

int makeudb_check_opts(const vsg_makeudb_opts * o, const char * caller) { return check_opts(o, caller); }

}  // namespace vsg

using namespace vsg;

extern "C" void vsg_makeudb_opts_default(vsg_makeudb_opts * o)
{
  if (o == nullptr) { return; }
  o->wordlength = 8;
  o->dbmask = VSG_DBMASK_DUST;
  o->hardmask = 0;
  o->notrunclabels = 0;
  o->minseqlength = 32;     // cli.cc: --makeudb_usearch's default
  o->maxseqlength = 50000;
}

extern "C" int vsg_udb_make(vsg_ctx * c, const char * cat, const int64_t * off, const int32_t * len, const char * const * headers,
                            int64_t n, const vsg_makeudb_opts * opts, vsg_udb ** out)
{
  if (c == nullptr || opts == nullptr || out == nullptr || (n > 0 && (cat == nullptr || off == nullptr || len == nullptr || headers == nullptr))) {
    Error::set("vsg_udb_make: null argument");
    return VSG_EINVAL;
  }
  *out = nullptr;
  int rc = check_opts(opts, "vsg_udb_make");
  if (rc != VSG_OK) { return rc; }
  if (n < 0 || n > INT32_MAX) { Error::set("vsg_udb_make: the sequence count is outside 0..2^31-1"); return VSG_EINVAL; }
  std::unique_ptr<vsg_udb> u(new (std::nothrow) vsg_udb());
  if (!u) { Error::set("out of host memory"); return VSG_ENOMEM; }
  int const k = opts->wordlength;

  // sequences (upper-cased) and headers, as the file holds them
  static Upcase const up;
  uint64_t nt = 0, hc = 0;
  int64_t longest_header = 0;
  int32_t shortest = 0, longest = 0;
  for (int64_t i = 0; i < n; i++) {
    if (len[i] < 0) { Error::set("vsg_udb_make: negative sequence length"); return VSG_EINVAL; }
    nt += static_cast<uint64_t>(len[i]);
    int64_t const hl = static_cast<int64_t>(std::strlen(headers[i]));
    hc += static_cast<uint64_t>(hl) + 1;
    longest_header = std::max(longest_header, hl);
    shortest = i == 0 ? len[i] : std::min(shortest, len[i]);
    longest = std::max(longest, len[i]);
  }
  if (hc > UINT32_MAX) { Error::set("vsg_udb_make: the headers exceed the file's 32-bit header offsets"); return VSG_EINVAL; }
  u->cat.resize(static_cast<size_t>(nt) + 1);
  u->off.resize(static_cast<size_t>(n));
  u->len.assign(len, len + n);
  u->headers.resize(static_cast<size_t>(hc) + 1);
  u->header_off.resize(static_cast<size_t>(n) + 1);
  {
    uint64_t p = 0, h = 0;
    for (int64_t i = 0; i < n; i++) {
      const unsigned char * src = reinterpret_cast<const unsigned char *>(cat + off[i]);
      char * dst = u->cat.data() + p;
      for (int32_t j = 0; j < len[i]; j++) { dst[j] = up.map[src[j]]; }
      u->off[static_cast<size_t>(i)] = static_cast<int64_t>(p);
      p += static_cast<uint64_t>(len[i]);
      size_t const hl = std::strlen(headers[i]);
      u->header_off[static_cast<size_t>(i)] = static_cast<uint32_t>(h);
      std::memcpy(u->headers.data() + h, headers[i], hl + 1);
      h += hl + 1;
    }
    u->header_off[static_cast<size_t>(n)] = static_cast<uint32_t>(h);
    u->cat[static_cast<size_t>(nt)] = '\0';
    u->headers[static_cast<size_t>(hc)] = '\0';
  }
  u->info.sequences = n;
  u->info.nucleotides = static_cast<int64_t>(nt);
  u->info.header_chars = static_cast<int64_t>(hc);
  u->info.longest_header = longest_header;
  u->info.wordlength = k;
  u->info.dbaccel = 100;
  u->info.shortest = shortest;
  u->info.longest = longest;
  u->kmercount.assign(static_cast<size_t>(1) << (2 * k), 0u);

  if (n > 0) {
    VSG_CUDA_OK(cudaSetDevice(c->device));
    vsg_seqset * raw = nullptr;
    if ((rc = vsg_seqset_create(c, u->cat.data(), u->off.data(), u->len.data(), n, 1, &raw)) != VSG_OK) { return rc; }
    SeqsetPtr s(raw);
    if (opts->dbmask == VSG_DBMASK_DUST) {
      // DUST on the device, then its mask onto the file's bytes: lower case, or 'N' with --hardmask (dust_core)
      if ((rc = vsg_seqset_dust(c, s.get())) != VSG_OK) { return rc; }
      std::vector<uint8_t> sym(static_cast<size_t>(nt));
      if ((rc = vsg_seqset_symbols(c, s.get(), sym.data(), static_cast<int64_t>(nt))) != VSG_OK) { return rc; }
      char * const a = u->cat.data();
      if (opts->hardmask != 0) {
        for (size_t i = 0; i < sym.size(); i++) { if (sym[i] & 0x10) { a[i] = 'N'; } }
      } else {
        for (size_t i = 0; i < sym.size(); i++) { a[i] = static_cast<char>(a[i] | (sym[i] & 0x10) << 1); }
      }
    }
    // --dbmask none: windows with a symbol outside ACGTU are skipped; soft / dust: lower case too (Dbindex::prepare's
    // seqmask).  With --hardmask the masked symbols are 'N' in the file and lower case on the device: the same windows.
    int const mask_lower = opts->dbmask != VSG_DBMASK_NONE ? 1 : 0;
    // scratch: two 8-byte keys per window of a range in a quarter of the direction-bit budget, capped at 1 GiB
    size_t const budget = std::min<size_t>(c->dir_budget / 4, static_cast<size_t>(1) << 30);
    size_t const cap = std::max<size_t>(budget / (2 * sizeof(uint64_t)), 1024);
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device);
    IndexBuilder b{c, s->d, k, mask_lower, bits_for(static_cast<uint64_t>(n - 1)), sms * 16, cap, u->kmercount, u->kmerindex};
    rc = b.build(0, static_cast<uint64_t>(1) << (2 * k), true);
    b.keys.release(); b.small.release(); b.flags.release();
    if (rc != VSG_OK) { return rc; }
  }
  u->info.index_entries = static_cast<int64_t>(u->kmerindex.size());
  *out = u.release();
  return VSG_OK;
}

namespace {

// largewrite (makeudb_usearch.cpp:82-100): blocks of 16 MiB
bool write_all(std::FILE * f, const void * p, uint64_t n)
{
  for (uint64_t i = 0; i < n; i += 4096ull * 4096ull) {
    size_t const r = static_cast<size_t>(std::min<uint64_t>(4096ull * 4096ull, n - i));
    if (std::fwrite(static_cast<const char *>(p) + i, 1, r, f) != r) { return false; }
  }
  return true;
}

}  // namespace

extern "C" int vsg_udb_write(const vsg_udb * u, const char * path)
{
  if (u == nullptr || path == nullptr) { Error::set("vsg_udb_write: null argument"); return VSG_EINVAL; }
  std::FILE * f = std::fopen(path, "wb");
  if (f == nullptr) { Error::set(std::string("vsg_udb_write: unable to open output file for writing (") + path + ")"); return VSG_EINVAL; }
  uint32_t const seqcount = static_cast<uint32_t>(u->info.sequences);
  uint64_t const nt = static_cast<uint64_t>(u->info.nucleotides), hc = static_cast<uint64_t>(u->info.header_chars);
  uint32_t head[50] = {};
  head[0] = 0x55444246u;   // UDBF
  head[2] = 32;            // bits
  head[4] = static_cast<uint32_t>(u->info.wordlength);
  head[5] = 1;             // dbstep
  head[6] = static_cast<uint32_t>(u->info.dbaccel);
  head[13] = seqcount;
  head[17] = 0x0000746eu;  // "nt"
  head[49] = 0x55444266u;  // UDBf
  uint32_t const sig3 = 0x55444233u;
  uint32_t const head2[8] = {0x55444234u, 0x005e0db3u, seqcount, static_cast<uint32_t>(nt), static_cast<uint32_t>(nt >> 32),
                             static_cast<uint32_t>(hc), static_cast<uint32_t>(hc >> 32), 0x005e0db4u};
  std::vector<uint32_t> lens(u->len.begin(), u->len.end());
  bool ok = write_all(f, head, sizeof head) &&
            write_all(f, u->kmercount.data(), sizeof(uint32_t) * u->kmercount.size()) &&
            write_all(f, &sig3, sizeof sig3) &&
            write_all(f, u->kmerindex.data(), sizeof(uint32_t) * u->kmerindex.size()) &&
            write_all(f, head2, sizeof head2) &&
            write_all(f, u->header_off.data(), sizeof(uint32_t) * seqcount) &&
            write_all(f, u->headers.data(), hc) &&
            write_all(f, lens.data(), sizeof(uint32_t) * lens.size()) &&
            write_all(f, u->cat.data(), nt);
  ok = (std::fclose(f) == 0) && ok;
  if (!ok) {
    std::remove(path);
    Error::set(std::string("vsg_udb_write: unable to write to UDB file (") + path + ")");
    return VSG_EINVAL;
  }
  return VSG_OK;
}
