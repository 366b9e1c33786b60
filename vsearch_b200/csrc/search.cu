// search.cu — the per-query accept/reject driver on top of the device ranker and aligner.
//
// Replaces search_batch (reference core/search.hpp:135-145, core/search.cpp:397-593), i.e. for every
// query: search_onequery (core/searchcore.cpp:884-957) -> align_delayed (:740-881) -> align_trim
// (:343-464) -> search_acceptable_aligned (:664-737) -> search_joinhits (:1028-1052).
//
// The reference walks one query at a time and aligns its candidates in groups of MAXDELAYED = 8
// (searchcore.hpp:71).  Here every query of a batch advances in lock step: each ROUND gathers, for
// all still-active queries, exactly the group of <= 8 candidates the reference would hand to search16
// next, aligns all groups of the round in one batched device call, and then replays the reference's
// sequential accept/reject bookkeeping on the results.  The set of pairs aligned, the order in which
// hits are examined and every counter are those of the reference, so the hit tables are identical.
#include "vsg_internal.h"
#include "hit_logic.h"
#include "workers.h"

#include <algorithm>
#include <atomic>
#include <cmath>
#include <climits>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <chrono>
#include <cstdio>
#include <functional>

using namespace vsg;

namespace {

struct QState {
  int strand = 0, qlen = 0;
  int64_t ql = 0;  // the query's index in the batch
  int ncand = 0, next = 0;
  const uint32_t * cs = nullptr;
  const uint32_t * cc = nullptr;
  const uint8_t * cf = nullptr;  // per-candidate device verdicts of the sequence-content filters (0 = pass)
  int64_t hit_base = 0;  // index of this state's first Hit in the batch-wide hit array (room for ncand)
  int hit_count = 0, accepts = 0, rejects = 0, finalized = 0, delayed = 0;
  int gpos = -1;  // lazy mode: next hit of the open group to examine (-1: no group open)
  int gend = 0, greq = 0;  // lazy mode: end of the requested hit range, number of pairs requested
  int cache_first = -1, cache_off = 0;  // tail mode: results of hits >= cache_first sit at tail cache[cache_off + x - cache_first]
  bool done = false, waiting = false;
};

struct SearchScratch {  // per host thread, see vsg_ctx::search_scratch
  std::vector<uint32_t> h_seqno, h_count;
  std::vector<uint8_t> h_flags;
  std::vector<int32_t> h_n;
  std::vector<int64_t> cfirst;   // state i's candidates are h_seqno / h_count / h_flags[cfirst[i] ...], h_n[i] of them
  std::vector<int64_t> lfirst;   // unbounded ranker: one strand's lists (rank_lists)
  std::vector<uint32_t> lseq, lcnt;
  std::vector<QState> st;
  Hit * hits = nullptr;
  size_t hits_cap = 0;
  std::vector<uint32_t> pq, pt, lq, lt;
  std::vector<int> pstate, px, lstate;
  std::vector<int32_t> plead, lead_tmp;   // traceback on demand: each pair's group leader (index into the round's pair list) or -1
  std::vector<int64_t> ldest;
  PairResults a, l, t;  // the round's pairs; tail mode: its one device call, the cache later rounds replay from
  std::vector<Hit> joined;
  SearchScratch() = default;
  SearchScratch(const SearchScratch &) = delete;
  SearchScratch & operator=(const SearchScratch &) = delete;
  ~SearchScratch() { std::free(hits); }
};

// idprefix / idsuffix / selfid of search_acceptable_unaligned (searchcore.cpp:588-607) for every candidate
// of every query of a ranked batch: one warp per (query, candidate) compares 4-bit codes as seqcmp does
// (utils/seqcmp.cpp:72-92).  flags: 1 = idprefix fails, 2 = idsuffix fails, 4 = selfid fails.
// Candidate lists at a stride of tophits (ncand[qi] of them valid), or, with first != nullptr, back to back: query qi's
// are cand[first[qi] .. first[qi + 1]).
__global__ void prefilter_kernel(DevSeqs qs, int64_t q0, int nq, DevSeqs db, const uint32_t * __restrict__ cand,
                                 const int32_t * __restrict__ ncand, int tophits, const int64_t * __restrict__ first,
                                 int idprefix, int idsuffix, int selfid, uint8_t * __restrict__ flags)
{
  int64_t const w = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  int const lane = threadIdx.x & 31;
  int qi;
  if (first == nullptr) {
    if (w >= static_cast<int64_t>(nq) * tophits) { return; }
    qi = static_cast<int>(w / tophits);
    if (static_cast<int>(w % tophits) >= ncand[qi]) { return; }
  } else {
    if (w >= first[nq]) { return; }
    int lo = 0, hi = nq - 1;   // the last query whose list starts at or before w
    while (lo < hi) { int const mid = (lo + hi + 1) >> 1; if (first[mid] <= w) { lo = mid; } else { hi = mid - 1; } }
    qi = lo;
  }
  uint32_t const t = cand[w];
  const uint8_t * __restrict__ q = qs.sym + qs.off[q0 + qi];
  const uint8_t * __restrict__ d = db.sym + db.off[t];
  int const ql = qs.len[q0 + qi], dl = db.len[t];
  auto differ = [&](const uint8_t * a, const uint8_t * b, int n) -> bool {
    int bad = 0;
    for (int i = lane; i < n; i += 32) { bad |= ((a[i] ^ b[i]) & 15) != 0; }
    return __any_sync(0xffffffffu, bad) != 0;
  };
  unsigned f = 0;
  if (idprefix > 0 && (ql < idprefix || dl < idprefix || differ(q, d, idprefix))) { f |= 1u; }
  if (idsuffix > 0 && (ql < idsuffix || dl < idsuffix || differ(q + ql - idsuffix, d + dl - idsuffix, idsuffix))) { f |= 2u; }
  if (selfid != 0 && ql == dl && !differ(q, d, ql)) { f |= 4u; }
  if (lane == 0) { flags[w] = static_cast<uint8_t>(f); }
}

}  // namespace

extern "C" void vsg_search_opts_default(vsg_search_opts * o)
{
  if (o == nullptr) { return; }
  o->id = 0.0; o->weak_id = 10.0; o->maxaccepts = 1; o->maxrejects = 32; o->wordlength = 8;
  o->minwordmatches = -1; o->iddef = 2; o->strand_both = 0; o->mask_lower = 0; o->lazy = 0;
  o->minqt = 0.0; o->maxqt = 1.7976931348623157e308; o->minsl = 0.0; o->maxsl = 1.7976931348623157e308;
  o->maxid = 1.0; o->mid = 0.0; o->query_cov = 0.0; o->target_cov = 0.0;
  o->maxsubs = 2147483647; o->maxgaps = 2147483647; o->mincols = 0; o->maxdiffs = 2147483647;
  o->leftjust = 0; o->rightjust = 0;
  o->maxqsize = INT64_MAX; o->mintsize = 0; o->minsizeratio = 0.0; o->maxsizeratio = 1.7976931348623157e308;
  o->idprefix = 0; o->idsuffix = 0; o->self = 0; o->selfid = 0; o->qmask_dust = 0; o->unoise = 0; o->unoise_alpha = 2.0; o->sizeorder = 0; o->reserved1 = 0;
  o->query_sizes = nullptr; o->target_sizes = nullptr; o->query_labels = nullptr; o->target_labels = nullptr;
}

namespace {

// a joined hit list (search_joinhits order) of query q, the index within the call; called once per query, from the
// driver's worker threads
using RowSink = std::function<void(int64_t q, const std::vector<Hit> & joined)>;

// the result record of a hit (search.cpp:466-488)
vsg_search_result result_of(Hit const & h, int qlen, int tlen)
{
  vsg_search_result r;
  r.target = h.target; r.matches = h.matches; r.mismatches = h.mismatches; r.gaps = h.nwgaps;
  r.alignment_length = h.nwalignmentlength;
  r.query_length = qlen;
  r.target_length = tlen;
  r.accepted = h.accepted ? 1 : 0; r.strand = h.strand; r.nwscore = h.nwscore; r.id = h.id;
  r.internal_alignment_length = h.internal_alignmentlength; r.internal_gaps = h.internal_gaps;
  return r;
}

int search_core(vsg_ctx * c, const vsg_index * ix, const vsg_seqset * db, const vsg_seqset * queries, int64_t q0,
                int64_t nq, const vsg_search_opts * opts, RowSink const & sink, int64_t * work)
{
  if (index_db(ix) != db) { Error::set("vsg_search_batch: index was built for another sequence set"); return VSG_EINVAL; }
  if (q0 < 0 || nq < 0 || q0 + nq > queries->d.n) { Error::set("vsg_search_batch: query range out of bounds"); return VSG_EINVAL; }
  if (opts->wordlength != index_wordlength(ix)) { Error::set("vsg_search_batch: wordlength differs from the index"); return VSG_EINVAL; }
  if (opts->iddef < 0 || opts->iddef > 4) { Error::set("vsg_search_batch: iddef must be 0..4"); return VSG_EINVAL; }

  int64_t const seqcount = db->d.n;
  SearchLimits lim;
  if (int const r = search_limits(*opts, seqcount, "vsg_search_batch", lim); r != VSG_OK) { return r; }
  int64_t const maxaccepts = lim.maxaccepts, maxrejects = lim.maxrejects;
  double const opt_id = lim.opt_id, opt_weak_id = lim.opt_weak_id;
  int64_t total_pairs = 0, total_cells = 0, aligned_pairs = 0, aligned_cells = 0;
  bool const lazy = opts->lazy != 0;
  // Traceback on demand (align_ckpt.cuh, TbGate) needs the device's verdict on a group's first candidate to be the
  // host's: that holds when search_acceptable_aligned reduces to its identity test, i.e. every optional
  // post-alignment filter is at its default and no pair can be diverted to the caller's aligner.  VSG_TB_GATE=0 turns
  // it off (A/B runs; the results do not depend on it).
  // VSG_TB_GATE_FORCE=1 (tests): the device takes EVERY leader for accepted, so every follower the replay needs goes
  // through the re-alignment below; =2: EVERY leader is rejected, so every follower is walked (and every score-only
  // checkpoint task re-run with stores, align_ckpt.cuh)
  int const tb_force = [] { const char * e = std::getenv("VSG_TB_GATE_FORCE"); return e != nullptr && (e[0] == '1' || e[0] == '2') ? e[0] - '0' : 0; }();
  bool tb_gate = false;
  {
    vsg_search_opts d;
    vsg_search_opts_default(&d);
    const char * const e = std::getenv("VSG_TB_GATE");
    tb_gate = (e == nullptr || e[0] != '0') && !lazy && !c->sp.fallback &&
              opts->maxsubs == d.maxsubs && opts->maxgaps == d.maxgaps && opts->mincols == d.mincols && opts->maxdiffs == d.maxdiffs &&
              opts->leftjust == 0 && opts->rightjust == 0 && opts->query_cov == d.query_cov && opts->target_cov == d.target_cov &&
              opts->maxid == d.maxid && opts->mid == d.mid && opts->iddef >= 0 && opts->iddef <= 4 && opt_weak_id <= opt_id &&
              opts->unoise == 0;
  }
  if (seqcount == 0 || nq == 0) { if (work) { work[0] = work[1] = work[2] = work[3] = 0; } return VSG_OK; }
  // tophits beyond what the ranker keeps in shared memory: the unbounded ranker's lists
  bool const unbounded = lim.tophits > RANK_TOPHITS_MAX;
  int const tophits = static_cast<int>(std::min<int64_t>(lim.tophits, RANK_TOPHITS_MAX));
  int const nstrands = opts->strand_both ? 2 : 1;
  if (opts->self != 0 && (opts->query_labels == nullptr || opts->target_labels == nullptr)) {
    Error::set("vsg_search_batch: --self needs query_labels and target_labels"); return VSG_EINVAL;
  }
  if (opts->idprefix < 0 || opts->idsuffix < 0) { Error::set("vsg_search_batch: idprefix/idsuffix must not be negative"); return VSG_EINVAL; }
  bool const content_filters = opts->idprefix > 0 || opts->idsuffix > 0 || opts->selfid != 0;

  // Sub-batches run on a few host threads, each with its own child context (stream + scratch):
  // while one thread replays accept/reject decisions or builds task lists, the kernels of the
  // others keep the GPU busy.  Results land in disjoint slots, so no ordering is needed.
  int64_t BATCH = 4096;
  if (const char * e = std::getenv("VSG_SUBBATCH")) { BATCH = std::max<int64_t>(256, std::atoll(e)); }
  // With the unbounded lists the host holds every candidate of a sub-batch at once: its list entry, its hit slot and, in
  // the round that aligns it, its pair (about 200 bytes each).  Such sub-batches are therefore cut from the ranker's
  // count pass by candidate volume, both strands counted: at most SUBBATCH_CANDIDATES (about 0.8 GB of host memory each,
  // a few GB for the sub-batches of all host threads in flight) and at most BATCH queries; a query with more candidates
  // than that is a sub-batch of its own.
  constexpr int64_t SUBBATCH_CANDIDATES = int64_t(1) << 22;
  std::vector<int64_t> pieces;   // unbounded: sub-batch i is queries [pieces[i], pieces[i + 1])
  if (unbounded) {
    std::vector<int32_t> n, nrc;
    if (int const r = rank_counts(c, index_targets(ix, opts->mask_lower), queries, q0, nq, lim.minwordmatches, n); r != VSG_OK) { return r; }
    if (nstrands == 2) {
      SeqsetPtr rc_all;
      int r = seqset_revcomp(c, queries, q0, nq, rc_all);
      if (r == VSG_OK && opts->qmask_dust != 0) { r = vsg_seqset_dust(c, rc_all.get()); }
      if (r == VSG_OK) { r = rank_counts(c, index_targets(ix, opts->mask_lower), rc_all.get(), 0, nq, lim.minwordmatches, nrc); }
      if (r != VSG_OK) { return r; }
    }
    pieces.push_back(0);
    int64_t vol = 0;
    for (int64_t q = 0; q < nq; q++) {
      int64_t v = std::min<int64_t>(n[static_cast<size_t>(q)], lim.tophits);
      if (nstrands == 2) { v += std::min<int64_t>(nrc[static_cast<size_t>(q)], lim.tophits); }
      if (q > pieces.back() && (vol + v > SUBBATCH_CANDIDATES || q - pieces.back() >= BATCH)) { pieces.push_back(q); vol = 0; }
      vol += v;
    }
    pieces.push_back(nq);
  }
  int64_t const nbatches = unbounded ? static_cast<int64_t>(pieces.size()) - 1 : (nq + BATCH - 1) / BATCH;
  int nthreads = 8;
  if (const char * e = std::getenv("VSG_HOST_THREADS")) { nthreads = std::max(1, std::atoi(e)); }
  nthreads = static_cast<int>(std::min<int64_t>(nthreads, nbatches));
  int64_t tail_pairs = 4096;  // the tail starts when the round's pairs + all remaining candidates fit in this (0: never)
  if (const char * e = std::getenv("VSG_TAIL_PAIRS")) { tail_pairs = std::max<int64_t>(0, std::atoll(e)); }
  if (int const r = prepare_children(c, nthreads); r != VSG_OK) { return r; }

  vsg_ctx * const parent = c;
  auto const t_call0 = std::chrono::steady_clock::now();
  auto run_batch = [&](vsg_ctx * c, int64_t b0, int64_t bn_req, int64_t & total_pairs, int64_t & total_cells, int64_t & al_pairs, int64_t & al_cells) -> int {
  // host buffers live in the worker's context: a batch touches ~20 MB of them, and fresh pages per
  // batch (malloc -> mmap -> page faults) cost more than the bookkeeping itself
  if (!c->search_scratch) { c->search_scratch = std::make_shared<SearchScratch>(); }
  SearchScratch & sc = *static_cast<SearchScratch *>(c->search_scratch.get());
  auto & st = sc.st;
  Hit *& hits = sc.hits;  // one slot per candidate of the sub-batch, deliberately uninitialised (each is zeroed when popped)
  auto & pq = sc.pq; auto & pt = sc.pt;
  auto & pstate = sc.pstate;  // which state each pair belongs to
  auto & px = sc.px;          // which of the state's hits
  auto & plead = sc.plead;
  PairResults & a = sc.a;
  int64_t tb_redone = 0;
  VSG_CUDA_OK(cudaSetDevice(c->device));
  static const bool trace = std::getenv("VSG_TRACE") != nullptr;
  auto now = []() { return std::chrono::steady_clock::now(); };
  auto ms = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) {
    return std::chrono::duration<double, std::milli>(b - a).count();
  };
  double t_rank = 0, t_init = 0, t_gather = 0, t_align = 0, t_replay = 0, t_join = 0;
  auto tp0 = now();
  {

    int64_t const bn = std::min(bn_req, nq - b0);
    SeqsetPtr rc_set;
    if (nstrands == 2) {
      int r = seqset_revcomp(c, queries, q0 + b0, bn, rc_set);
      if (r != VSG_OK) { return r; }
      // each strand is masked on its own (search.cpp:437-449); dust() upper-cases first, so the case the
      // reverse complement inherited from the masked plus strand does not matter
      if (opts->qmask_dust != 0 && (r = vsg_seqset_dust(c, rc_set.get())) != VSG_OK) { return r; }
    }
    size_t const nst = static_cast<size_t>(bn) * nstrands;
    auto & cfirst = sc.cfirst;
    cfirst.assign(nst + 1, 0);
    sc.h_n.resize(nst);
    if (unbounded) {
      // lists back to back, each as long as the query's candidates (up to tophits)
      sc.h_seqno.clear(); sc.h_count.clear(); sc.h_flags.clear();
      for (int s = 0; s < nstrands; s++) {
        const vsg_seqset * qset = (s == 0) ? queries : rc_set.get();
        int64_t const qq0 = (s == 0) ? q0 + b0 : 0;
        int r = rank_lists(c, index_targets(ix, opts->mask_lower), qset, qq0, bn, lim.minwordmatches, lim.tophits, sc.lfirst, sc.lseq, sc.lcnt);
        if (r != VSG_OK) { return r; }
        int64_t const base = static_cast<int64_t>(sc.h_seqno.size());
        for (int64_t q = 0; q < bn; q++) {
          size_t const i = static_cast<size_t>(s) * bn + q;
          cfirst[i] = base + sc.lfirst[static_cast<size_t>(q)];
          sc.h_n[i] = static_cast<int32_t>(sc.lfirst[static_cast<size_t>(q) + 1] - sc.lfirst[static_cast<size_t>(q)]);
        }
        sc.h_seqno.insert(sc.h_seqno.end(), sc.lseq.begin(), sc.lseq.end());
        sc.h_count.insert(sc.h_count.end(), sc.lcnt.begin(), sc.lcnt.end());
        if (content_filters) {
          size_t const n = sc.lseq.size();
          sc.h_flags.resize(sc.h_seqno.size(), 0);
          if (n == 0) { continue; }
          size_t const fb = sizeof(int64_t) * (static_cast<size_t>(bn) + 1);
          if ((r = c->rank_tmp.reserve(fb + sizeof(uint32_t) * n + 16)) != VSG_OK || (r = c->pre_flags.reserve(n + 16)) != VSG_OK) { return r; }
          int64_t * const d_first = static_cast<int64_t *>(c->rank_tmp.p);
          uint32_t * const d_cand = reinterpret_cast<uint32_t *>(d_first + bn + 1);
          VSG_CUDA_OK(cudaMemcpyAsync(d_first, sc.lfirst.data(), fb, cudaMemcpyHostToDevice, c->stream));
          VSG_CUDA_OK(cudaMemcpyAsync(d_cand, sc.lseq.data(), sizeof(uint32_t) * n, cudaMemcpyHostToDevice, c->stream));
          prefilter_kernel<<<static_cast<unsigned>((static_cast<int64_t>(n) * 32 + 255) / 256), 256, 0, c->stream>>>(
              qset->d, qq0, static_cast<int>(bn), db->d, d_cand, nullptr, 0, d_first, opts->idprefix, opts->idsuffix, opts->selfid,
              static_cast<uint8_t *>(c->pre_flags.p));
          count_launch();
          VSG_CUDA_OK(cudaMemcpyAsync(sc.h_flags.data() + base, c->pre_flags.p, n, cudaMemcpyDeviceToHost, c->stream));
          VSG_CUDA_OK(cudaStreamSynchronize(c->stream));
        }
      }
    } else {
      size_t const cells = static_cast<size_t>(bn) * tophits;
      for (size_t i = 0; i < nst; i++) { cfirst[i] = static_cast<int64_t>(i) * tophits; }
      sc.h_seqno.resize(cells * nstrands); sc.h_count.resize(cells * nstrands);
      if (content_filters) { sc.h_flags.resize(cells * nstrands); }
      for (int s = 0; s < nstrands; s++) {
        const vsg_seqset * qset = (s == 0) ? queries : rc_set.get();
        int64_t const qq0 = (s == 0) ? q0 + b0 : 0;
        RankTop rt;
        int r = rank_enqueue(c, ix, qset, qq0, bn, lim.minwordmatches, tophits, opts->mask_lower, rt);
        if (r != VSG_OK) { return r; }
        if (content_filters) {
          if ((r = c->pre_flags.reserve(cells + 16)) != VSG_OK) { return r; }
          VSG_CUDA_OK(cudaMemsetAsync(c->pre_flags.p, 0, cells, c->stream));
          int64_t const nwarps = bn * tophits;
          prefilter_kernel<<<static_cast<unsigned>((nwarps * 32 + 255) / 256), 256, 0, c->stream>>>(
              qset->d, qq0, static_cast<int>(bn), db->d, rt.seqno, rt.n, tophits, nullptr, opts->idprefix, opts->idsuffix, opts->selfid,
              static_cast<uint8_t *>(c->pre_flags.p));
          count_launch();
          VSG_CUDA_OK(cudaMemcpyAsync(sc.h_flags.data() + cells * s, c->pre_flags.p, cells, cudaMemcpyDeviceToHost, c->stream));
        }
        if ((r = rank_download(c, rt, bn, tophits, sc.h_seqno.data() + cells * s, sc.h_count.data() + cells * s,
                               sc.h_n.data() + bn * s, "vsg_search_batch")) != VSG_OK) { return r; }
      }
    }

    t_rank += ms(tp0, now()); tp0 = now();
    // one state per (query, strand); a hit slot per candidate
    st.assign(nst, QState());
    {
      size_t need = 0;
      for (size_t i = 0; i < nst; i++) { st[i].hit_base = static_cast<int64_t>(need); need += static_cast<size_t>(sc.h_n[i]); }
      if (need > sc.hits_cap) {
        std::free(hits);
        hits = static_cast<Hit *>(std::malloc(sizeof(Hit) * need));
        sc.hits_cap = hits != nullptr ? need : 0;
        if (hits == nullptr) { Error::set("out of host memory"); return VSG_ENOMEM; }
      }
    }
    for (int s = 0; s < nstrands; s++) {
      for (int64_t q = 0; q < bn; q++) {
        QState & S = st[static_cast<size_t>(s) * bn + q];
        S.strand = s; S.ql = q;
        S.qlen = s == 0 ? queries->h_len[static_cast<size_t>(q0 + b0 + q)] : rc_set->h_len[static_cast<size_t>(q)];
        size_t const i = static_cast<size_t>(s) * bn + q;
        S.ncand = sc.h_n[i];
        S.cs = sc.h_seqno.data() + cfirst[i];
        S.cc = sc.h_count.data() + cfirst[i];
        S.cf = content_filters ? sc.h_flags.data() + cfirst[i] : nullptr;
      }
    }
    // search_onequery's candidate loop (searchcore.cpp:915-954) up to its next align_delayed; false when the
    // query's search has ended.  search_acceptable_unaligned (searchcore.cpp:541-609) pre-rejects candidates.  With the
    // unbounded ranker's lists, where a query can have thousands of candidates, an exhaustible list is one group.
    auto next_group = [&](QState & S) -> bool {
      bool const whole = unbounded && exhaustible(S.ncand, S.finalized, S.accepts, S.rejects, maxaccepts, maxrejects);
      while ((S.finalized + S.delayed < maxaccepts + maxrejects - 1) && (S.rejects < maxrejects) &&
             (S.accepts < maxaccepts) && (S.next < S.ncand)) {
        Hit & h = hits[static_cast<size_t>(S.hit_base) + S.hit_count];
        std::memset(&h, 0, sizeof(Hit));
        h.target = static_cast<int>(S.cs[S.next]); h.count = S.cc[S.next]; h.strand = S.strand;
        unsigned const content = S.cf != nullptr ? S.cf[S.next] : 0u;
        S.next++;
        int64_t const qsize = opts->query_sizes != nullptr ? opts->query_sizes[b0 + S.ql] : 1;
        int64_t const tsize = opts->target_sizes != nullptr ? opts->target_sizes[h.target] : 1;
        bool const same_label = opts->self != 0 && opts->query_labels[b0 + S.ql] == opts->target_labels[h.target];
        if (acceptable_unaligned(*opts, S.qlen, db->h_len[static_cast<size_t>(h.target)], qsize, tsize, same_label, content)) {
          S.delayed++;
        } else {
          h.rejected = true;
        }
        S.hit_count++;
        if (S.delayed == MAXDELAYED && !whole) { return true; }
      }
      if (S.delayed == 0) { S.done = true; return false; }
      return true;
    };

    t_init += ms(tp0, now());
    bool any = true;
    bool tail_mode = false;
    bool gated_round = false;
    while (any) {
      gated_round = false;
      tp0 = now();
      any = false;
      pq.clear(); pt.clear(); pstate.clear(); px.clear(); plead.clear();
      // gather: run each active query's candidate loop up to its next align_delayed (searchcore.cpp:915-954)
      if (lazy) {
        // same decisions, alignments on demand: open the group the reference would hand to search16,
        // but align only the hit the replay is about to examine
        for (size_t si = 0; si < st.size(); si++) {
          QState & S = st[si];
          if (S.done) { continue; }
          for (;;) {
            if (S.gpos < 0) {
              if (!next_group(S)) { break; }
              S.gpos = S.finalized;
              for (int x = S.finalized; x < S.hit_count; x++) {   // what the reference's search16 call covers
                Hit const & h = hits[static_cast<size_t>(S.hit_base) + x];
                if (!h.rejected) { total_pairs++; total_cells += static_cast<int64_t>(S.qlen) * db->h_len[static_cast<size_t>(h.target)]; }
              }
            }
            bool need = false;
            while (S.gpos < S.hit_count && S.rejects < maxrejects && S.accepts < maxaccepts) {
              Hit const & h = hits[static_cast<size_t>(S.hit_base) + S.gpos];
              if (h.rejected) { S.rejects++; S.gpos++; continue; }
              need = true;
              break;
            }
            if (need) {
              // the group's first candidate alone (it is accepted most of the time); if the replay gets
              // past it, the rest of the group in one go — at most two device round trips per group
              int const xend = (S.gpos == S.finalized) ? S.gpos + 1 : S.hit_count;
              S.greq = 0;
              for (int x = S.gpos; x < xend; x++) {
                Hit const & h = hits[static_cast<size_t>(S.hit_base) + x];
                if (h.rejected) { continue; }
                pq.push_back(static_cast<uint32_t>(S.strand == 0 ? q0 + b0 + S.ql : S.ql));
                pt.push_back(static_cast<uint32_t>(h.target));
                pstate.push_back(static_cast<int>(si));
                px.push_back(x);
                S.greq++;
              }
              S.gend = xend;
              S.waiting = true;
              any = true;
              break;
            }
            // group exhausted or a limit reached: align_delayed ends, the candidate loop resumes
            S.finalized = S.hit_count; S.delayed = 0; S.gpos = -1;
          }
        }
      } else
      for (size_t si = 0; si < st.size(); si++) {
        QState & S = st[si];
        if (S.done || !next_group(S)) { continue; }
        // align_delayed's search16 call: every not-yet-finalized, not pre-rejected hit
        // traceback on demand (align_ckpt.cuh): if accepting the group's first candidate ends this query's search,
        // the others are walked back only when that candidate turns out not to be accepted
        bool const gate_group = tb_gate && (S.accepts + 1 >= maxaccepts);
        int32_t leader = -1;
        for (int x = S.finalized; x < S.hit_count; x++) {
          Hit const & h = hits[static_cast<size_t>(S.hit_base) + x];
          if (!h.rejected) {
            plead.push_back(gate_group ? leader : -1);
            if (leader < 0) { leader = static_cast<int32_t>(pq.size()); }
            pq.push_back(static_cast<uint32_t>(S.strand == 0 ? q0 + b0 + S.ql : S.ql));
            pt.push_back(static_cast<uint32_t>(h.target));
            pstate.push_back(static_cast<int>(si));
            px.push_back(x);
          }
        }
        S.waiting = true;
        any = true;
      }
      if (!any) { break; }
      size_t const np = pq.size();
      t_gather += ms(tp0, now()); tp0 = now();
      a.resize(np);
      // pairs of the plus strand index `queries`, those of the minus strand index rc_set: two calls
      // (states are ordered plus first, minus second, so pairs are too)
      auto device_align = [&](size_t n, const uint32_t * Q, const uint32_t * T, const int * state_of, PairResults & out,
                              const int32_t * lead) -> int {
        size_t split = n;
        if (nstrands == 2) {
          split = 0;
          while (split < n && static_cast<int64_t>(state_of[split]) < bn) { split++; }
        }
        for (int part = 0; part < 2; part++) {
          size_t const lo = part == 0 ? 0 : split, hi = part == 0 ? split : n;
          if (hi <= lo) { continue; }
          const vsg_seqset * qset = part == 0 ? queries : rc_set.get();
          const int32_t * lead_part = nullptr;
          if (lead != nullptr) {
            // leaders as indices into this part's own pair list (a group never straddles the strands)
            sc.lead_tmp.assign(lead + lo, lead + hi);
            if (lo > 0) { for (auto & v : sc.lead_tmp) { if (v >= 0) { v -= static_cast<int32_t>(lo); } } }
            lead_part = sc.lead_tmp.data();
          }
          int const r = align_into(c, qset, db, hi - lo, Q + lo, T + lo, out, lo, lead_part,
                                   tb_force == 1 ? -1.0 : (tb_force == 2 ? 1e9 : 100.0 * opt_id + 1e-7), opts->iddef);
          if (r != VSG_OK) { return r; }
        }
        return VSG_OK;
      };
      bool const from_cache = tail_mode;
      // what the tail shortcut would add to this round: every candidate the active queries have left
      auto count_extras = [&]() -> size_t {
        size_t extras = 0;
        for (size_t k = 0; k < np; k++) {
          if (k + 1 == np || pstate[k + 1] != pstate[k]) {
            QState const & S = st[static_cast<size_t>(pstate[k])];
            extras += static_cast<size_t>(std::max(0, S.ncand - (lazy ? S.gend : S.hit_count)));
          }
        }
        return extras;
      };
      if (tail_mode) {
        // every query still active had all its remaining candidates aligned when the tail began
        for (size_t k = 0; k < np; k++) {
          QState const & S = st[static_cast<size_t>(pstate[k])];
          a.copy(k, sc.t, static_cast<size_t>(S.cache_off + px[k] - S.cache_first));
        }
      } else if (tail_pairs > 0 && np <= static_cast<size_t>(tail_pairs) && np + count_extras() <= static_cast<size_t>(tail_pairs)) {
        // TAIL: few queries are left and each would need up to five more rounds of eight candidates
        // (searchcore.cpp:915-954), every round a device round trip with almost nothing in it.  Align
        // all their remaining candidates now; later rounds replay from these results.  The decisions
        // (and work[0..1], the reference's own pairs) are unchanged; work[2..3] include the extras.
        auto & lq = sc.lq; auto & lt = sc.lt; auto & lstate = sc.lstate; auto & ldest = sc.ldest;
        lq.clear(); lt.clear(); lstate.clear(); ldest.clear();
        int64_t ncache = 0;
        for (size_t k = 0; k < np; k++) {
          lq.push_back(pq[k]); lt.push_back(pt[k]); lstate.push_back(pstate[k]); ldest.push_back(static_cast<int64_t>(k));
          if (k + 1 == np || pstate[k + 1] != pstate[k]) {
            QState & S = st[static_cast<size_t>(pstate[k])];
            int const first_extra = lazy ? S.gend : S.hit_count;
            S.cache_first = first_extra; S.cache_off = static_cast<int>(ncache);
            for (int idx = first_extra; idx < S.ncand; idx++) {
              lq.push_back(pq[k]); lt.push_back(S.cs[idx]); lstate.push_back(pstate[k]); ldest.push_back(-(ncache + 1));
              al_cells += static_cast<int64_t>(S.qlen) * db->h_len[static_cast<size_t>(S.cs[idx])];
              ncache++;
            }
          }
        }
        size_t const nl = lq.size();
        sc.l.resize(nl);
        sc.t.resize(static_cast<size_t>(ncache));
        int const r = device_align(nl, lq.data(), lt.data(), lstate.data(), sc.l, nullptr);
        if (r != VSG_OK) { return r; }
        for (size_t k = 0; k < nl; k++) {
          if (ldest[k] >= 0) { a.copy(static_cast<size_t>(ldest[k]), sc.l, k); }
          else { sc.t.copy(static_cast<size_t>(-ldest[k] - 1), sc.l, k); }
        }
        al_pairs += static_cast<int64_t>(nl);
        tail_mode = true;
      } else {
        gated_round = tb_gate && !lazy && plead.size() == np;
        int const r = device_align(np, pq.data(), pt.data(), pstate.data(), a, gated_round ? plead.data() : nullptr);
        if (r != VSG_OK) { return r; }
        al_pairs += static_cast<int64_t>(np);
      }
      if (!lazy) { total_pairs += static_cast<int64_t>(np); }
      t_align += ms(tp0, now()); tp0 = now();
      // replay: the second half of align_delayed (searchcore.cpp:780-880)
      size_t pi = 0;
      for (size_t si = 0; si < st.size(); si++) {
        QState & S = st[si];
        if (!S.waiting) { continue; }
        S.waiting = false;
        size_t i = pi;
        int const xlo = lazy ? S.gpos : S.finalized, xhi = lazy ? S.gend : S.hit_count;
        for (int x = xlo; x < xhi; x++) {
          Hit & h = hits[static_cast<size_t>(S.hit_base) + x];
          if (!h.rejected) {
            int64_t const cl = static_cast<int64_t>(S.qlen) * db->h_len[static_cast<size_t>(h.target)];
            if (!from_cache) { al_cells += cl; }
            if (!lazy) { total_cells += cl; }
          }
        }
        for (int x = xlo; x < xhi; x++) {
          if (S.rejects < maxrejects && S.accepts < maxaccepts) {
            Hit & h = hits[static_cast<size_t>(S.hit_base) + x];
            if (h.rejected) { S.rejects++; continue; }
            if (gated_round && plead[i] >= 0 && a.walk_skipped(i)) {
              // its walk was skipped because the device took the group's leader for accepted, yet the replay is here:
              // the two verdicts differ (a borderline identity); align this pair now
              int const r = align_into(c, S.strand == 0 ? queries : rc_set.get(), db, 1, &pq[i], &pt[i], a, i);
              if (r != VSG_OK) { return r; }
              tb_redone++;
            }
            int const dlen = db->h_len[static_cast<size_t>(h.target)];
            int const r = fill_hit(h, a, i, S.qlen, dlen, opts->iddef, *parent, q0 + b0 + S.ql, S.strand, "vsg_search_batch");
            if (r != VSG_OK) { return r; }
            int64_t const qsz = opts->query_sizes != nullptr ? opts->query_sizes[b0 + S.ql] : 1;
            int64_t const tsz = opts->target_sizes != nullptr ? opts->target_sizes[h.target] : 1;
            if (acceptable_aligned(h, opt_id, opt_weak_id, *opts, S.qlen, dlen, qsz, tsz)) { S.accepts++; } else { S.rejects++; }
            ++i;
          }
        }
        // the pairs of this state, examined or not, are consumed
        size_t mine = 0;
        while (pi + mine < np && static_cast<size_t>(pstate[pi + mine]) == si) { mine++; }
        pi += mine;
        if (lazy) { S.gpos = S.gend; }
        else { S.finalized = S.hit_count; S.delayed = 0; }
      }
      t_replay += ms(tp0, now());
    }

    tp0 = now();
    // search_joinhits + result records (search.cpp:466-488)
    for (int64_t q = 0; q < bn; q++) {
      std::vector<Hit> & joined = sc.joined;
      joined.clear();
      for (int s = 0; s < nstrands; s++) {
        QState const & S = st[static_cast<size_t>(s) * bn + q];
        for (int x = 0; x < S.hit_count; x++) {
          Hit const & h = hits[static_cast<size_t>(S.hit_base) + x];
          if (h.accepted || h.weak) { joined.push_back(h); }
        }
      }
      std::stable_sort(joined.begin(), joined.end(), hit_less);
      sink(b0 + q, joined);
    }
    t_join += ms(tp0, now());
  }
  c->prof_tb_redone += tb_redone;
  if (trace) {
    std::fprintf(stderr, "[vsg trace] batch@%lld: rank %.1f init %.1f gather %.1f align %.1f replay %.1f join %.1f ms; done at %.1f ms; %lld skipped walks redone\n",
                 static_cast<long long>(b0), t_rank, t_init, t_gather, t_align, t_replay, t_join, ms(t_call0, now()), static_cast<long long>(tb_redone));
  }
  return VSG_OK;
  };

  std::atomic<int64_t> next{0};
  std::vector<int64_t> tp(static_cast<size_t>(nthreads), 0), tc(static_cast<size_t>(nthreads), 0), ap(static_cast<size_t>(nthreads), 0), ac(static_cast<size_t>(nthreads), 0);
  int const rc = run_parallel(nthreads, [&](int t) -> int {
    vsg_ctx * wc = c->children[static_cast<size_t>(t)];
    if (unbounded) {   // the sub-batches cut above, in order
      for (;;) {
        int64_t const i = next.fetch_add(1);
        if (i >= nbatches) { return VSG_OK; }
        int64_t const b0 = pieces[static_cast<size_t>(i)], bn = pieces[static_cast<size_t>(i) + 1] - b0;
        int const r = run_batch(wc, b0, bn, tp[static_cast<size_t>(t)], tc[static_cast<size_t>(t)], ap[static_cast<size_t>(t)], ac[static_cast<size_t>(t)]);
        if (r != VSG_OK) { next.store(nbatches); return r; }
      }
    }
    // Sub-batches are cut from a shared cursor.  A thread's FIRST one is shortened to (t+1)/nthreads of
    // the regular size: identical sub-batches started together run in lockstep (all threads rank, then
    // all gather on the host, then all align ...) and the device idles through every host phase;
    // staggered, some thread always has a kernel in flight.
    bool first = true;
    for (;;) {
      int64_t want = BATCH;
      if (first && nthreads > 1) { want = std::max<int64_t>(256, BATCH * (t + 1) / nthreads); }
      first = false;
      int64_t const b0 = next.fetch_add(want);
      if (b0 >= nq) { return VSG_OK; }
      int const r = run_batch(wc, b0, want, tp[static_cast<size_t>(t)], tc[static_cast<size_t>(t)], ap[static_cast<size_t>(t)], ac[static_cast<size_t>(t)]);
      if (r != VSG_OK) { next.store(nq); return r; }
    }
  });
  absorb_children(c, nthreads);
  if (rc != VSG_OK) { return rc; }
  for (int t = 0; t < nthreads; t++) {
    total_pairs += tp[static_cast<size_t>(t)]; total_cells += tc[static_cast<size_t>(t)];
    aligned_pairs += ap[static_cast<size_t>(t)]; aligned_cells += ac[static_cast<size_t>(t)];
  }
  if (work != nullptr) { work[0] = total_pairs; work[1] = total_cells; work[2] = aligned_pairs; work[3] = aligned_cells; }
  return VSG_OK;
}

}  // namespace

extern "C" int vsg_search_batch(vsg_ctx * c, const vsg_index * ix, const vsg_seqset * db,
                                const vsg_seqset * queries, int64_t q0, int64_t nq,
                                const vsg_search_opts * opts, vsg_search_result * results, int max_results,
                                int32_t * counts, int64_t * work)
{
  if (c == nullptr || ix == nullptr || db == nullptr || queries == nullptr || opts == nullptr ||
      results == nullptr || counts == nullptr || max_results < 1) {
    Error::set("vsg_search_batch: bad argument");
    return VSG_EINVAL;
  }
  for (int64_t q = 0; q < nq; q++) { counts[q] = 0; }
  return search_core(c, ix, db, queries, q0, nq, opts, [&](int64_t q, const std::vector<Hit> & joined) {
    int const n = static_cast<int>(std::min<size_t>(joined.size(), static_cast<size_t>(max_results)));
    int const qlen = queries->h_len[static_cast<size_t>(q0 + q)];
    for (int j = 0; j < n; j++) {
      Hit const & h = joined[static_cast<size_t>(j)];
      results[static_cast<size_t>(q) * max_results + j] = result_of(h, qlen, db->h_len[static_cast<size_t>(h.target)]);
    }
    counts[q] = n;
  }, work);
}

namespace vsg {

int search_hits_host(vsg_ctx * c, const vsg_index * ix, const vsg_seqset * db, const vsg_seqset * queries, int64_t q0,
                     int64_t nq, const vsg_search_opts * opts, int64_t maxhits, std::vector<vsg_search_result> & rows,
                     std::vector<int64_t> & first, int64_t * work)
{
  if (c == nullptr || ix == nullptr || db == nullptr || queries == nullptr || opts == nullptr || nq < 0 || maxhits < 0) {
    Error::set("vsg_search_hits: bad argument");
    return VSG_EINVAL;
  }
  std::vector<std::vector<vsg_search_result>> perq(static_cast<size_t>(nq));
  int const rc = search_core(c, ix, db, queries, q0, nq, opts, [&](int64_t q, const std::vector<Hit> & joined) {
    size_t const n = maxhits > 0 ? std::min<size_t>(joined.size(), static_cast<size_t>(maxhits)) : joined.size();
    int const qlen = queries->h_len[static_cast<size_t>(q0 + q)];
    auto & out = perq[static_cast<size_t>(q)];
    out.reserve(n);
    for (size_t j = 0; j < n; j++) { out.push_back(result_of(joined[j], qlen, db->h_len[static_cast<size_t>(joined[j].target)])); }
  }, work);
  if (rc != VSG_OK) { return rc; }
  first.assign(static_cast<size_t>(nq) + 1, 0);
  for (int64_t q = 0; q < nq; q++) { first[static_cast<size_t>(q) + 1] = first[static_cast<size_t>(q)] + static_cast<int64_t>(perq[static_cast<size_t>(q)].size()); }
  rows.clear();
  rows.reserve(static_cast<size_t>(first[static_cast<size_t>(nq)]));
  for (auto & v : perq) { rows.insert(rows.end(), v.begin(), v.end()); }
  return VSG_OK;
}

int hits_out(const std::vector<vsg_search_result> & rows, const std::vector<int64_t> & first, const char * caller,
             vsg_search_result * hits, int64_t cap, int64_t * first_out, int64_t * nhits)
{
  std::memcpy(first_out, first.data(), sizeof(int64_t) * first.size());
  *nhits = static_cast<int64_t>(rows.size());
  if (*nhits > cap) { Error::set(std::string(caller) + ": hit buffer too small"); return VSG_ECAP; }
  if (!rows.empty()) { std::memcpy(hits, rows.data(), sizeof(vsg_search_result) * rows.size()); }
  return VSG_OK;
}

}  // namespace vsg

extern "C" int vsg_search_hits(vsg_ctx * c, const vsg_index * ix, const vsg_seqset * db, const vsg_seqset * queries, int64_t q0,
                               int64_t nq, const vsg_search_opts * opts, int64_t maxhits, vsg_search_result * hits, int64_t cap,
                               int64_t * first, int64_t * nhits, int64_t * work)
{
  if (first == nullptr || nhits == nullptr || cap < 0 || (cap > 0 && hits == nullptr)) { Error::set("vsg_search_hits: bad argument"); return VSG_EINVAL; }
  *nhits = 0;
  std::vector<vsg_search_result> rows;
  std::vector<int64_t> f;
  int const rc = search_hits_host(c, ix, db, queries, q0, nq, opts, maxhits, rows, f, work);
  if (rc != VSG_OK) { return rc; }
  return hits_out(rows, f, "vsg_search_hits", hits, cap, first, nhits);
}


// ---- all-against-all -----------------------------------------------------------------------------
extern "C" int vsg_allpairs_partition(const int32_t * len, int64_t n, int nparts, int64_t * bounds)
{
  if (n < 0 || nparts < 1 || bounds == nullptr || (n > 0 && len == nullptr)) { Error::set("vsg_allpairs_partition: bad argument"); return VSG_EINVAL; }
  // cells(i) = len[i] * sum_{j>i} len[j]
  std::vector<double> row(static_cast<size_t>(n));
  double suffix = 0.0, total = 0.0;
  for (int64_t i = n - 1; i >= 0; i--) { row[static_cast<size_t>(i)] = static_cast<double>(len[i]) * suffix; suffix += len[i]; total += row[static_cast<size_t>(i)]; }
  bounds[0] = 0;
  double acc = 0.0;
  int p = 1;
  for (int64_t i = 0; i < n && p < nparts; i++) {
    acc += row[static_cast<size_t>(i)];
    while (p < nparts && acc >= total * p / nparts) { bounds[p++] = i + 1; }
  }
  while (p <= nparts) { bounds[p++] = n; }
  return VSG_OK;
}

extern "C" int vsg_allpairs(vsg_ctx * c, const vsg_seqset * set, int64_t row0, int64_t nrows,
                            const vsg_search_opts * opts, vsg_pair_hit * hits, int64_t cap, int64_t * nhits,
                            int64_t * work)
{
  if (c == nullptr || set == nullptr || opts == nullptr || nhits == nullptr || (cap > 0 && hits == nullptr)) {
    Error::set("vsg_allpairs: bad argument");
    return VSG_EINVAL;
  }
  int64_t const n = set->d.n;
  if (row0 < 0 || nrows < 0 || row0 + nrows > n) { Error::set("vsg_allpairs: row range out of bounds"); return VSG_EINVAL; }
  if (opts->iddef < 0 || opts->iddef > 4) { Error::set("vsg_allpairs: iddef must be 0..4"); return VSG_EINVAL; }
  double const opt_id = opts->id, opt_weak_id = weak_id_of(*opts);
  *nhits = 0;

  // blocks of consecutive rows with about PAIRS_PER_BLOCK pairs each, handed to host threads that own
  // a child context each; every block writes its hits to a private vector, concatenated in row order
  int64_t const PAIRS_PER_BLOCK = 1 << 20;
  std::vector<int64_t> block_first;
  {
    int64_t acc = 0;
    block_first.push_back(row0);
    for (int64_t i = row0; i < row0 + nrows; i++) {
      acc += n - i - 1;
      if (acc >= PAIRS_PER_BLOCK && i + 1 < row0 + nrows) { block_first.push_back(i + 1); acc = 0; }
    }
    block_first.push_back(row0 + nrows);
  }
  int64_t const nblocks = static_cast<int64_t>(block_first.size()) - 1;
  int nthreads = 8;
  if (const char * e = std::getenv("VSG_HOST_THREADS")) { nthreads = std::max(1, std::atoi(e)); }
  nthreads = static_cast<int>(std::max<int64_t>(1, std::min<int64_t>(nthreads, nblocks)));
  if (int const r = prepare_children(c, nthreads); r != VSG_OK) { return r; }
  std::vector<std::vector<vsg_pair_hit>> out(static_cast<size_t>(nblocks));
  std::vector<int64_t> bpairs(static_cast<size_t>(nblocks), 0), bcells(static_cast<size_t>(nblocks), 0);

  auto run_block = [&](vsg_ctx * wc, int64_t bi) -> int {
    int64_t const r0 = block_first[static_cast<size_t>(bi)], r1 = block_first[static_cast<size_t>(bi) + 1];
    std::vector<uint32_t> pq, pt;
    int64_t cells = 0;
    {
      int64_t cap_pairs = 0;
      for (int64_t i = r0; i < r1; i++) { cap_pairs += n - i - 1; }
      pq.reserve(static_cast<size_t>(cap_pairs)); pt.reserve(static_cast<size_t>(cap_pairs));
    }
    for (int64_t i = r0; i < r1; i++) {
      int const ql = set->h_len[static_cast<size_t>(i)];
      int64_t tl = 0;
      for (int64_t j = i + 1; j < n; j++) {
        int const dl = set->h_len[static_cast<size_t>(j)];
        if (!acceptable_unaligned(*opts, ql, dl, 1, 1, false, 0u)) { continue; }  // allpairs_global.cpp:407-414 (defaults for the rest)
        pq.push_back(static_cast<uint32_t>(i)); pt.push_back(static_cast<uint32_t>(j)); tl += dl;
      }
      cells += static_cast<int64_t>(ql) * tl;
    }
    int64_t const np = static_cast<int64_t>(pq.size());
    if (np == 0) { return VSG_OK; }
    PairResults res;
    res.resize(static_cast<size_t>(np));
    int const r = align_into(wc, set, set, static_cast<size_t>(np), pq.data(), pt.data(), res, 0);
    if (r != VSG_OK) { return r; }
    std::vector<vsg_pair_hit> & o = out[static_cast<size_t>(bi)];
    int64_t k = 0;
    while (k < np) {
      int64_t const i = pq[static_cast<size_t>(k)];
      size_t const first = o.size();
      int const qlen = set->h_len[static_cast<size_t>(i)];
      for (; k < np && pq[static_cast<size_t>(k)] == i; k++) {
        Hit h;
        std::memset(&h, 0, sizeof h);
        h.target = static_cast<int>(pt[static_cast<size_t>(k)]);
        int const dlen = set->h_len[static_cast<size_t>(h.target)];
        int const rh = fill_hit(h, res, static_cast<size_t>(k), qlen, dlen, opts->iddef, *c, i, 0, "vsg_allpairs");
        if (rh != VSG_OK) { return rh; }
        if (acceptable_aligned(h, opt_id, opt_weak_id, *opts, qlen, dlen)) {
          vsg_pair_hit ph;
          ph.query = static_cast<int32_t>(i); ph.target = h.target; ph.matches = h.matches; ph.mismatches = h.mismatches;
          ph.gaps = h.nwgaps; ph.alignment_length = h.nwalignmentlength; ph.nwscore = h.nwscore;
          ph.internal_alignment_length = h.internal_alignmentlength; ph.id = h.id;
          o.push_back(ph);
        }
      }
      std::sort(o.begin() + static_cast<std::ptrdiff_t>(first), o.end(), [](const vsg_pair_hit & a, const vsg_pair_hit & b) {
        if (a.id != b.id) { return a.id > b.id; }
        return a.target < b.target;
      });
    }
    bpairs[static_cast<size_t>(bi)] = np; bcells[static_cast<size_t>(bi)] = cells;
    return VSG_OK;
  };

  std::atomic<int64_t> next{0};
  int const rc = run_parallel(nthreads, [&](int t) -> int {
    vsg_ctx * wc = c->children[static_cast<size_t>(t)];
    cudaSetDevice(wc->device);
    for (;;) {
      int64_t const bi = next.fetch_add(1);
      if (bi >= nblocks) { return VSG_OK; }
      int const r = run_block(wc, bi);
      if (r != VSG_OK) { next.store(nblocks); return r; }
    }
  });
  absorb_children(c, nthreads);
  if (rc != VSG_OK) { return rc; }
  int64_t total = 0, tp = 0, tc = 0;
  for (int64_t bi = 0; bi < nblocks; bi++) { total += static_cast<int64_t>(out[static_cast<size_t>(bi)].size()); tp += bpairs[static_cast<size_t>(bi)]; tc += bcells[static_cast<size_t>(bi)]; }
  *nhits = total;
  if (work != nullptr) { work[0] = tp; work[1] = tc; }
  if (total > cap) { Error::set("vsg_allpairs: hit buffer too small"); return VSG_ECAP; }
  int64_t pos = 0;
  for (int64_t bi = 0; bi < nblocks; bi++) {
    auto const & o = out[static_cast<size_t>(bi)];
    if (!o.empty()) { std::memcpy(hits + pos, o.data(), sizeof(vsg_pair_hit) * o.size()); pos += static_cast<int64_t>(o.size()); }
  }
  return VSG_OK;
}
