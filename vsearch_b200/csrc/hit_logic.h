// hit_logic.h — the host-side accept/reject arithmetic shared by the search, all-pairs and cluster drivers
// (search.cu, cluster.cu): the option clamps, the per-pair aligner results, struct hit's fields, align_trim,
// search_acceptable_unaligned / search_acceptable_aligned and the hit orders of the reference
// (core/searchcore.cpp:133-179, 343-464, 541-737).
#pragma once

#include "vsg_internal.h"

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdint>

namespace vsg {

constexpr int MAXDELAYED = 8;  // searchcore.hpp:71
// searchcore.hpp:75-76
constexpr int minwordmatches_defaults[16] = {-1, -1, -1, 18, 17, 16, 15, 14, 12, 11, 10, 9, 8, 7, 5, 3};

// --weak_id is never above --id (vsearch_apply_defaults_fixups, vsearch.cc:186-276)
inline double weak_id_of(const vsg_search_opts & o) { return (o.id >= 0.0 && o.weak_id > o.id) ? o.id : o.weak_id; }

struct SearchLimits {
  int64_t maxaccepts, maxrejects, tophits;
  int minwordmatches;
  double opt_id, opt_weak_id;
};

// The option fix-ups of vsearch_apply_defaults_fixups (vsearch.cc:186-276) and the clamps against the number of
// targets of search_prep / search_session_init (commands/usearch_global.cpp:598-614) and cluster()
// (core/cluster.cpp:1213-1232).  o.wordlength must index minwordmatches_defaults.
inline int search_limits(const vsg_search_opts & o, int64_t seqcount, const char * caller, SearchLimits & l)
{
  l.maxaccepts = o.maxaccepts; l.maxrejects = o.maxrejects < 0 ? 32 : o.maxrejects;
  if (l.maxaccepts < 0) { Error::set(std::string(caller) + ": maxaccepts must not be negative"); return VSG_EINVAL; }
  if (l.maxaccepts > seqcount || l.maxaccepts == 0) { l.maxaccepts = seqcount; }
  if (l.maxrejects > seqcount || l.maxrejects == 0) { l.maxrejects = seqcount; }
  l.tophits = std::min<int64_t>(l.maxaccepts + l.maxrejects + MAXDELAYED, seqcount);
  l.minwordmatches = o.minwordmatches < 0 ? minwordmatches_defaults[o.wordlength] : o.minwordmatches;
  l.opt_id = o.id;
  l.opt_weak_id = weak_id_of(o);
  return VSG_OK;
}

// True when search_onequery's candidate loop (searchcore.cpp:915-954) will examine every candidate a query strand has
// left: after `finalized` of its ncand candidates, neither limit nor the loop's guard can be reached before the list
// ends, because each hit examined adds one accept or one reject.  Then none of that work is speculative, and the whole
// remaining list can be one group, aligned in one device call instead of eight candidates per round; the pairs aligned
// and the decisions are those of the groups of eight.  The search and cluster drivers apply it to the unbounded
// ranker's lists, where a query can have thousands of candidates.
inline bool exhaustible(int64_t ncand, int64_t finalized, int64_t accepts, int64_t rejects, int64_t maxaccepts, int64_t maxrejects)
{
  int64_t const left = ncand - finalized;
  return left > MAXDELAYED && accepts + left <= maxaccepts && rejects + left <= maxrejects && ncand <= maxaccepts + maxrejects - 1;
}

// The statistics an aligner call returns, one entry per pair: score, aligned, matches, mismatches, gaps, and four
// trims (vsg_align_pairs).
struct PairResults {
  std::vector<int16_t> score;
  std::vector<uint16_t> aligned, matches, mismatches, gaps;
  std::vector<int32_t> trims;   // 4 per pair
  void resize(size_t n)
  {
    score.resize(n); aligned.resize(n); matches.resize(n); mismatches.resize(n); gaps.resize(n); trims.resize(4 * n);
  }
  void copy(size_t k, const PairResults & from, size_t j)
  {
    score[k] = from.score[j]; aligned[k] = from.aligned[j]; matches[k] = from.matches[j];
    mismatches[k] = from.mismatches[j]; gaps[k] = from.gaps[j];
    for (int z = 0; z < 4; z++) { trims[4 * k + z] = from.trims[4 * j + z]; }
  }
  // traceback on demand skipped this pair's walk (align_pairs_gated)
  bool walk_skipped(size_t k) const { return aligned[k] == 0xffffu && matches[k] == 0xffffu && mismatches[k] == 0xffffu; }
};

// n pairs aligned into entries [at, at + n) of `out`; leader_of / threshold / iddef as in align_pairs_gated
inline int align_into(vsg_ctx * c, const vsg_seqset * queries, const vsg_seqset * targets, size_t n, const uint32_t * qidx,
                      const uint32_t * tidx, PairResults & out, size_t at, const int32_t * leader_of = nullptr,
                      double threshold = 0.0, int iddef = 2)
{
  return align_pairs_gated(c, queries, targets, static_cast<int64_t>(n), qidx, tidx, out.score.data() + at,
                           out.aligned.data() + at, out.matches.data() + at, out.mismatches.data() + at, out.gaps.data() + at,
                           out.trims.data() + 4 * at, nullptr, 0, nullptr, leader_of, threshold, iddef);
}

struct Hit {  // the fields of struct hit (searchcore.hpp:78-126) this path needs; POD, zeroed on use
  int target, strand;
  unsigned count;
  bool accepted, rejected, aligned, weak;
  bool forbidden_gap;  // fallback callback's alignment_uses_forbidden_gap verdict (searchcore.cpp:612-660)
  int nwscore, nwdiff, nwgaps, nwindels, nwalignmentlength;
  int matches, mismatches;
  int internal_alignmentlength, internal_gaps, internal_indels;
  int trim_q_left, trim_q_right, trim_t_left, trim_t_right;
  double id, id0, id1, id2, id3, id4;
  int shortest, longest;
};

// align_trim's arithmetic (searchcore.cpp:409-463) from the first/last CIGAR run
inline void finish_hit(Hit & h, const int32_t * trims, int iddef)
{
  h.trim_q_left = trims[0]; h.trim_t_left = trims[1]; h.trim_q_right = trims[2]; h.trim_t_right = trims[3];
  if (h.trim_q_left >= h.nwalignmentlength) { h.trim_q_right = 0; }
  if (h.trim_t_left >= h.nwalignmentlength) { h.trim_t_right = 0; }
  int const tr = h.trim_q_left + h.trim_t_left + h.trim_q_right + h.trim_t_right;
  h.internal_alignmentlength = h.nwalignmentlength - tr;
  h.internal_indels = h.nwindels - tr;
  h.internal_gaps = h.nwgaps - ((h.trim_q_left + h.trim_t_left) > 0 ? 1 : 0) - ((h.trim_q_right + h.trim_t_right) > 0 ? 1 : 0);
  h.id0 = h.shortest > 0 ? 100.0 * h.matches / h.shortest : 0.0;
  h.id1 = h.nwalignmentlength > 0 ? 100.0 * h.matches / h.nwalignmentlength : 0.0;
  h.id2 = h.internal_alignmentlength > 0 ? 100.0 * h.matches / h.internal_alignmentlength : 0.0;
  h.id3 = std::max(0.0, 100.0 * (1.0 - (1.0 * (h.mismatches + h.nwgaps) / h.longest)));
  h.id4 = h.nwalignmentlength > 0 ? 100.0 * h.matches / h.nwalignmentlength : 0.0;
  switch (iddef) {
    case 0: h.id = h.id0; break; case 1: h.id = h.id1; break; case 2: h.id = h.id2; break;
    case 3: h.id = h.id3; break; default: h.id = h.id4; break;
  }
}

// struct hit from entry k of `r`, the statistics search16 returned for (query, h.target) (searchcore.cpp:842-857,
// cluster.cpp:786-809).  A pair the 16-bit aligner deferred is resolved by fb's vsg_ctx_set_fallback callback, the
// host side of the reference's LinearMemoryAligner path (searchcore.cpp:806-832); without one the call fails as `caller`.
inline int fill_hit(Hit & h, const PairResults & r, size_t k, int qlen, int dlen, int iddef, const vsg_ctx & fb_ctx,
                    int64_t query, int strand, const char * caller)
{
  int64_t fb[10] = {r.score[k], r.aligned[k], r.matches[k], r.mismatches[k], r.gaps[k],
                    r.trims[4 * k], r.trims[4 * k + 1], r.trims[4 * k + 2], r.trims[4 * k + 3], 0};
  if (r.score[k] == VSG_SCORE_SENTINEL) {
    std::fill(fb, fb + 10, 0);
    if (fb_ctx.fallback == nullptr || fb_ctx.fallback(fb_ctx.fallback_user, query, strand, h.target, fb) != 0) {
      Error::set(std::string(caller) + ": a pair was deferred to the linear-memory aligner (core/linmemalign.cpp) "
                 "and no vsg_ctx_set_fallback callback resolved it");
      return VSG_EINVAL;
    }
  }
  int64_t const nal = fb[1], nma = fb[2], nmi = fb[3];
  int32_t const trims4[4] = {static_cast<int32_t>(fb[5]), static_cast<int32_t>(fb[6]), static_cast<int32_t>(fb[7]),
                             static_cast<int32_t>(fb[8])};
  h.aligned = true;
  h.shortest = std::min(qlen, dlen);
  h.longest = std::max(qlen, dlen);
  h.nwscore = static_cast<int>(fb[0]);
  h.forbidden_gap = fb[9] != 0;
  h.nwalignmentlength = static_cast<int>(nal);
  h.nwdiff = static_cast<int>(nal - nma);
  h.nwgaps = static_cast<int>(fb[4]);
  h.nwindels = static_cast<int>(nal - nma - nmi);
  h.matches = static_cast<int>(nal) - h.nwdiff;
  h.mismatches = h.nwdiff - h.nwindels;
  finish_hit(h, trims4, iddef);
  return VSG_OK;
}

// abundance_ratio_cmp (searchcore.cpp:480-537): sign of value - ratio * reference; the double product
// below 2^53, the exact 128-bit product of the ratio's mantissa above it
inline int size_ratio_sign(int64_t value, double ratio, int64_t reference)
{
  if (reference <= 0 || ratio <= 0.0) { return value > 0 ? 1 : 0; }
  if (!std::isfinite(ratio)) { return -1; }
  int64_t const lim = static_cast<int64_t>(1) << 53;
  if (value < lim && reference < lim) {
    double const prod = ratio * static_cast<double>(reference), v = static_cast<double>(value);
    return v < prod ? -1 : (v > prod ? 1 : 0);
  }
  int ex = 0;
  int64_t const mant = static_cast<int64_t>(std::ldexp(std::frexp(ratio, &ex), 53));
  ex -= 53;
  unsigned __int128 lhs = static_cast<uint64_t>(value);
  unsigned __int128 rhs = static_cast<unsigned __int128>(static_cast<uint64_t>(mant)) * static_cast<uint64_t>(reference);
  for (; ex > 0; ex--) { if ((rhs >> 126) != 0) { return -1; } rhs <<= 1; }
  for (; ex < 0; ex++) { if ((lhs >> 126) != 0) { return 1; } lhs <<= 1; }
  return lhs < rhs ? -1 : (lhs > rhs ? 1 : 0);
}

// search_acceptable_unaligned (searchcore.cpp:541-609).  The sequence-content tests (idprefix, idsuffix,
// selfid) arrive as `content`, computed on the device by prefilter_kernel below (0 = all pass).
inline bool acceptable_unaligned(const vsg_search_opts & o, int qseqlen, int64_t dseqlen, int64_t qsize, int64_t tsize,
                          bool same_label, unsigned content)
{
  return (qsize <= o.maxqsize) && (tsize >= o.mintsize) &&
         (size_ratio_sign(qsize, o.minsizeratio, tsize) >= 0) &&
         (size_ratio_sign(qsize, o.maxsizeratio, tsize) <= 0) &&
         (qseqlen >= o.minqt * static_cast<double>(dseqlen)) &&
         (qseqlen <= o.maxqt * static_cast<double>(dseqlen)) &&
         (qseqlen < dseqlen ? qseqlen >= o.minsl * static_cast<double>(dseqlen)
                            : static_cast<double>(dseqlen) >= o.minsl * qseqlen) &&
         (qseqlen < dseqlen ? qseqlen <= o.maxsl * static_cast<double>(dseqlen)
                            : static_cast<double>(dseqlen) <= o.maxsl * qseqlen) &&
         (content == 0u) && (o.self == 0 || !same_label);
}

// search_acceptable_aligned (searchcore.cpp:664-737)
inline bool acceptable_aligned(Hit & h, double opt_id, double opt_weak_id, const vsg_search_opts & o, int qseqlen, int dseqlen,
                               int64_t qsize = 1, int64_t tsize = 1)
{
  double const mid = 100.0 * h.matches / (h.matches + h.mismatches);  // 0/0 -> NaN fails the test, as in the reference
  if (h.id >= 100.0 * opt_weak_id && h.mismatches <= o.maxsubs && h.internal_gaps <= o.maxgaps &&
      !h.forbidden_gap &&  // '*' gap penalties, searchcore.cpp:677-680
      h.internal_alignmentlength >= o.mincols &&
      (o.leftjust == 0 || h.trim_q_left + h.trim_t_left == 0) &&
      (o.rightjust == 0 || h.trim_q_right + h.trim_t_right == 0) &&
      (h.matches + h.mismatches >= o.query_cov * qseqlen) &&
      (h.matches + h.mismatches >= o.target_cov * static_cast<double>(dseqlen)) &&
      h.id <= 100.0 * o.maxid && mid >= o.mid && (h.mismatches + h.internal_indels <= o.maxdiffs)) {
    if (o.unoise != 0) {   // searchcore.cpp:700-717
      double const skew = 1.0 * static_cast<double>(qsize) / static_cast<double>(tsize);
      double const beta = 1.0 / std::pow(2, (1.0 * o.unoise_alpha * h.mismatches) + 1);
      if (skew <= beta || h.mismatches == 0) { h.accepted = true; h.weak = false; return true; }
      h.rejected = true; h.weak = true; return false;
    }
    if (h.id >= 100.0 * opt_id) { h.accepted = true; h.weak = false; return true; }
    h.rejected = true; h.weak = true; return false;
  }
  h.rejected = true; h.weak = false; return false;
}

// hit_compare_byid (searchcore.cpp:133-179)
inline bool hit_less(const Hit & a, const Hit & b)
{
  if (a.rejected != b.rejected) { return a.rejected < b.rejected; }
  if (a.aligned != b.aligned) { return a.aligned > b.aligned; }
  if (!a.aligned) { return false; }
  if (a.id != b.id) { return a.id > b.id; }
  return a.target < b.target;
}

// hit_compare_bysize (searchcore.cpp:182-240): abundance of the target first
inline bool hit_less_bysize(const Hit & a, const Hit & b, int64_t a_size, int64_t b_size)
{
  if (a.rejected != b.rejected) { return a.rejected < b.rejected; }
  if (a.aligned != b.aligned) { return a.aligned > b.aligned; }
  if (!a.aligned) { return false; }
  if (a_size != b_size) { return a_size > b_size; }
  if (a.id != b.id) { return a.id > b.id; }
  return a.target < b.target;
}

}  // namespace vsg
