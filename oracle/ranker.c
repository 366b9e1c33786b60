/* oracle/ranker.c — TEST INFRASTRUCTURE ONLY (the checker, never the product).
 *
 * Scalar restatement of the k-mer candidate ranker and the per-query accept/reject
 * driver of the reference:
 *   oracle_unique_kmers     unique_count_bitmap / unique_count_hash  (src/core/unique.cpp:155-353)
 *                           (both produce the distinct unmasked k-mers in first-occurrence order;
 *                            the bitmap / CityHash table is only the dedup device)
 *   oracle_index_build      Dbindex::prepare + add_all_sequences      (src/core/dbindex.cpp:121-255)
 *                           restated as pure CSR postings: the reference's per-k-mer bitmaps
 *                           (k-mers present in >= seqcount/8 targets) are a storage variant with the
 *                           same "target t contains k-mer x" meaning
 *   oracle_topscores        search_topscores                          (src/core/searchcore.cpp:260-340)
 *                           + the heap's total order                  (src/core/minheap.cpp:82-136)
 *   oracle_search_onequery  search_onequery / align_delayed / align_trim /
 *                           search_acceptable_aligned / search_joinhits
 *                                                   (src/core/searchcore.cpp:343-464, 664-957, 1028-1052)
 * Pre-alignment filters (search_acceptable_unaligned, :541-609) are at their defaults here
 * (every candidate passes); the non-default ones are length/abundance/label comparisons that do
 * not touch the accelerated path.
 */
#include "oracle.h"
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#include <math.h>

/* k >= 10: the reference switches from the 4^k-bit map to an open-addressing table of 2 * seqlen buckets keyed by the
 * k-mer itself (unique_count_hash, unique.cpp:243-334).  The bucket a k-mer lands in (CityHash there, a
 * multiplicative hash here) decides nothing: a k-mer is reported the first time it is seen, in sequence order. */
static unsigned int unique_kmers_hash(int k, const char * seq, int64_t len, int mask_lower, uint32_t * out)
{
  uint64_t const mask = (1ULL << (2 * k)) - 1ULL;
  uint64_t size = 1;
  while (size < (uint64_t)(2 * len) || size < 2) { size *= 2; }
  uint32_t * tab = (uint32_t *)malloc(sizeof(uint32_t) * (size_t)size);
  if (!tab) { abort(); }
  memset(tab, 0xff, sizeof(uint32_t) * (size_t)size); /* 0xffffffff = empty (a k-mer has at most 30 bits) */
  uint64_t bad = 0, kmer = 0;
  unsigned int unique = 0;
  for (int64_t p = 0; p < len; p++) {
    unsigned char const c = (unsigned char)seq[p];
    bad = (bad << 2) | (mask_lower ? oracle_map_mask_lower(c) : oracle_map_mask_ambig(c));
    kmer = (kmer << 2) | oracle_map_2bit(c);
    if (p >= k - 1) {
      bad &= mask;
      kmer &= mask;
      if (bad == 0) {
        uint64_t j = ((uint32_t)kmer * 2654435761u) & (size - 1);
        while (tab[j] != 0xffffffffu && tab[j] != (uint32_t)kmer) { j = (j + 1) & (size - 1); }
        if (tab[j] == 0xffffffffu) { tab[j] = (uint32_t)kmer; out[unique++] = (uint32_t)kmer; }
      }
    }
  }
  free(tab);
  return unique;
}

unsigned int oracle_unique_kmers(int k, const char * seq, int64_t len, int mask_lower, uint32_t * out)
{
  if (k >= 10) { return unique_kmers_hash(k, seq, len, mask_lower, out); } /* unique.cpp:337-353 */
  uint64_t const size = 1ULL << (2 * k);
  uint64_t const mask = size - 1ULL;
  uint8_t * seen = (uint8_t *)calloc((size_t)(size >> 3) + 1, 1);
  if (!seen) { abort(); }
  uint64_t bad = 0, kmer = 0;
  unsigned int unique = 0;
  for (int64_t p = 0; p < len; p++) {
    unsigned char const c = (unsigned char)seq[p];
    bad = (bad << 2) | (mask_lower ? oracle_map_mask_lower(c) : oracle_map_mask_ambig(c));
    kmer = (kmer << 2) | oracle_map_2bit(c);
    if (p >= k - 1) { /* a full window ends here (unique.cpp:206-229) */
      bad &= mask;
      kmer &= mask;
      if (bad == 0 && !(seen[kmer >> 3] & (1U << (kmer & 7)))) {
        seen[kmer >> 3] |= (uint8_t)(1U << (kmer & 7));
        out[unique++] = (uint32_t)kmer;
      }
    }
  }
  free(seen);
  return unique;
}

struct oracle_index {
  int k;
  int n;            /* indexed sequences; index number == seqno (add_all_sequences order) */
  uint64_t * start; /* k <= 12: 4^k + 1 list heads.  k >= 13 (4^k heads would take gigabytes; the reference pays that,
                       dbindex.cpp:163-182, a test helper need not): nkeys + 1 heads of the k-mers that occur */
  uint32_t * keys;  /* k >= 13: those k-mers, ascending; NULL otherwise */
  uint64_t nkeys;
  uint32_t * post;  /* ascending target numbers per k-mer */
};

static int pair_cmp(const void * a, const void * b)
{
  uint64_t const x = *(uint64_t const *)a, y = *(uint64_t const *)b;
  return x < y ? -1 : (x > y ? 1 : 0);
}

oracle_index * oracle_index_build(int k, int n, const char * cat, const int64_t * off,
                                  const int * len, int mask_lower)
{
  oracle_index * ix = (oracle_index *)calloc(1, sizeof *ix);
  uint64_t const size = 1ULL << (2 * k);
  ix->k = k; ix->n = n;
  int maxlen = 1;
  for (int t = 0; t < n; t++) { if (len[t] > maxlen) { maxlen = len[t]; } }
  uint32_t * tmp = (uint32_t *)malloc(sizeof(uint32_t) * (size_t)maxlen);
  if (k >= 13) {
    /* same postings, found by sorting (k-mer, target) pairs */
    uint64_t total = 0;
    for (int t = 0; t < n; t++) { total += oracle_unique_kmers(k, cat + off[t], len[t], mask_lower, tmp); }
    uint64_t * pairs = (uint64_t *)malloc(sizeof(uint64_t) * (size_t)(total + 1));
    uint64_t m = 0;
    for (int t = 0; t < n; t++) {
      unsigned int const u = oracle_unique_kmers(k, cat + off[t], len[t], mask_lower, tmp);
      for (unsigned int i = 0; i < u; i++) { pairs[m++] = ((uint64_t)tmp[i] << 32) | (uint32_t)t; }
    }
    qsort(pairs, (size_t)m, sizeof(uint64_t), pair_cmp);
    ix->keys = (uint32_t *)malloc(sizeof(uint32_t) * (size_t)(m + 1));
    ix->start = (uint64_t *)malloc(sizeof(uint64_t) * (size_t)(m + 2));
    ix->post = (uint32_t *)malloc(sizeof(uint32_t) * (size_t)(m + 1));
    for (uint64_t i = 0; i < m; i++) {
      uint32_t const km = (uint32_t)(pairs[i] >> 32);
      if (ix->nkeys == 0 || ix->keys[ix->nkeys - 1] != km) { ix->keys[ix->nkeys] = km; ix->start[ix->nkeys] = i; ix->nkeys++; }
      ix->post[i] = (uint32_t)pairs[i];
    }
    ix->start[ix->nkeys] = m;
    free(pairs); free(tmp);
    return ix;
  }
  ix->start = (uint64_t *)calloc((size_t)size + 1, sizeof(uint64_t));
  for (int t = 0; t < n; t++) { /* counting pass (dbindex.cpp:184-200) */
    unsigned int const u = oracle_unique_kmers(k, cat + off[t], len[t], mask_lower, tmp);
    for (unsigned int i = 0; i < u; i++) { ix->start[tmp[i] + 1]++; }
  }
  for (uint64_t i = 0; i < size; i++) { ix->start[i + 1] += ix->start[i]; }
  ix->post = (uint32_t *)malloc(sizeof(uint32_t) * (size_t)(ix->start[size] + 1));
  uint64_t * fill = (uint64_t *)malloc(sizeof(uint64_t) * (size_t)size);
  memcpy(fill, ix->start, sizeof(uint64_t) * (size_t)size);
  for (int t = 0; t < n; t++) { /* fill pass (dbindex.cpp:121-148) */
    unsigned int const u = oracle_unique_kmers(k, cat + off[t], len[t], mask_lower, tmp);
    for (unsigned int i = 0; i < u; i++) { ix->post[fill[tmp[i]]++] = (uint32_t)t; }
  }
  free(fill); free(tmp);
  return ix;
}

/* list of k-mer km: [*a, *b) in ix->post */
static void oracle_list(const oracle_index * ix, uint32_t km, uint64_t * a, uint64_t * b)
{
  if (ix->keys == NULL) { *a = ix->start[km]; *b = ix->start[km + 1]; return; }
  uint64_t lo = 0, hi = ix->nkeys;
  while (lo < hi) { uint64_t const mid = (lo + hi) >> 1; if (ix->keys[mid] < km) { lo = mid + 1; } else { hi = mid; } }
  if (lo < ix->nkeys && ix->keys[lo] == km) { *a = ix->start[lo]; *b = ix->start[lo + 1]; } else { *a = *b = 0; }
}

/* the index as plain arrays (tests compare a UDB file's stored word index with it, udb.cpp:296-350):
 * start has 4^k + 1 entries; post has start[4^k] entries, ascending target numbers per word */
void oracle_index_starts(const oracle_index * ix, uint64_t * start)
{
  uint64_t const size = 1ULL << (2 * ix->k);
  for (uint64_t km = 0; km < size; km++) { uint64_t a, b; oracle_list(ix, (uint32_t)km, &a, &b); start[km + 1] = b - a; }
  start[0] = 0;
  for (uint64_t km = 0; km < size; km++) { start[km + 1] += start[km]; }
}

void oracle_index_postings(const oracle_index * ix, uint32_t * post)
{
  uint64_t const total = ix->keys ? ix->start[ix->nkeys] : ix->start[(size_t)1 << (2 * ix->k)];
  memcpy(post, ix->post, sizeof(uint32_t) * (size_t)total);
}

void oracle_index_free(oracle_index * ix)
{
  if (ix) { free(ix->start); free(ix->keys); free(ix->post); free(ix); }
}

int oracle_index_wordlength(const oracle_index * ix) { return ix->k; }

int oracle_index_count(const oracle_index * ix) { return ix->n; }

const uint32_t * oracle_index_list(const oracle_index * ix, uint32_t km, uint64_t * n)
{
  uint64_t a, b;
  oracle_list(ix, km, &a, &b);
  *n = b - a;
  return ix->post + a;
}

typedef struct { uint32_t count, seqno, length; } elem;

/* best first: count desc, length asc, seqno asc (minheap_compare reversed, minheap.cpp:108-136) */
static int elem_cmp(const void * a, const void * b)
{
  elem const * x = (elem const *)a; elem const * y = (elem const *)b;
  if (x->count != y->count) { return x->count > y->count ? -1 : 1; }
  if (x->length != y->length) { return x->length < y->length ? -1 : 1; }
  if (x->seqno != y->seqno) { return x->seqno < y->seqno ? -1 : 1; }
  return 0;
}

int oracle_topscores(const oracle_index * ix, const int * target_len,
                     const uint32_t * kmers, unsigned int nkmers,
                     int minwordmatches, int tophits,
                     uint32_t * out_seqno, uint32_t * out_count)
{
  uint16_t * cnt = (uint16_t *)calloc((size_t)ix->n + 1, sizeof(uint16_t));
  for (unsigned int i = 0; i < nkmers; i++) {
    uint64_t a, b;
    oracle_list(ix, kmers[i], &a, &b);
    for (uint64_t p = a; p < b; p++) {
      uint16_t * c = &cnt[ix->post[p]];
      if (*c < 32767) { (*c)++; } /* saturate at INT16_MAX (searchcore.cpp:306-315) */
    }
  }
  unsigned int const minmatches = (unsigned int)minwordmatches < nkmers ? (unsigned int)minwordmatches : nkmers;
  elem * cand = (elem *)malloc(sizeof(elem) * ((size_t)ix->n + 1));
  int nc = 0;
  for (int t = 0; t < ix->n; t++) {
    if (cnt[t] >= minmatches) {
      cand[nc].count = cnt[t]; cand[nc].seqno = (uint32_t)t; cand[nc].length = (uint32_t)target_len[t];
      nc++;
    }
  }
  qsort(cand, (size_t)nc, sizeof(elem), elem_cmp);
  int const m = nc < tophits ? nc : tophits;
  for (int i = 0; i < m; i++) { out_seqno[i] = cand[i].seqno; out_count[i] = cand[i].count; }
  free(cand); free(cnt);
  return m;
}

/* first/last CIGAR run -> terminal-gap trims (align_trim, searchcore.cpp:343-464) */
static void trim_and_ids(oracle_hit * h, const char * cigar, int iddef)
{
  h->trim_q_left = h->trim_t_left = h->trim_q_right = h->trim_t_right = 0;
  const char * p = cigar;
  if (*p) {
    long long run = 1; int scan = 0;
    sscanf(p, "%lld%n", &run, &scan);
    char const op = p[scan];
    if (op != 'M') { if (op == 'D') { h->trim_q_left = (int)run; } else { h->trim_t_left = (int)run; } }
  }
  const char * e = cigar + strlen(cigar);
  if (e > cigar) {
    p = e - 1;
    char const op = *p;
    if (op != 'M') {
      while (p > cigar && *(p - 1) <= '9') { p--; }
      long long run = 1;
      sscanf(p, "%lld", &run);
      if (op == 'D') { h->trim_q_right = (int)run; } else { h->trim_t_right = (int)run; }
    }
  }
  if (h->trim_q_left >= h->nwalignmentlength) { h->trim_q_right = 0; }
  if (h->trim_t_left >= h->nwalignmentlength) { h->trim_t_right = 0; }
  int const tr = h->trim_q_left + h->trim_t_left + h->trim_q_right + h->trim_t_right;
  h->internal_alignmentlength = h->nwalignmentlength - tr;
  h->internal_indels = h->nwindels - tr;
  h->internal_gaps = h->nwgaps - ((h->trim_q_left + h->trim_t_left) > 0 ? 1 : 0)
                               - ((h->trim_q_right + h->trim_t_right) > 0 ? 1 : 0);
  h->id0 = h->shortest > 0 ? 100.0 * h->matches / h->shortest : 0.0;
  h->id1 = h->nwalignmentlength > 0 ? 100.0 * h->matches / h->nwalignmentlength : 0.0;
  h->id2 = h->internal_alignmentlength > 0 ? 100.0 * h->matches / h->internal_alignmentlength : 0.0;
  {
    double const x = 100.0 * (1.0 - (1.0 * (h->mismatches + h->nwgaps) / h->longest));
    h->id3 = x > 0.0 ? x : 0.0;
  }
  h->id4 = h->id1;
  switch (iddef) {
    case 0: h->id = h->id0; break; case 1: h->id = h->id1; break; case 2: h->id = h->id2; break;
    case 3: h->id = h->id3; break; default: h->id = h->id4; break;
  }
}

/* search_acceptable_aligned at default option values (searchcore.cpp:664-737) */
static int acceptable_aligned(const oracle_search_opts * o, oracle_hit * h)
{
  double const mid = 100.0 * h->matches / (h->matches + h->mismatches); /* NaN when 0/0, fails >= */
  if (h->id >= 100.0 * o->weak_id && mid >= 0.0 && h->id <= 100.0 * 1.0) {
    if (h->id >= 100.0 * o->id) { h->accepted = 1; h->weak = 0; return 1; }
    h->rejected = 1; h->weak = 1; return 0;
  }
  h->rejected = 1; h->weak = 0; return 0;
}

static int hit_cmp(const void * a, const void * b) /* hit_compare_byid, searchcore.cpp:133-179 */
{
  oracle_hit const * x = (oracle_hit const *)a; oracle_hit const * y = (oracle_hit const *)b;
  if (x->rejected != y->rejected) { return x->rejected < y->rejected ? -1 : 1; }
  if (x->aligned != y->aligned) { return x->aligned > y->aligned ? -1 : 1; }
  if (x->aligned == 0) { return 0; }
  if (x->id > y->id) { return -1; }
  if (x->id < y->id) { return 1; }
  if (x->target != y->target) { return x->target < y->target ? -1 : 1; }
  return 0;
}

int oracle_search_onequery(const oracle_index * ix, const oracle_scoring * sc,
                           const oracle_search_opts * opt,
                           int n, const char * cat, const int64_t * off, const int * len,
                           const char * q, int qlen, int strand,
                           oracle_hit * hits_out, int hits_cap,
                           int64_t * pairs_aligned, int64_t * cells_aligned)
{
  (void)n;
  uint32_t * kmers = (uint32_t *)malloc(sizeof(uint32_t) * (size_t)(qlen > 0 ? qlen : 1));
  unsigned int const nk = oracle_unique_kmers(ix->k, q, qlen, opt->mask_lower, kmers);
  int const th = opt->tophits;
  uint32_t * cs = (uint32_t *)malloc(sizeof(uint32_t) * (size_t)(th + 1));
  uint32_t * cc = (uint32_t *)malloc(sizeof(uint32_t) * (size_t)(th + 1));
  int const ncand = oracle_topscores(ix, len, kmers, nk, opt->minwordmatches, th, cs, cc);
  oracle_hit * hits = (oracle_hit *)calloc((size_t)th + 1, sizeof(oracle_hit));
  int hit_count = 0, accepts = 0, rejects = 0, finalized = 0, delayed = 0, next = 0;
  int64_t np = 0, ncell = 0;

  for (;;) {
    int const more = (finalized + delayed < opt->maxaccepts + opt->maxrejects - 1) &&
                     (rejects < opt->maxrejects) && (accepts < opt->maxaccepts) && (next < ncand);
    if (more) { /* searchcore.cpp:915-944 */
      oracle_hit * h = &hits[hit_count++];
      memset(h, 0, sizeof *h);
      h->target = (int)cs[next]; h->count = cc[next]; h->strand = strand;
      next++;
      delayed++; /* default pre-alignment filters accept every candidate */
    }
    if ((more && delayed == 8) || (!more && delayed > 0)) { /* align_delayed, :740-881 */
      for (int x = finalized; x < hit_count; x++) { /* search16 sees every delayed target */
        int const t = hits[x].target;
        np++; ncell += (int64_t)qlen * (int64_t)len[t];
      }
      for (int x = finalized; x < hit_count; x++) {
        if (rejects < opt->maxrejects && accepts < opt->maxaccepts) {
          oracle_hit * h = &hits[x];
          int const t = h->target;
          int const dlen = len[t];
          size_t const cap = (size_t)qlen + (size_t)dlen + 32;
          char * cigar = (char *)malloc(cap);
          int16_t score; uint16_t al, ma, mi, ga;
          oracle_nw16(sc, q, qlen, cat + off[t], dlen, &score, &al, &ma, &mi, &ga, cigar, cap);
          if (score == ORACLE_SENTINEL) {
            /* the reference re-aligns with LinearMemoryAligner here (:806-832); the oracle
               restates only the 16-bit path and reports the pair as not alignable */
            fprintf(stderr, "oracle_search_onequery: pair diverted to the linear-memory aligner (not restated)\n");
            abort();
          }
          h->aligned = 1;
          h->shortest = qlen < dlen ? qlen : dlen;
          h->longest = qlen > dlen ? qlen : dlen;
          h->nwscore = score;
          h->nwdiff = al - ma;
          h->nwgaps = ga;
          h->nwindels = al - ma - mi;
          h->nwalignmentlength = al;
          h->matches = al - h->nwdiff;
          h->mismatches = h->nwdiff - h->nwindels;
          trim_and_ids(h, cigar, opt->iddef);
          if (acceptable_aligned(opt, h)) { accepts++; } else { rejects++; }
          free(cigar);
        }
      }
      finalized = hit_count;
      delayed = 0;
    }
    if (!more) { break; }
  }

  int kept = 0;
  for (int x = 0; x < hit_count; x++) {
    if ((hits[x].accepted || hits[x].weak) && kept < hits_cap) { hits_out[kept++] = hits[x]; }
  }
  qsort(hits_out, (size_t)kept, sizeof(oracle_hit), hit_cmp);
  if (pairs_aligned) { *pairs_aligned = np; }
  if (cells_aligned) { *cells_aligned = ncell; }
  free(hits); free(cs); free(cc); free(kmers);
  return kept;
}
