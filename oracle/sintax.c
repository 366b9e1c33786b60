/* oracle/sintax.c — TEST INFRASTRUCTURE ONLY (the checker, never the product).
 *
 * Scalar restatement of SINTAX's bootstraps for one query: the subsampling of sintax_query and the best target of
 * sintax_search_topscores (reference src/commands/sintax.cpp:299-507), written from their specification, one strand,
 * one bootstrap and one draw at a time:
 *   - the distinct k-mers of each strand in first-occurrence order (no masking of the query); the minus strand is the
 *     reverse complement;
 *   - one SplitMix64 generator per query, seeded with the first output of SplitMix64(seed ^ query_number * gamma); the
 *     plus strand draws first and the minus strand continues the same stream; a strand with fewer than 32 distinct
 *     k-mers draws nothing;
 *   - 100 bootstraps of 32 draws of an index below the distinct count (Lemire's multiply-shift with rejection); an
 *     index drawn twice in a bootstrap counts once;
 *   - per bootstrap, every target's number of sampled k-mers from the index's postings; the winner has the largest
 *     count, then the shorter length, then the lower number, and is kept only if its count is above 1;
 *   - the minus strand iff its largest winning count is higher, or equal with more successful bootstraps.
 */
#include "oracle.h"
#include <stdlib.h>
#include <string.h>

#define BOOTS ORACLE_SINTAX_BOOTSTRAPS
#define SUBSET ORACLE_SINTAX_SUBSET

static uint64_t const GAMMA = 0x9E3779B97F4A7C15ULL;

static uint64_t splitmix_next(uint64_t * state)
{
  *state += GAMMA;
  uint64_t z = *state;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}

/* an index in [0, range): the high word of draw * range, redrawn while the low word falls below 2^64 mod range */
static uint64_t draw_below(uint64_t * state, uint64_t range)
{
  uint64_t const threshold = (0 - range) % range;
  for (;;) {
    unsigned __int128 const p = (unsigned __int128)splitmix_next(state) * range;
    if ((uint64_t)p >= threshold) { return (uint64_t)(p >> 64); }
  }
}

/* one bootstrap: count the sampled k-mers of every target, pick the best */
static void one_bootstrap(const oracle_index * ix, const int * target_len, const uint32_t * samp, int nsamp,
                          uint32_t * count, int32_t * touched, oracle_sintax_boot * r)
{
  int ntouched = 0;
  for (int i = 0; i < nsamp; i++) {
    uint64_t n = 0;
    const uint32_t * list = oracle_index_list(ix, samp[i], &n);
    for (uint64_t j = 0; j < n; j++) {
      if (count[list[j]]++ == 0) { touched[ntouched++] = (int32_t)list[j]; }
    }
  }
  r->winner = -1; r->count = 0; r->ntied = 0; r->tied_lo = -1; r->tied_hi = -1;
  for (int i = 0; i < ntouched; i++) {
    int32_t const t = touched[i];
    int32_t const c = (int32_t)count[t];
    if (c > r->count) {
      r->count = c; r->winner = t; r->ntied = 1; r->tied_lo = t; r->tied_hi = t;
    } else if (c == r->count) {
      r->ntied++;
      if (t < r->tied_lo) { r->tied_lo = t; }
      if (t > r->tied_hi) { r->tied_hi = t; }
      if (target_len[t] < target_len[r->winner] || (target_len[t] == target_len[r->winner] && t < r->winner)) {
        r->winner = t;
      }
    }
    count[t] = 0;
  }
  if (r->count < 2) { r->winner = -1; }
}

void oracle_sintax_trace(const oracle_index * ix, const int * target_len, const char * q, int qlen,
                         uint64_t query_number, uint64_t seed, int strand_both, int32_t out[205],
                         oracle_sintax_boot * trace)
{
  int const k = oracle_index_wordlength(ix);
  int const n = oracle_index_count(ix);
  int const nstrands = strand_both ? 2 : 1;
  size_t const cap = qlen > 0 ? (size_t)qlen : 1;
  char * seq = (char *)malloc(cap);
  uint32_t * kmers = (uint32_t *)malloc(sizeof(uint32_t) * cap);
  uint32_t * count = (uint32_t *)calloc((size_t)n + 1, sizeof(uint32_t));
  int32_t * touched = (int32_t *)malloc(sizeof(int32_t) * ((size_t)n + 1));
  uint8_t * drawn = (uint8_t *)malloc(cap);
  if (!seq || !kmers || !count || !touched || !drawn) { abort(); }

  for (int i = 0; i < 5 + 2 * BOOTS; i++) { out[i] = i < 5 ? 0 : -1; }
  uint64_t state = seed ^ (query_number * GAMMA);
  state = splitmix_next(&state);

  for (int s = 0; s < nstrands; s++) {
    for (int i = 0; i < qlen; i++) { seq[i] = s == 0 ? q[i] : oracle_complement((unsigned char)q[qlen - 1 - i]); }
    unsigned int const distinct = oracle_unique_kmers(k, seq, qlen, 0, kmers);
    for (int b = 0; b < BOOTS; b++) {
      oracle_sintax_boot r;
      memset(&r, 0, sizeof r);
      r.winner = -1; r.tied_lo = -1; r.tied_hi = -1;
      if (distinct >= SUBSET) {
        memset(drawn, 0, distinct);
        for (int j = 0; j < SUBSET; j++) {
          uint64_t const x = draw_below(&state, distinct);
          if (!drawn[x]) { drawn[x] = 1; r.samp[r.nsamp++] = kmers[x]; }
        }
        one_bootstrap(ix, target_len, r.samp, r.nsamp, count, touched, &r);
        if (r.winner >= 0) {
          out[5 + BOOTS * s + out[1 + s]] = r.winner;
          out[1 + s]++;
          if (r.count > out[3 + s]) { out[3 + s] = r.count; }
        }
      }
      if (trace) { trace[s * BOOTS + b] = r; }
    }
  }
  out[0] = nstrands == 2 && (out[4] > out[3] || (out[4] == out[3] && out[2] > out[1])) ? 1 : 0;
  free(seq); free(kmers); free(count); free(touched); free(drawn);
}

void oracle_sintax(const oracle_index * ix, const int * target_len, const char * q, int qlen,
                   uint64_t query_number, uint64_t seed, int strand_both, int32_t out[205])
{
  oracle_sintax_trace(ix, target_len, q, qlen, query_number, seed, strand_both, out, NULL);
}
