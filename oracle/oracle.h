/* oracle/oracle.h — TEST INFRASTRUCTURE ONLY (the checker, never the product).
 *
 * Plain-C, scalar restatement of the vsearch hot path (reference @ v2.31.0):
 *   - nw16.c   : the 16-bit saturating affine-gap global aligner `search16`
 *                (src/core/align_simd.cpp:752-1245, 1282-2060), one pair at a time
 *   - ranker.c : unique k-mers, k-mer index, `search_topscores`, and the
 *                accept/reject driver `search_onequery`
 *                (src/core/unique.cpp:155-353, dbindex.cpp:121-255,
 *                 searchcore.cpp:260-464, 541-957, minheap.cpp:82-263)
 *   - nt_maps.c: nucleotide code tables (src/utils/maps.cpp:75-118, 153-266)
 *   - sintax.c : SINTAX's bootstraps for one query (src/commands/sintax.cpp:299-507),
 *                pinned in tests/test_sintax_oracle_cpu.py
 *
 * Parity status: PINNED.  tests/test_oracle_vs_ref.py checks every function here
 * against the unmodified reference compiled into oracle/_ref/libvsref.so
 * (oracle/Makefile, oracle/ref_shim.cpp) on randomized inputs incl. IUPAC codes,
 * lower case, N, empty/length-1 sequences, overflow-provoking lengths; and against
 * the reference's own goldens (api_examples/data/expected_search.tsv) through the
 * committed fixtures in tests/golden/.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs may load this library.
 */
#ifndef VSEARCH_B200_ORACLE_H
#define VSEARCH_B200_ORACLE_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* The 14 scores/penalties in search16_init's own order (align_simd.hpp:76-91):
   match, mismatch, then gap OPEN for (query,target) x (left,interior,right) in the
   order q_l, t_l, q_i, t_i, q_r, t_r, then gap EXTENSION in the same order.
   "open" excludes the first extension, i.e. the values after
   vsearch_apply_defaults_fixups (vsearch.cc:250-259). */
typedef struct oracle_scoring {
  int64_t v[14];
  int n_mismatch;
} oracle_scoring;

#define ORACLE_SENTINEL 32767 /* SHRT_MAX: "not computed, use the scalar fallback" */

/* default vsearch scoring after fixups: +2/-4, interior 20/2 -> open 18, terminal 2/1 -> open 1 */
void oracle_default_scoring(oracle_scoring * s);

/* nt_maps.c */
unsigned char oracle_map_4bit(unsigned char c);
unsigned int oracle_map_2bit(unsigned char c);
unsigned int oracle_map_mask_ambig(unsigned char c);
unsigned int oracle_map_mask_lower(unsigned char c);
int oracle_is_ambiguous_4bit(unsigned int code);
char oracle_complement(unsigned char c);

/* nw16.c — one (query,target) pair exactly as one lane of search16 would treat it.
   cigar must hold qlen+dlen+1 bytes (cigar_cap checked).  Returns 0, or -1 if cigar_cap
   is too small.  score == ORACLE_SENTINEL means diverted (stats 0, cigar ""). */
int oracle_nw16(const oracle_scoring * sc,
                const char * q, int64_t qlen, const char * d, int64_t dlen,
                int16_t * score, uint16_t * aligned, uint16_t * matches,
                uint16_t * mismatches, uint16_t * gaps,
                char * cigar, size_t cigar_cap);

/* search16_fits (align_simd.cpp:130-134) */
int oracle_fits(uint64_t qlen, uint64_t dlen);

/* ranker.c */
/* distinct k-mers in first-occurrence order; mask_lower selects map_mask_lower.
   out needs max(len,1) slots.  Returns the count. */
unsigned int oracle_unique_kmers(int k, const char * seq, int64_t len, int mask_lower,
                                 uint32_t * out);

typedef struct oracle_index oracle_index; /* CSR postings over 4^k k-mers */
oracle_index * oracle_index_build(int k, int n, const char * cat, const int64_t * off,
                                  const int * len, int mask_lower);
void oracle_index_starts(const oracle_index * ix, uint64_t * start);
void oracle_index_postings(const oracle_index * ix, uint32_t * post);
void oracle_index_free(oracle_index * ix);
int oracle_index_wordlength(const oracle_index * ix);
int oracle_index_count(const oracle_index * ix);   /* indexed targets */
/* the postings of k-mer km: *n ascending target numbers */
const uint32_t * oracle_index_list(const oracle_index * ix, uint32_t km, uint64_t * n);

/* search_topscores: best-first (count desc, length asc, seqno asc) list of at most
   tophits targets with count >= min(minwordmatches, nkmers).  Returns the count. */
int oracle_topscores(const oracle_index * ix, const int * target_len,
                     const uint32_t * kmers, unsigned int nkmers,
                     int minwordmatches, int tophits,
                     uint32_t * out_seqno, uint32_t * out_count);

typedef struct oracle_hit {
  int target;
  int strand;
  unsigned int count;
  int accepted, rejected, aligned, weak;
  int nwscore, nwdiff, nwgaps, nwindels, nwalignmentlength;
  int matches, mismatches;
  int internal_alignmentlength, internal_gaps, internal_indels;
  int trim_q_left, trim_q_right, trim_t_left, trim_t_right;
  double id, id0, id1, id2, id3, id4;
  int shortest, longest;
} oracle_hit;

typedef struct oracle_search_opts {
  double id;          /* --id */
  double weak_id;     /* --weak_id (<= id) */
  int maxaccepts;     /* after the seqcount clamp */
  int maxrejects;
  int minwordmatches;
  int tophits;        /* min(maxaccepts+maxrejects+8, seqcount) */
  int iddef;          /* 0..4, default 2 */
  int mask_lower;     /* query k-mer masking mode */
} oracle_search_opts;

/* search_onequery + search_joinhits for one strand: hits kept (accepted|weak), sorted
   by (rejected, aligned desc, id desc, target asc).  Also reports how many pairs and
   cells went through the aligner (the reference's search16 calls). Returns kept count. */
int oracle_search_onequery(const oracle_index * ix, const oracle_scoring * sc,
                           const oracle_search_opts * opt,
                           int n, const char * cat, const int64_t * off, const int * len,
                           const char * q, int qlen, int strand,
                           oracle_hit * hits_out, int hits_cap,
                           int64_t * pairs_aligned, int64_t * cells_aligned);

/* sintax.c — the bootstraps of one query (sintax_query + sintax_search_topscores, src/commands/sintax.cpp:299-507)
   against the index of the whole database.  out is laid out as vsg_sintax_result: out[0] = strand, out[1..2] =
   successful bootstraps per strand, out[3..4] = largest winning count per strand, out[5 + 100 * s + i] = winner i of
   strand s (-1 beyond the successful ones). */
#define ORACLE_SINTAX_BOOTSTRAPS 100
#define ORACLE_SINTAX_SUBSET 32
void oracle_sintax(const oracle_index * ix, const int * target_len, const char * q, int qlen,
                   uint64_t query_number, uint64_t seed, int strand_both, int32_t out[205]);

/* one bootstrap as oracle_sintax saw it */
typedef struct oracle_sintax_boot {
  int32_t winner;            /* -1: no draws, or no target holds two of the sampled k-mers */
  int32_t count;             /* the largest count of any target */
  int32_t ntied;             /* targets with that count */
  int32_t tied_lo, tied_hi;  /* the lowest and the highest number among them */
  int32_t nsamp;             /* distinct sampled k-mers */
  uint32_t samp[ORACLE_SINTAX_SUBSET];
} oracle_sintax_boot;

/* oracle_sintax, and (trace != NULL) every bootstrap of strand s at trace[100 * s + b] */
void oracle_sintax_trace(const oracle_index * ix, const int * target_len, const char * q, int qlen,
                         uint64_t query_number, uint64_t seed, int strand_both, int32_t out[205],
                         oracle_sintax_boot * trace);

#ifdef __cplusplus
}
#endif
#endif
