/* include/vsg.h — C ABI of libvsg.so, the H100-native (sm_90a CUDA) implementation of the
 * vsearch hot path: the 16-bit affine-gap global aligner `search16` and the k-mer candidate
 * ranker `search_topscores`, batched over many queries.
 *
 * Plain pointers and sizes only; no C++ or torch types cross this boundary.  Every entry point
 * names the reference interface it replaces (reference = torognes/vsearch v2.31.0, paths relative
 * to its src/).  Errors: functions return 0 on success or a negative VSG_E* code and leave a
 * message retrievable with vsg_last_error(); nothing throws (the reference is built
 * -fno-exceptions, Makefile.am:53) and nothing falls back to a CPU path: without a CUDA device
 * vsg_ctx_create fails with VSG_ENODEVICE.
 *
 * In-band "cannot align this pair" is signalled exactly as the reference does it: score ==
 * VSG_SCORE_SENTINEL (SHRT_MAX), zero statistics, empty CIGAR (core/align_simd.cpp:1463-1479,
 * 1838-1846, 1871-1881); the caller re-aligns such pairs with its linear-memory aligner
 * (core/searchcore.cpp:806-832).
 */
#ifndef VSG_H
#define VSG_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VSG_OK 0
#define VSG_ENODEVICE (-1) /* no CUDA device / driver */
#define VSG_ECUDA (-2)     /* a CUDA call failed */
#define VSG_EINVAL (-3)    /* bad argument */
#define VSG_ENOMEM (-4)    /* host or device allocation failed */
#define VSG_ECAP (-5)      /* caller-provided output buffer too small */

#define VSG_SCORE_SENTINEL 32767

typedef struct vsg_ctx vsg_ctx;       /* one per host thread; owns a CUDA stream + scratch  */
typedef struct vsg_seqset vsg_seqset; /* a set of sequences resident in HBM                 */
typedef struct vsg_index vsg_index;   /* k-mer postings index resident in HBM               */

/* Scores/penalties in search16_init's own argument order (core/align_simd.hpp:76-91):
 * v[0]=match v[1]=mismatch, v[2..7]=gap open {query_left,target_left,query_interior,
 * target_interior,query_right,target_right}, v[8..13]=gap extension in the same order.
 * "open" excludes the first extension, i.e. the values vsearch_apply_defaults_fixups leaves
 * in Parameters (vsearch.cc:250-259). */
typedef struct vsg_scoring {
  int64_t v[14];
  int32_t n_mismatch; /* opt_n_mismatch */
} vsg_scoring;

const char * vsg_last_error(void);
const char * vsg_version(void);
/* number of kernels this library has launched in the calling process (bench "gpu_launches") */
int64_t vsg_launch_count(void);

/* ---- context: replaces search16_init / search16_exit (core/align_simd.cpp:1282-1403) ---- */
int vsg_ctx_create(int device, const vsg_scoring * scoring, vsg_ctx ** out);
void vsg_ctx_destroy(vsg_ctx * ctx);
/* the CUDA stream (cudaStream_t) all work of this context is enqueued on */
void * vsg_ctx_stream(vsg_ctx * ctx);
int vsg_ctx_sync(vsg_ctx * ctx);

/* ---- pairs the 16-bit aligner cannot take (score == VSG_SCORE_SENTINEL): the reference re-aligns
 *      them with its scalar LinearMemoryAligner (core/searchcore.cpp:806-832,
 *      commands/allpairs_global.cpp:447-473).  That routine stays on the host side of the boundary:
 *      the embedding application registers it here and vsg_search_batch / vsg_allpairs call it for
 *      exactly those pairs.  query/target are indices into the sequence sets of the call, strand is
 *      1 when the query is to be reverse-complemented.  out[10] = {nwscore, alignment length,
 *      matches, mismatches, gaps, trim_q_left, trim_t_left, trim_q_right, trim_t_right, forbidden}
 *      (trims as in vsg_align_pairs).  `forbidden` (preset to 0) is the application's verdict of
 *      alignment_uses_forbidden_gap (core/searchcore.cpp:612-660): non-zero iff the alignment uses a
 *      gap class whose penalty was given as '*'; such a hit is rejected exactly as
 *      search_acceptable_aligned does (:677-680).  '*' penalties reach the library as values that do
 *      not fit a 16-bit cell, which defers every pair to this callback (align_simd.cpp:1463-1479).
 *      Return 0 on success.  Called from the library's worker threads, possibly
 *      concurrently.  Without a callback such a pair makes the call fail with VSG_EINVAL. ---- */
typedef int (*vsg_fallback_fn)(void * user, int64_t query, int32_t strand, int64_t target, int64_t * out);
int vsg_ctx_set_fallback(vsg_ctx * ctx, vsg_fallback_fn fn, void * user);

/* ---- sequences: replaces Database::add / getsequence / getsequencelen
 *      (core/db.hpp:137-201, core/db.cpp:170-226).  ASCII, one byte per nucleotide, any case,
 *      IUPAC allowed; offsets index into `cat`. `host` selects where cat/off/len live
 *      (1 = host memory; 0 = device memory of ctx's device, e.g. after an NCCL broadcast).  Either way the
 *      data is COPIED (encoded into the library's own symbol buffer): the caller may free its arrays when
 *      the call returns.  A seqset / index belongs to the device of the context that made it; passing it to
 *      a context of another device is an error (VSG_EINVAL). ---- */
int vsg_seqset_create(vsg_ctx * ctx, const char * cat, const int64_t * off, const int32_t * len,
                      int64_t n, int host, vsg_seqset ** out);
void vsg_seqset_destroy(vsg_seqset * s);
int64_t vsg_seqset_count(const vsg_seqset * s);
/* DUST soft-masking in place on the device: replaces dust() / dust_all() (core/mask.cpp:79-188;
 * default --qmask dust / --dbmask dust).  Afterwards lower case marks exactly the regions the
 * reference would have masked; pass mask_lower = 1 to vsg_index_create / vsg_rank / vsg_search_batch. */
int vsg_seqset_dust(vsg_ctx * ctx, vsg_seqset * s);
/* the symbol bytes as stored in HBM (bits 0-3 = 4-bit nucleotide code, bit 4 = lower case), in the
 * order and at the offsets given to vsg_seqset_create; cap >= total sequence bytes.  For tools/tests. */
int vsg_seqset_symbols(vsg_ctx * ctx, const vsg_seqset * s, uint8_t * out, int64_t cap);
/* reverse_complement (utils/reverse_complement.cpp) of the sequences [q0, q0 + n) of `src`, made on the device into a
 * new set of n sequences: entry i is the reverse complement of src's sequence q0 + i.  The complement of an IUPAC code
 * is its complement code, any other byte becomes 'N', and every symbol keeps its case, so a soft mask carries over.
 * q0 / n must lie inside `src` (n = 0 gives an empty set) and `src` must belong to ctx's device, else VSG_EINVAL.
 * E.g. the CIGAR of a minus-strand clustering hit is vsg_align_pairs(ctx, rc, set, ...) with rc the whole set's. */
int vsg_seqset_revcomp(vsg_ctx * ctx, const vsg_seqset * src, int64_t q0, int64_t n, vsg_seqset ** out);

/* ---- batched alignment: replaces search16_qprep + search16 (core/align_simd.cpp:1406-2060)
 *      for npairs (query,target) pairs at once.  qidx[i] indexes `queries`, tidx[i] indexes
 *      `targets`.  Outputs are caller-allocated arrays of npairs elements, identical in meaning
 *      to search16's pscores/paligned/pmatches/pmismatches/pgaps.
 *      trims (optional, may be NULL): 4 x int32 per pair {trim_q_left, trim_t_left, trim_q_right,
 *      trim_t_right} = run length of a leading / trailing D resp. I CIGAR op, before the
 *      "covers the whole alignment" fix-up of align_trim (core/searchcore.cpp:357-417).
 *      CIGARs (optional): if cigar_buf != NULL the NUL-terminated CIGAR of pair i is written at
 *      cigar_buf + cigar_off[i] (cigar_off is an OUTPUT, npairs+1 entries, dense); cigar_cap is
 *      the buffer size; VSG_ECAP if it does not fit (a capacity of sum(qlen+dlen+1) always fits).
 *      All pointers are HOST pointers; the sequences themselves are already resident in HBM
 *      (vsg_seqset_create), only the pair list goes up and the fixed-size results come back. ---- */
int vsg_align_pairs(vsg_ctx * ctx, const vsg_seqset * queries, const vsg_seqset * targets,
                    int64_t npairs, const uint32_t * qidx, const uint32_t * tidx,
                    int16_t * score, uint16_t * aligned, uint16_t * matches,
                    uint16_t * mismatches, uint16_t * gaps, int32_t * trims,
                    char * cigar_buf, int64_t cigar_cap, int64_t * cigar_off);

/* vsg_align_pairs (statistics only) with traceback on demand, as vsg_search_batch calls it.  For tools/tests.
 *      leader_of[i] = -1 for a group leader or an ungated pair, else the index in this call of pair i's leader,
 *      which must itself have -1 (VSG_EINVAL otherwise).  A follower whose leader passes the identity test
 *      (threshold = 100 * id + margin, under iddef) may come back "not computed": aligned = matches = mismatches =
 *      0xffff, trims and gaps unspecified; its score is always computed.  ck_counts (optional, 3 x int64): checkpoint
 *      tasks that stored their checkpoints, that ran score-only, and the score-only ones re-run with stores. */
int vsg_align_pairs_gated(vsg_ctx * ctx, const vsg_seqset * queries, const vsg_seqset * targets,
                          int64_t npairs, const uint32_t * qidx, const uint32_t * tidx,
                          int16_t * score, uint16_t * aligned, uint16_t * matches,
                          uint16_t * mismatches, uint16_t * gaps, int32_t * trims,
                          const int32_t * leader_of, double threshold, int iddef, int64_t * ck_counts);

/* Layout of the per-pair statistics record the kernels produce (8 x int32, device side);
 * exposed so that tools reading the raw buffers agree on it. */
#define VSG_STAT_SCORE 0
#define VSG_STAT_ALIGNED 1
#define VSG_STAT_MATCHES 2
#define VSG_STAT_MISMATCHES 3
#define VSG_STAT_GAPS 4
#define VSG_STAT_TRIM_LEFT 5  /* +run: leading D (gap in target) ; -run: leading I ; 0: leading M */
#define VSG_STAT_TRIM_RIGHT 6 /* same for the trailing op */
#define VSG_STAT_CIGARLEN 7   /* strlen of the CIGAR */
#define VSG_STAT_WORDS 8

/* Cumulative device-side profile of this context since the last vsg_profile_reset: DP cells
 * (sum qlen*dlen of the pairs that went through a forward kernel), forward / traceback / ranker
 * kernel time (cudaEvents on the context's stream, ms), pair counts per kernel and the number of
 * forward launches.  bench.py computes its roofline from these. */
typedef struct vsg_profile {
  int64_t cells;
  int64_t fast_pairs;
  int64_t exact_pairs;
  int64_t fwd_launches;
  float fwd_ms;
  float traceback_ms;
  float rank_ms;
  float reserved;
  int64_t tb_skipped;   /* pairs whose walk back was skipped by traceback on demand (vsg_search_batch; their DP was computed) */
  int64_t tb_redone;    /* skipped pairs vsg_search_batch needed after all and re-aligned one by one: the device's verdict
                           on their group leader differed from the host's (only a borderline identity can do that) */
} vsg_profile;
int vsg_profile_reset(vsg_ctx * ctx);
int vsg_profile_get(vsg_ctx * ctx, vsg_profile * out);
/* Measured integer issue peak of this device: thread-instructions per second of an even mix of packed 16x2 DPX
 * (ALU pipe) and 32-bit multiply-add (FMA pipe) instructions with no memory traffic — each processes the two
 * packed cells of a register, so 2 x this / (instructions per cell pair) is the DP roofline's denominator. */
int vsg_measure_int_peak(vsg_ctx * ctx, double * packed_lane_ops_per_s);

/* ---- k-mer index: replaces Dbindex::prepare + add_all_sequences + the getters
 *      (core/dbindex.hpp:79-120, core/dbindex.cpp:121-255).  mask_lower != 0 means soft-masked
 *      (lower-case) symbols do not seed k-mers (unique.cpp:198-199). ---- */
int vsg_index_create(vsg_ctx * ctx, const vsg_seqset * db, int wordlength, int mask_lower,
                     vsg_index ** out);
void vsg_index_destroy(vsg_index * ix);
/* wordlength 3..15, as the reference (cli.cc --wordlength).  3..10: list heads for all 4^k words per shard of 32 766
 * targets, targets de-duplicated through a bitmap (unique_count_bitmap, core/unique.cpp:155-240).  11..15: only the
 * words that occur get a list, found by sorting (what unique_count_hash's table finds, core/unique.cpp:243-334),
 * looked up by binary search. */

/* ---- candidate ranking: replaces unique_count + search_topscores + minheap
 *      (core/unique.cpp:337-353, core/searchcore.cpp:260-340, core/minheap.cpp) for every query
 *      of `queries` in [q0, q0+nq).  For query q the best-first list (count desc, target length
 *      asc, target number asc) of at most tophits targets with count >= min(minwordmatches,
 *      number of distinct query k-mers) is written to cand_seqno/cand_count[(q-q0)*tophits ...],
 *      its length to ncand[q-q0].  Host pointers.  Any tophits >= 1: up to 1024 the lists are kept in shared
 *      memory; above, every target at the threshold is counted, written out and sorted in device memory. ---- */
int vsg_rank(vsg_ctx * ctx, const vsg_index * ix, const vsg_seqset * queries, int64_t q0,
             int64_t nq, int minwordmatches, int tophits, int mask_lower,
             uint32_t * cand_seqno, uint32_t * cand_count, int32_t * ncand);
/* CTAs per SM the device holds of the ranker's two instances (cudaOccupancyMaxActiveBlocksPerMultiprocessor): the
 * full one, and the short-query one that vsg_rank and vsg_search_batch use when tophits <= 64 and every query of the
 * call has np2 + nwin + 1 <= 512 (nwin: its k-mer windows; np2: nwin rounded up to a power of two; at wordlength 8,
 * queries of up to 262 nt). */
int vsg_rank_occupancy(vsg_ctx * ctx, int * ctas_full, int * ctas_short);

/* ---- whole-path search: replaces search_batch (core/search.hpp:135-145, search.cpp:511-593) /
 *      the body of search_thread_run (commands/usearch_global.cpp:376-497) for plus-strand (and
 *      optionally minus-strand) queries with the reference's default pre-alignment filters.
 *      result layout mirrors search_result_s (core/search.hpp:67-80). ---- */
typedef struct vsg_search_opts {
  double id;              /* --id                         */
  double weak_id;         /* --weak_id (10.0 = default)   */
  int32_t maxaccepts;     /* --maxaccepts (default 1)     */
  int32_t maxrejects;     /* --maxrejects (default 32)    */
  int32_t wordlength;     /* --wordlength (default 8)     */
  int32_t minwordmatches; /* <0: reference default table  */
  int32_t iddef;          /* --iddef (default 2)          */
  int32_t strand_both;    /* --strand both                */
  int32_t mask_lower;     /* queries are soft-masked      */
  int32_t lazy;           /* 0 (default): align exactly the groups of <= 8 candidates the reference
                             hands to search16; 1: align a candidate only when the replay is about to
                             examine it (same decisions and hit tables, fewer DP cells)           */
  /* optional accept/reject filters, reference defaults from vsg_search_opts_default():
     before alignment (search_acceptable_unaligned, core/searchcore.cpp:573-587) */
  double minqt, maxqt;    /* --minqt / --maxqt : query/target length ratio          */
  double minsl, maxsl;    /* --minsl / --maxsl : shorter/longer length ratio        */
  /* after alignment (search_acceptable_aligned, core/searchcore.cpp:671-699) */
  double maxid;           /* --maxid  (1.0)                */
  double mid;             /* --mid    (0.0)                */
  double query_cov;       /* --query_cov (0.0)             */
  double target_cov;      /* --target_cov (0.0)            */
  int64_t maxsubs;        /* --maxsubs  (INT_MAX)          */
  int64_t maxgaps;        /* --maxgaps  (INT_MAX)          */
  int64_t mincols;        /* --mincols  (0)                */
  int64_t maxdiffs;       /* --maxdiffs (INT_MAX)          */
  int32_t leftjust;       /* --leftjust                    */
  int32_t rightjust;      /* --rightjust                   */
  /* the remaining pre-alignment filters of search_acceptable_unaligned (core/searchcore.cpp:561-608);
     vsg_search_batch only (vsg_allpairs ignores them, as allpairs_global's defaults do) */
  int64_t maxqsize;       /* --maxqsize (INT64_MAX): query abundance <= maxqsize           */
  int64_t mintsize;       /* --mintsize (0):         target abundance >= mintsize          */
  double minsizeratio;    /* --minsizeratio (0.0):   query abundance >= ratio * target's   */
  double maxsizeratio;    /* --maxsizeratio (DBL_MAX)                                      */
  int32_t idprefix;       /* --idprefix (0): first n nucleotides identical (compared on the device) */
  int32_t idsuffix;       /* --idsuffix (0): last n nucleotides identical                   */
  int32_t self;           /* --self:   reject a target whose label equals the query's      */
  int32_t selfid;         /* --selfid: reject a target whose sequence equals the query's   */
  int32_t qmask_dust;     /* --qmask dust with --strand both: the caller has DUST-masked `queries`
                             (vsg_seqset_dust); the reverse complements made inside the call are masked
                             on their own, as search_batch_worker_fn does per strand (core/search.cpp:437-449) */
  int32_t unoise;         /* --cluster_unoise acceptance (searchcore.cpp:700-717): a hit that passes the filters is accepted
                             iff it has no mismatch or query abundance / target abundance <= 1 / 2^(unoise_alpha * mismatches + 1),
                             instead of the --id test; needs query_sizes / target_sizes */
  const int64_t * query_sizes;   /* abundance of query q0+i at [i]; NULL = 1 everywhere (db.getabundance / qsize) */
  const int64_t * target_sizes;  /* abundance of target t at [t];   NULL = 1 everywhere                     */
  const int64_t * query_labels;  /* --self: label identities, [i] for query q0+i resp. [t] for target t; two  */
  const int64_t * target_labels; /*         sequences carry the same header iff their identities are equal  */
  double unoise_alpha;    /* --unoise_alpha (2.0) */
  int32_t sizeorder;      /* --sizeorder (vsg_cluster_fast / sessions, with maxaccepts > 1): among the accepted hits the centroid of
                             highest abundance wins, then identity, then the earlier one (search_findbest2_bysize,
                             searchcore.cpp:182-240, 994-1025) instead of identity first; needs target_sizes */
  int32_t reserved1;
} vsg_search_opts;

typedef struct vsg_search_result {
  int32_t target;
  int32_t matches;
  int32_t mismatches;
  int32_t gaps;
  int32_t alignment_length;
  int32_t query_length;
  int32_t target_length;
  int32_t accepted;
  int32_t strand;
  int32_t nwscore;
  double id;
  int32_t internal_alignment_length;   /* alignment columns / gap opens without the terminal gaps that align_trim   */
  int32_t internal_gaps;               /* removes (core/searchcore.cpp:409-463): the --blast6out columns 4 and 6     */
} vsg_search_result;

void vsg_search_opts_default(vsg_search_opts * o);
/* results[(q)*max_results + j], counts[q]; work (optional, 4 x int64): {pairs, DP cells} the
 * reference's driver hands to search16 for the same queries, then {pairs, DP cells} actually
 * aligned here (identical unless opts->lazy). */
int vsg_search_batch(vsg_ctx * ctx, const vsg_index * ix, const vsg_seqset * db,
                     const vsg_seqset * queries, int64_t q0, int64_t nq,
                     const vsg_search_opts * opts, vsg_search_result * results, int max_results,
                     int32_t * counts, int64_t * work);
/* The same search with variable-length hit lists, for limits that leave a query thousands of hits (--maxaccepts 0
 * --maxrejects 0: every target, usearch_global.cpp:598-614).  The rows of query q0+i are hits[first[i] .. first[i+1])
 * (first: nq + 1 offsets), at most maxhits of them (0: all), in search_joinhits order: the rows vsg_search_batch gives
 * with a large enough max_results.  *nhits receives the number of rows produced; if it exceeds cap the call returns
 * VSG_ECAP with first filled and hits untouched.  work as for vsg_search_batch. */
int vsg_search_hits(vsg_ctx * ctx, const vsg_index * ix, const vsg_seqset * db, const vsg_seqset * queries, int64_t q0,
                    int64_t nq, const vsg_search_opts * opts, int64_t maxhits, vsg_search_result * hits, int64_t cap,
                    int64_t * first, int64_t * nhits, int64_t * work);

/* ---- all-against-all: replaces the per-query body of allpairs_thread_run
 *      (commands/allpairs_global.cpp:340-549) for query rows [row0, row0+nrows) of `set`: every
 *      target j > i is aligned (no k-mer filter, default pre-alignment filters), a pair is kept iff
 *      search_acceptable_aligned accepts it (id >= opts->id under opts->iddef), kept pairs of a
 *      query are ordered by (id desc, target asc) as allpairs_hit_compare does, queries ascending.
 *      hits: caller-allocated, `cap` records; *nhits receives the number produced (VSG_ECAP if it
 *      exceeds cap).  Rows are independent, so N GPUs take disjoint row ranges (SURVEY.md §8e).
 *      work (optional, 2 x int64): pairs and DP cells aligned. ---- */
typedef struct vsg_pair_hit {
  int32_t query;
  int32_t target;
  int32_t matches;
  int32_t mismatches;
  int32_t gaps;
  int32_t alignment_length;
  int32_t nwscore;
  int32_t internal_alignment_length;
  double id;
} vsg_pair_hit;
/* Row ranges of equal DP work for `nparts` workers (GPUs): bounds[p] .. bounds[p+1] are the rows of
 * part p, chosen so that every part has about the same sum over its rows i of len[i] * (sum of len[j],
 * j > i) — the triangle balancing SURVEY.md §8(e) asks for; equal row counts would give the first
 * GPU almost twice the work of the average.  Pure host arithmetic; bounds has nparts+1 entries. */
int vsg_allpairs_partition(const int32_t * len, int64_t n, int nparts, int64_t * bounds);
int vsg_allpairs(vsg_ctx * ctx, const vsg_seqset * set, int64_t row0, int64_t nrows,
                 const vsg_search_opts * opts, vsg_pair_hit * hits, int64_t cap, int64_t * nhits,
                 int64_t * work);

/* ---- greedy centroid clustering: replaces cluster_core_parallel / cluster_core_serial with cluster_query_core,
 *      evaluate_extra_hits and Dbindex::add_sequence (core/cluster.cpp:162-189, 601-856, 877-1115;
 *      core/dbindex.cpp:121-148) for --cluster_fast-style clustering of `set` IN THE ORDER GIVEN (the reference
 *      sorts by decreasing length first, core/db.cpp:433-449; mask the set with vsg_seqset_dust and pass
 *      opts->mask_lower = 1 for the default --qmask dust).  round_size = the reference's --threads: sequences are
 *      searched in rounds of that many against the centroids found so far and then resolved one by one, centroids
 *      of the same round included (cluster.cpp:881-882, 946-1025) — the assignments depend on it, so compare
 *      with `vsearch --cluster_fast --threads round_size`.  results[i] for sequence i: its cluster number
 *      (creation order of the centroids) and either centroid = -1 (it founded the cluster: an "S" record of
 *      --uc) or the sequence number of the centroid it matched plus that alignment's statistics and identity
 *      (an "H" record; the CIGAR is one vsg_align_pairs call away).  NOTE the reference's default --maxrejects for
 *      --cluster_fast is 8, not 32 (cli.cc:4163-4172): set opts->maxrejects accordingly.  opts: id, iddef, maxaccepts, maxrejects,
 *      wordlength, minwordmatches, mask_lower, strand_both, the length / abundance / post-alignment filters (target_sizes
 *      and target_labels are per sequence of `set`).  strand_both = --strand both (cluster.cpp:162-189, 920-957): every
 *      sequence is also searched as its reverse complement, which keeps the set's soft mask; strand = 1 marks a hit
 *      of the reverse complement (the "-" of --uc column 5), whose statistics and CIGAR are those of the reverse-complemented
 *      sequence against the centroid: vsg_align_pairs(ctx, rc, set, ...) with rc from vsg_seqset_revcomp.  A centroid is
 *      always its plus strand.  A pair deferred to the fallback callback reaches it as (sequence, strand, centroid).
 *      The both-strands query set costs 2 bytes of device memory per nucleotide of `set`.  Any maxaccepts / maxrejects
 *      is offered, clamped as cluster() clamps them (0 or more than the set: the number of sequences,
 *      core/cluster.cpp:1213-1235), so --maxaccepts 0 --maxrejects 0 clusters exhaustively.  Above
 *      maxaccepts + maxrejects + 8 = 1024 every round's candidates are kept on the host: about 144 bytes per candidate of
 *      the round's query strands (a hit record and a list entry).  work (optional, 2 x int64): pairs and DP cells handed
 *      to the aligner, both strands counted. ---- */
typedef struct vsg_cluster_result {
  int32_t cluster;
  int32_t centroid;
  int32_t matches;
  int32_t mismatches;
  int32_t gaps;
  int32_t alignment_length;
  int32_t nwscore;
  int32_t strand;
  double id;
} vsg_cluster_result;
int vsg_cluster_fast(vsg_ctx * ctx, const vsg_seqset * set, const vsg_search_opts * opts, int round_size,
                     vsg_cluster_result * results, int64_t * nclusters, int64_t * work);

/* ---- the same clustering as a SESSION that is fed ranges of the set: replaces cluster_session_init /
 *      cluster_assign_single / cluster_assign_batch / cluster_session_cleanup (core/cluster.hpp:78-118,
 *      core/cluster.cpp:1633-1930).  The session owns the device index of the centroids found so far and the cluster
 *      numbers; `set` (already masked and sorted, as for vsg_cluster_fast), the context and the arrays `opts` points
 *      to must outlive it.  vsg_cluster_session_assign handles the sequences [start, start + count) in rounds of
 *      round_size (cluster_assign_batch: the caller's --threads; cluster_assign_single: count = round_size = 1);
 *      ranges must be ascending and contiguous (cluster.hpp:104-111), results[i] belongs to sequence start + i.
 *      A session fed the whole set in one call gives vsg_cluster_fast's results.  It offers the same limits (any
 *      maxaccepts / maxrejects, clamped as vsg_cluster_fast clamps them) at the same host memory per round. ---- */
typedef struct vsg_cluster_session vsg_cluster_session;
int vsg_cluster_session_create(vsg_ctx * ctx, const vsg_seqset * set, const vsg_search_opts * opts, vsg_cluster_session ** out);
int vsg_cluster_session_assign(vsg_cluster_session * session, int64_t start, int64_t count, int round_size,
                               vsg_cluster_result * results);
int64_t vsg_cluster_session_clusters(const vsg_cluster_session * session);
void vsg_cluster_session_destroy(vsg_cluster_session * session);

/* ---- the cluster driver's own index of the centroids, exposed for tests: the incremental k-mer index that
 *      vsg_cluster_fast, cluster sessions and vsg_cluster_command grow as centroids are created (shards of 32 768
 *      targets; wordlength 3..10).  Every list capacity is sized from the whole `set`, which must outlive the index.
 *      vsg_cluster_index_append adds the sequences seqnos[0 .. n) as new targets; their numbers must be strictly
 *      ascending, after the last one appended and inside the set (VSG_EINVAL otherwise).  Targets get DENSE numbers in
 *      append order, and vsg_cluster_index_rank returns those: as vsg_rank, for every query of `queries` in [q0, q0+nq)
 *      the best-first list (count desc, target length asc, dense number asc) of at most tophits targets with count >=
 *      min(minwordmatches, distinct query k-mers), with the index's mask_lower on the query side; tophits > 1024 takes
 *      the unbounded lists. ---- */
typedef struct vsg_cluster_index vsg_cluster_index;
int vsg_cluster_index_create(vsg_ctx * ctx, const vsg_seqset * set, int wordlength, int mask_lower, vsg_cluster_index ** out);
int vsg_cluster_index_append(vsg_ctx * ctx, vsg_cluster_index * ix, const uint32_t * seqnos, int64_t n);
int64_t vsg_cluster_index_count(const vsg_cluster_index * ix);
int vsg_cluster_index_rank(vsg_ctx * ctx, vsg_cluster_index * ix, const vsg_seqset * queries, int64_t q0, int64_t nq,
                           int minwordmatches, int tophits, uint32_t * cand, uint32_t * count, int32_t * ncand);
void vsg_cluster_index_destroy(vsg_cluster_index * ix);

/* ---- several GPUs behind one process (SURVEY.md §8e; the reference is a single process, LIBRARY_API.md:138-156):
 *      vsg_group_create uploads the database ONCE (to devices[0]; dust_db != 0 also DUST-masks it there,
 *      core/mask.cpp dust_all), copies the packed sequences device to device over NVLink to every other GPU and
 *      builds the k-mer index on each.  vsg_group_search shards the queries (host arrays, as for
 *      vsg_seqset_create) into contiguous ranges of equal nucleotide count, one per device, and runs
 *      vsg_search_batch on all devices concurrently; results land in the caller's arrays in query order.
 *      vsg_group_allpairs shards the rows of the group's own sequence set with vsg_allpairs_partition.  No
 *      collective is involved beyond the one-to-all copy of the database.  stats: ms3 = {upload+mask on the first
 *      device, device-to-device copies, index builds}, bytes copied between devices. ---- */
typedef struct vsg_group vsg_group;
int vsg_group_create(const int * devices, int ndev, const vsg_scoring * scoring, const char * cat,
                     const int64_t * off, const int32_t * len, int64_t n, int wordlength, int mask_lower,
                     int dust_db, vsg_group ** out);
void vsg_group_destroy(vsg_group * g);
int vsg_group_size(const vsg_group * g);
vsg_ctx * vsg_group_ctx(vsg_group * g, int i);
vsg_seqset * vsg_group_db(vsg_group * g, int i);
vsg_index * vsg_group_index(vsg_group * g, int i);
int vsg_group_stats(const vsg_group * g, double * ms3, int64_t * broadcast_bytes);
int vsg_group_set_fallback(vsg_group * g, vsg_fallback_fn fn, void * user);
int vsg_group_search(vsg_group * g, const char * qcat, const int64_t * qoff, const int32_t * qlen, int64_t nq,
                     int dust_queries, const vsg_search_opts * opts, vsg_search_result * results, int max_results,
                     int32_t * counts, int64_t * work);
/* vsg_group_search with the hit lists of vsg_search_hits: query i's rows are hits[first[i] .. first[i+1]) */
int vsg_group_search_hits(vsg_group * g, const char * qcat, const int64_t * qoff, const int32_t * qlen, int64_t nq,
                          int dust_queries, const vsg_search_opts * opts, int64_t maxhits, vsg_search_result * hits,
                          int64_t cap, int64_t * first, int64_t * nhits, int64_t * work);
int vsg_group_allpairs(vsg_group * g, const vsg_search_opts * opts, vsg_pair_hit * hits, int64_t cap,
                       int64_t * nhits, int64_t * work);

/* ---- streaming --usearch_global driver (SURVEY.md §8 f1): replaces the query loop of search_thread_run /
 *      search_output_results (commands/usearch_global.cpp:150-300, 376-534) for FASTA in, --blast6out out
 *      (core/results.cpp:221-271).  Three stages run concurrently on batches of batch_queries sequences:
 *      a reader thread parses the FASTA file (headers cut at the first blank unless notrunclabels), the calling
 *      thread runs vsg_group_search on every GPU of the group (query upload, optional DUST, ranking, alignment,
 *      accept/reject, hit table download), a writer thread formats the rows of min(maxhits, hits) per query IN INPUT
 *      ORDER (the reference's order with --threads 1).  target_labels: the database headers as the reference would
 *      print them.  output_no_hits != 0: the "*" row for queries without a hit.  stats (optional) receives counts and
 *      the busy seconds of each stage. ---- */
typedef struct vsg_stream_stats {
  int64_t queries, matched, rows, batches, nucleotides;
  double parse_s, search_s, write_s, wall_s;
} vsg_stream_stats;
int vsg_usearch_stream(vsg_group * g, const char * const * target_labels, const char * query_fasta,
                       const vsg_search_opts * opts, int qmask_dust, int notrunclabels, int batch_queries,
                       int64_t maxhits, int output_no_hits, const char * blast6out_path, vsg_stream_stats * stats);

/* ---- UDB database files (SURVEY.md §8 f3): replaces udb_detect_isudb and udb_read (core/udb.cpp:120-175, 196-578).
 *      vsg_udb_detect: 1 if the file starts with the UDB signature, 0 if not, < 0 on error.  vsg_udb_open parses and
 *      validates the whole file on the host (no GPU needed; every "Invalid UDB file" check of udb_read, as VSG_EINVAL);
 *      the accessors hand out views that live until vsg_udb_close: the sequences (ASCII, back to back; case carries
 *      the masking the file was made with), the NUL-terminated headers, the stored word index (kmercount[4^k], then
 *      the ascending sequence numbers of every word).  vsg_udb_load makes the device-resident database: sequences
 *      uploaded, the device index built at the file's word length and CHECKED against the stored one (per word, the
 *      number of sequences holding it); *mask_lower (optional) receives whether the stored index excludes lower-case
 *      symbols (--dbmask dust/soft when the file was made) — pass it on as the index's masking.  A file whose stored
 *      counts match neither convention is rejected.  vsg_group_create_udb: the same for a vsg_group. ---- */
typedef struct vsg_udb vsg_udb;
typedef struct vsg_udb_info {
  int64_t sequences, nucleotides, header_chars, index_entries, longest_header;
  int32_t wordlength, dbaccel, shortest, longest;
} vsg_udb_info;
int vsg_udb_detect(const char * path);
int vsg_udb_open(const char * path, vsg_udb ** out);
void vsg_udb_close(vsg_udb * udb);
int vsg_udb_info_get(const vsg_udb * udb, vsg_udb_info * out);
int vsg_udb_sequences(const vsg_udb * udb, const char ** cat, const int64_t ** off, const int32_t ** len);
const char * vsg_udb_header(const vsg_udb * udb, int64_t i);
int vsg_udb_words(const vsg_udb * udb, const uint32_t ** kmercount, const uint32_t ** kmerindex);
int vsg_udb_load(vsg_ctx * ctx, const vsg_udb * udb, vsg_seqset ** db, vsg_index ** index, int * mask_lower);
int vsg_group_create_udb(const int * devices, int ndev, const vsg_scoring * scoring, const vsg_udb * udb, vsg_group ** out);

/* ---- making UDB files: replaces makeudb_usearch (commands/makeudb_usearch.cpp:105-273) with Dbindex::prepare /
 *      add_all_sequences (core/dbindex.cpp:121-255) built on the device.  vsg_udb_make makes, from n records as db.read
 *      keeps them (any case; headers as they go into the file), the same in-memory database vsg_udb_open makes from a
 *      file: the records upper-cased (db.read(..., upcase = 1)), with --dbmask dust DUST-masked on the device (masked
 *      symbols lower case, or 'N' with hardmask), and the word index at `wordlength` built on the device: per word the
 *      ascending numbers of the sequences holding it, from the windows without a masked symbol (outside ACGTU; with
 *      --dbmask soft or dust also lower case).  Every accessor, vsg_udb_load and vsg_group_create_udb take the result.
 *      The device scratch is bounded by a quarter of the context's direction-bit budget (VSG_DIR_BUDGET_MB), at most
 *      1 GiB; the host holds kmercount[4^k] (4 GiB at k = 15) and the index.  The length limits of opts are not applied
 *      here.  vsg_udb_write writes the file makeudb_usearch writes, byte for byte; a failed write removes the file.
 *      vsg_makeudb_usearch is the --makeudb_usearch command: FASTA or FASTQ in (the format from the first byte; gzip and
 *      bzip2 refused), labels cut at the first blank unless notrunclabels, db.read's symbol rules (FASTA: core/fasta.cpp's
 *      table, other printable symbols stripped and counted, '.', '-' and control characters an error naming the line;
 *      FASTQ: IUPAC letters only), records outside [minseqlength, maxseqlength] discarded and counted (minseqlength < 1:
 *      no lower bound), then vsg_udb_make and vsg_udb_write.  A file is written even when every record is discarded
 *      (the reference's own reader, and vsg_udb_open, refuse such a file).  Errors leave no output file. ---- */
#define VSG_DBMASK_NONE 0
#define VSG_DBMASK_SOFT 1
#define VSG_DBMASK_DUST 2
typedef struct vsg_makeudb_opts {
  int32_t wordlength;     /* --wordlength, 3..15 (default 8) */
  int32_t dbmask;         /* --dbmask: VSG_DBMASK_NONE / _SOFT / _DUST (default dust) */
  int32_t hardmask;       /* --hardmask: DUST-masked symbols become 'N' (no effect with soft or none: the input is upper-cased) */
  int32_t notrunclabels;  /* --notrunclabels */
  int64_t minseqlength;   /* --minseqlength (default 32 for this command, cli.cc) */
  int64_t maxseqlength;   /* --maxseqlength (default 50 000) */
} vsg_makeudb_opts;
void vsg_makeudb_opts_default(vsg_makeudb_opts * opts);
typedef struct vsg_makeudb_stats {
  int64_t sequences;          /* records kept */
  int64_t discarded_short, discarded_long;
  int64_t stripped;           /* FASTA symbols stripped with a warning by the reference (digits, '*', blanks, ...) */
  int64_t nucleotides, index_entries;
  double parse_s, device_s, write_s, wall_s;
} vsg_makeudb_stats;
int vsg_udb_make(vsg_ctx * ctx, const char * cat, const int64_t * off, const int32_t * len, const char * const * headers,
                 int64_t n, const vsg_makeudb_opts * opts, vsg_udb ** out);
int vsg_udb_write(const vsg_udb * udb, const char * path);
int vsg_makeudb_usearch(vsg_ctx * ctx, const char * input_path, const vsg_makeudb_opts * opts, const char * output_path,
                        vsg_makeudb_stats * stats);

/* ---- SINTAX taxonomy classification: replaces sintax_query / sintax_search_topscores / sintax_analyse
 *      (commands/sintax.cpp:138-516) for --sintax with --randseed.  vsg_sintax runs the 100 bootstraps of every query
 *      of `queries` in [q0, q0 + nq) and of its reverse complement (strand_both) against an index made by
 *      vsg_index_create / vsg_udb_load: per strand, the distinct k-mers of the query in first-occurrence order (no
 *      masking but non-ACGTU; unique_count, core/unique.cpp:155-353), 32 draws per bootstrap from one SplitMix64
 *      generator per query seeded with random_substream_seed(seed, query number) (utils/random.cpp:70-91, plus strand
 *      first, minus strand continuing its stream), and per bootstrap the target with the most sampled k-mers (ties:
 *      shorter, then lower number), kept when its count is > 1.  out[i] belongs to query q0 + i.  A strand with fewer
 *      than 32 distinct k-mers has no bootstraps.  The database must hold what db.read keeps for --sintax: sequences of
 *      at least 32 nt (core/db.cpp minseqlength).  vsg_sintax_rows needs no device: the --tabbedout rows of nq results
 *      (the vote over the winners' tax= fields, core/tax.cpp:70-186), written back to back into buf; *len receives
 *      the bytes needed, VSG_ECAP (buf untouched) when they exceed cap.  target_headers are the full database headers
 *      (--notrunclabels, as --sintax reads them).  vsg_sintax_stream is the --sintax command over a FASTA file: reader
 *      thread, vsg_sintax on every device of the group, rows in input order from a writer thread; the input number of
 *      the first record is 0.  random_ties (--sintax_random) is not offered: VSG_EINVAL, as is a cutoff outside 0..1.
 *      ---- */
#define VSG_SINTAX_BOOTSTRAPS 100
typedef struct vsg_sintax_opts {
  uint64_t seed;          /* --randseed; with --randseed 0 the caller draws a seed */
  int64_t query_number0;  /* input number of queries[q0]: query q0 + i uses substream query_number0 + i (vsg_sintax) */
  int32_t strand_both;    /* --strand both */
  int32_t random_ties;    /* --sintax_random: not offered, VSG_EINVAL */
  double cutoff;          /* --sintax_cutoff, 0..1 (rows only) */
} vsg_sintax_opts;
typedef struct vsg_sintax_result {
  int32_t strand;                           /* chosen strand: 0 plus, 1 minus (sintax.cpp:480-507) */
  int32_t nboot[2];                         /* successful bootstraps per strand */
  int32_t best_count[2];                    /* largest winning k-mer count per strand */
  int32_t seqno[2][VSG_SINTAX_BOOTSTRAPS];  /* winners per strand in bootstrap order, [0, nboot[s]); -1 beyond */
} vsg_sintax_result;
int vsg_sintax(vsg_ctx * ctx, const vsg_index * ix, const vsg_seqset * queries, int64_t q0, int64_t nq,
               const vsg_sintax_opts * opts, vsg_sintax_result * out);
int vsg_sintax_rows(const vsg_sintax_result * results, int64_t nq, const char * const * query_headers,
                    const char * const * target_headers, const vsg_sintax_opts * opts, char * buf, int64_t cap, int64_t * len);
int vsg_sintax_stream(vsg_group * g, const char * const * target_headers, const char * query_fasta,
                      const vsg_sintax_opts * opts, int batch_queries, const char * tabbedout_path, vsg_stream_stats * stats);

/* ---- read orientation: replaces the read loop of orient() (commands/orient.cpp:116-441) with unique_count
 *      (core/unique.cpp:155-353), rc_kmer (orient.cpp:90-113) and Dbindex::getmatchcount.  vsg_orient decides for every
 *      query of `queries` in [q0, q0 + nq), of any length, against an index made by vsg_index_create / vsg_udb_load: for
 *      each DISTINCT k-mer w of the query at the index's word length (windows with a symbol outside ACGTU skipped, and with
 *      a lower-case one iff query_mask_lower, i.e. --qmask other than none; the query is not DUST-masked), f = the
 *      number of database sequences holding w and r = that of its reverse complement; count_fwd counts the w with
 *      f > 8 r, count_rev those with r > 8 f.  strand 0 ('+') iff count_fwd >= 1 and count_fwd >= 4 count_rev, else
 *      1 ('-') iff count_rev >= 1 and count_rev >= 4 count_fwd, else 2 ('?').  out[i] belongs to query q0 + i.  The first
 *      call on an index builds its per-k-mer table of 4^k words in device memory (64 MiB at k = 12, 4 GiB at k = 15),
 *      kept until vsg_index_destroy.  Device time goes into vsg_profile.rank_ms.
 *      vsg_orient_stream is the --orient command over a FASTA or FASTQ file (the format from the first byte, '@' =
 *      FASTQ; gzip / bzip2 files are refused): reader thread, vsg_orient on every device of the group, writer thread, all
 *      outputs in input order.  fastaout / fastqout: '+' reads as read, '-' reads reverse-complemented (reverse_complement,
 *      FASTQ qualities reversed); notmatched: '?' reads as read, in the input's format; tabbedout: "label\t+|-|?\tfwd\trev".
 *      Labels are cut at the first blank unless notrunclabels; FASTA lines wrap at fasta_width (0: one line).  An output
 *      path may be NULL (that output is off); all four NULL, or fastqout with FASTA input, is VSG_EINVAL, as are a FASTQ
 *      record without its '@', a '+' line other than empty or the header, a file that ends inside a record and quality
 *      that is not as long as the sequence (the message names the record).  nstrand (optional, 3 entries): the
 *      reads oriented '+', '-' and '?'.  stats: `matched` counts the oriented reads, `rows` every read.  Header rewriting
 *      (--relabel*, --sizeout, --xsize, --xee, --xlength, --lengthout, --label_suffix, --sample) is left to the
 *      reference's writers. ---- */
typedef struct vsg_orient_result {
  int32_t strand;     /* 0 '+', 1 '-', 2 '?' */
  uint32_t count_fwd, count_rev;
} vsg_orient_result;
int vsg_orient(vsg_ctx * ctx, const vsg_index * ix, const vsg_seqset * queries, int64_t q0, int64_t nq,
               int query_mask_lower, vsg_orient_result * out);
int vsg_orient_stream(vsg_group * g, const char * query_path, int query_mask_lower, int notrunclabels, int fasta_width,
                      int batch_queries, const char * fastaout, const char * fastqout, const char * notmatched,
                      const char * tabbedout, vsg_stream_stats * stats, int64_t * nstrand);

/* ---- clustering commands: replaces cluster() (core/cluster.cpp:1140-1430), which --cluster_fast, --cluster_size,
 *      --cluster_smallmem and --cluster_unoise all run (commands/cluster_{fast,size,smallmem,unoise}.cpp), for --uc,
 *      --centroids and --clusters output.  vsg_cluster_command: the whole file read as db.read(..., upcase = 0) keeps it
 *      (FASTA or FASTQ, the format from the first byte, gzip / bzip2 refused, labels cut at the first blank unless
 *      notrunclabels, case kept), records outside [minseqlength, maxseqlength] and, for --cluster_unoise, of abundance
 *      below minsize discarded and counted.  The abundance is always read from ";size=" (1 without it; zero or out of
 *      range is an error, header_get_size) and orders the records, drives --sizeorder and the unoise rule; sizein only
 *      decides whether the C records and --sizeout sum abundances or count members.  Sort on the host by command
 *      (db.cpp:433-485): _FAST by length desc, abundance desc, label (strcmp) asc, input order; _SIZE and _UNOISE by
 *      abundance desc, label asc, input order; _SMALLMEM keeps the input order, which must be length-descending unless
 *      usersort.  Then on the device: the set made, masked (qmask dust: vsg_seqset_dust; soft: lower case out of the
 *      words; soft + hardmask: lower case turned into 'N' first), clustered by vsg_cluster_fast with round_size =
 *      threads (the results depend on it, as the reference's depend on --threads), target_sizes = the abundances and,
 *      for --self, target_labels = label identities (the caller leaves those pointer fields of `s` NULL), unoise set
 *      for _UNOISE; the CIGARs of the H records from two vsg_align_pairs calls (plus-strand members against the set,
 *      minus-strand ones from a vsg_seqset_revcomp set).  The printed sequences have the input's letters and the
 *      device's case (the DUST mask).  Then vsg_cluster_write.  Refused with VSG_EINVAL and no output file: compressed
 *      input, --qmask dust --hardmask, a word length outside 3..10, an unsorted _SMALLMEM input without usersort, and a
 *      pair the 16-bit aligner defers (its CIGAR cannot come from the fallback callback).  Not offered: --alnout,
 *      --samout, --userout, --blast6out, --matched, --notmatched, OTU tables,
 *      --relabel_sha1 / _md5 / _self, --label_suffix, --sample, several GPUs.  The reference's stderr summary is `stats`.
 *      (--msaout, --consout and --profile: vsg_cluster_command_outputs, below.)
 *      vsg_cluster_cmd_opts_default fills each command's CLI defaults (cli.cc): maxrejects 8 for --cluster_fast and 32
 *      otherwise, weak_id 0.90, minsize 8 and id -1 (not given) for --cluster_unoise, minseqlength 32, maxseqlength 50 000,
 *      wordlength 8, qmask dust, fasta_width 80; the caller sets id and whatever else the user gave.
 *      vsg_cluster_write needs no device: the output files of n records in processing (sorted) order — headers as kept,
 *      sequences as printed (cat / off / len), abundances, the vsg_cluster_result of each and the CIGAR of each H record
 *      (cigar_buf + cigar_off[i], NUL-terminated; ignored for S records).  --uc: S / H records in processing order
 *      (results_show_uc_one; "=" when matches == the alignment length without terminal gaps for _FAST, == the
 *      alignment length otherwise, results.cpp:84-95), then one C record per cluster; --centroids (fasta_print_general
 *      with --sizeout, --xsize, --relabel, --clusterout_id, fasta_width); --clusters: file <prefix><cluster number> per
 *      cluster.  C records, centroids and cluster files follow cluster number, or with clusterout_sort the cluster
 *      abundance descending first.  Any path may be NULL (no such output).  A failed write removes every file the call
 *      made.  *singletons (optional): clusters of abundance 1. ---- */
#define VSG_CLUSTER_FAST 0
#define VSG_CLUSTER_SIZE 1
#define VSG_CLUSTER_SMALLMEM 2
#define VSG_CLUSTER_UNOISE 3
typedef struct vsg_cluster_cmd_opts {
  int32_t command;          /* VSG_CLUSTER_FAST / _SIZE / _SMALLMEM / _UNOISE */
  int32_t threads;          /* --threads: the round size of vsg_cluster_fast */
  int32_t qmask;            /* --qmask: VSG_DBMASK_NONE / _SOFT / _DUST (default dust) */
  int32_t hardmask;         /* --hardmask (with qmask soft: lower case becomes 'N'; refused with dust) */
  int32_t usersort;         /* --usersort (_SMALLMEM: any input order) */
  int32_t notrunclabels;    /* --notrunclabels */
  int32_t sizein;           /* --sizein: C records and --sizeout sum the abundances instead of counting members */
  int32_t sizeout;          /* --sizeout */
  int32_t xsize;            /* --xsize: ";size=" stripped from printed labels */
  int32_t clusterout_id;    /* --clusterout_id: ";clusterid=" on the centroids */
  int32_t clusterout_sort;  /* --clusterout_sort */
  int32_t fasta_width;      /* --fasta_width (default 80; 0: one line) */
  int64_t minseqlength;     /* --minseqlength (default 32) */
  int64_t maxseqlength;     /* --maxseqlength (default 50 000) */
  int64_t minsize;          /* --minsize (_UNOISE only; default 8) */
  const char * relabel;     /* --relabel prefix of the centroids and cluster files, or NULL */
} vsg_cluster_cmd_opts;
typedef struct vsg_cluster_cmd_stats {
  int64_t sequences;        /* records kept */
  int64_t discarded_short, discarded_long, discarded_minsize;
  int64_t clusters, singletons, nucleotides;
  int64_t pairs, cells;     /* vsg_cluster_fast's work */
  double parse_s, sort_s, device_s, cigar_s, write_s, wall_s;
} vsg_cluster_cmd_stats;
void vsg_cluster_cmd_opts_default(int command, vsg_cluster_cmd_opts * c, vsg_search_opts * s);
int vsg_cluster_command(vsg_ctx * ctx, const char * input_path, const vsg_cluster_cmd_opts * c, const vsg_search_opts * s,
                        const char * uc, const char * centroids, const char * clusters_prefix, vsg_cluster_cmd_stats * stats);
int vsg_cluster_write(int64_t n, const char * const * headers, const char * cat, const int64_t * off, const int32_t * len,
                      const int64_t * abundances, const vsg_cluster_result * results, const char * cigar_buf,
                      const int64_t * cigar_off, const vsg_cluster_cmd_opts * c, const char * uc, const char * centroids,
                      const char * clusters_prefix, int64_t * singletons);

/* ---- cluster consensus: replaces msa() (core/msa.cpp) as cluster() calls it for --msaout, --consout and --profile
 *      (core/cluster.cpp:1473-1539).  vsg_cluster_msa takes the n records of `set` in processing order (the set as
 *      clustered and masked: vsg_cluster_command's, or the one given to vsg_cluster_fast or a cluster session), their
 *      vsg_cluster_result, their weights (the abundance with --sizein, else 1; at least 1) and the CIGAR of every H record
 *      (cigar_buf + cigar_off[i], NUL-terminated, as vsg_cluster_write takes them; the member, reverse-complemented on
 *      strand 1, against its centroid).  Per cluster, in cluster-number order, the rows are the centroid then the members
 *      in processing order.  insertions: the widths of the len(centroid) + 1 insertion blocks of every cluster, back to
 *      back (sum of len(centroid) + 1 entries; block p comes before centroid symbol p, the last after the centroid; its
 *      width is the longest D run at p, find_max_insertions_per_position).  col_first: nclusters + 1 entries, cluster c's
 *      columns are [col_first[c], col_first[c + 1]).  profile: 6 counters per column, A, C, G, T / U, N (every other IUPAC
 *      code), gap, each the sum of the weights of the rows with that symbol in the column (upper case, minus-strand rows
 *      complemented).  consensus: one char per column, the consensus row --msaout prints: '+' in the first insertions[0]
 *      and last insertions[len] columns of the cluster, else the best of A, C, G, T (a tie goes to the first), or N when
 *      none of them occurs and N does, if its count reaches the gaps, otherwise '-'.  *ncolumns receives the number of
 *      columns; above cap the call returns VSG_ECAP with insertions and col_first filled, profile and consensus untouched.
 *      The device work runs in chunks of whole clusters under a quarter of the context's direction-bit budget
 *      (VSG_DIR_BUDGET_MB), at most 1 GiB; a cluster that needs more runs alone.  With VSG_TRACE the kernel time (CUDA
 *      events) goes to stderr.
 *      vsg_cluster_msa_write needs no device: the files of msa() for records as vsg_cluster_write takes them, with the
 *      arrays of vsg_cluster_msa.  Clusters come in cluster-number order, with clusterout_sort by cluster abundance
 *      descending first.  --msaout: per cluster an empty line, the centroid row under ">*" + its header, each member row
 *      under its header (the record's own abundance for --sizeout; --relabel does not apply), ">consensus" and the
 *      consensus row; rows print the sequences as given, minus-strand rows reverse-complemented with the reference's
 *      complement map (case kept, U to A, anything else N); fasta_width applies.  --consout: the consensus without '+'
 *      and '-' under "centroid=" + the centroid's header (fasta_print_general with --relabel <prefix><cluster + 1>,
 *      ";seqs=<rows>", ";clusterid=" with clusterout_id, ";size=<cluster abundance>" with --sizeout).  --profile: that
 *      header line alone, then per column "column\tconsensus symbol\tA\tC\tG\tT\tgap\tN" and an empty line.  Any path
 *      may be NULL.  A failed write removes every file the call made. ---- */
int vsg_cluster_msa(vsg_ctx * ctx, const vsg_seqset * set, int64_t n, const vsg_cluster_result * results, const uint64_t * weights,
                    const char * cigar_buf, const int64_t * cigar_off, int32_t * insertions, int64_t * col_first, uint64_t * profile,
                    char * consensus, int64_t cap, int64_t * ncolumns);
int vsg_cluster_msa_write(int64_t n, const char * const * headers, const char * cat, const int64_t * off, const int32_t * len,
                          const int64_t * abundances, const vsg_cluster_result * results, const char * cigar_buf,
                          const int64_t * cigar_off, const int32_t * insertions, const int64_t * col_first, const uint64_t * profile,
                          const char * consensus, const vsg_cluster_cmd_opts * c, const char * msaout, const char * consout,
                          const char * profile_path);
/* vsg_cluster_command_outputs: vsg_cluster_command with every output it offers; any path may be NULL.  With msaout,
 *      consout or profile, after the CIGARs: vsg_cluster_msa (weights: the abundances with sizein, else 1) and
 *      vsg_cluster_msa_write.  A failed call leaves none of the files it made.  vsg_cluster_command is this call with the
 *      first three paths. */
typedef struct vsg_cluster_cmd_outputs {
  const char * uc, * centroids, * clusters_prefix, * msaout, * consout, * profile;
} vsg_cluster_cmd_outputs;
int vsg_cluster_command_outputs(vsg_ctx * ctx, const char * input_path, const vsg_cluster_cmd_opts * c, const vsg_search_opts * s,
                                const vsg_cluster_cmd_outputs * outputs, vsg_cluster_cmd_stats * stats);

/* ---- exact-match search: replaces Dbhash (core/dbhash.cpp) and search_exact_onequery / add_hit
 *      (commands/search_exact.cpp:136-209).  vsg_exact_index_create hashes every sequence of `db` on the device (the
 *      4-bit codes and the length, so case and U / T do not matter and N only equals N, as seqcmp compares) and keeps the
 *      (hash, sequence number) pairs sorted: 12 bytes per target.  `db` must outlive the index.  vsg_search_exact finds, for
 *      every query of `queries` in [q0, q0 + nq) and with strand_both also for its reverse complement, every database
 *      sequence identical to it: the candidates of equal hash are all compared symbol by symbol.  Each match becomes the
 *      hit add_hit makes (100 % identity, nwscore = query length * match score, no gaps, no trims) and passes the two
 *      accept functions with --id 1.0; the size / length / idprefix / idsuffix / self / selfid filters, query_sizes /
 *      target_sizes and query_labels / target_labels of opts apply as for vsg_search_hits.  opts->id, maxaccepts,
 *      maxrejects, wordlength and iddef are ignored: every identical target is reported.  The rows of query q0 + i are
 *      hits[first[i] .. first[i+1]) (first: nq + 1 offsets), at most maxhits of them (0: all), in search_joinhits order
 *      (target ascending; a palindrome's two hits on one target plus strand first).  *nhits receives the number of rows;
 *      above cap the call returns VSG_ECAP with first filled and hits untouched.
 *      VSG_EXACT_HASH_BITS (environment, read at index creation; unset = 64) keeps only the low bits of every hash, which
 *      forces collisions through the comparison (a test aid; results are the same). ---- */
typedef struct vsg_exact_index vsg_exact_index;
int vsg_exact_index_create(vsg_ctx * ctx, const vsg_seqset * db, vsg_exact_index ** out);
void vsg_exact_index_destroy(vsg_exact_index * ix);
int vsg_search_exact(vsg_ctx * ctx, const vsg_exact_index * ix, const vsg_seqset * queries, int64_t q0, int64_t nq,
                     const vsg_search_opts * opts, int64_t maxhits, vsg_search_result * hits, int64_t cap, int64_t * first,
                     int64_t * nhits);

/* ---- the --search_exact command: replaces search_exact() (commands/search_exact.cpp:211-908).  The database is read
 *      whole as db.read keeps it (FASTA or FASTQ, gzip / bzip2 and UDB files refused, labels cut at the first blank unless
 *      notrunclabels, records outside [minseqlength, maxseqlength] discarded and counted); with dbmask soft + hardmask
 *      its lower case becomes 'N'.  Queries (FASTA or FASTQ) stream in batches of batch_queries over a reader thread, the
 *      device (upload, soft + hardmask as 'N' on the host, vsg_search_exact with query_sizes from ";size=", --self label
 *      identities) and a writer thread that writes the rows in input order (the reference's order with --threads 1):
 *      --blast6out (at most maxhits rows per query, the "*" row with output_no_hits), --uc (H rows: the first hit, or
 *      every reported hit with uc_allhits; an N row for a query without a hit), --matched / --notmatched (the query as
 *      masked: with qmask dust, DUST on the device, masked symbols lower case and the rest upper case).  At the end:
 *      --dbmatched / --dbnotmatched (the database as masked by dbmask, DUST on the device; with sizeout the abundance is
 *      the query abundance summed over the accepted hits with sizein, the number of accepted hits without), and the OTU
 *      tables --otutabout / --mothur_shared_out (core/otutable.cpp: the query's sample from "sample=" / "barcodelabel=",
 *      else its leading [A-Za-z0-9_] run; the OTU from the first hit's "otu=", else its label up to the first ';'; "tax="
 *      gives the taxonomy column; the query abundance from ";size=" counts; unmatched targets are added with 0).
 *      DUST runs only when a file printing masked sequences asks for it; matching never depends on case.  Any output path
 *      may be NULL; a failed call leaves none of the files it made.  Refused with VSG_EINVAL and no file: no output, gzip
 *      or bzip2 input, a UDB database, qmask or dbmask dust with hardmask (the device DUST would upper-case the rest first),
 *      a missing file.  Not offered: --alnout, --samout, --userout, --fastapairs, --qsegout, --tsegout, --biomout, --lcaout,
 *      --relabel*, --label_suffix, --sample, --lengthout, --xee, several GPUs.  s carries strand_both and the filters of
 *      vsg_search_exact; its size and label arrays are the command's own (pass them NULL).
 *      vsg_search_exact_opts_default fills the CLI's defaults for --search_exact (cli.cc): dbmask and qmask dust,
 *      minseqlength 1, maxseqlength 50 000, fasta_width 80, maxhits 0 (all), batch_queries 65 536. ---- */
typedef struct vsg_search_exact_opts {
  int32_t dbmask;           /* --dbmask: VSG_DBMASK_NONE / _SOFT / _DUST (default dust) */
  int32_t qmask;            /* --qmask (default dust) */
  int32_t hardmask;         /* --hardmask (with soft: lower case becomes 'N'; refused with dust) */
  int32_t sizein;           /* --sizein: --dbmatched abundances sum the query abundances */
  int32_t sizeout;          /* --sizeout */
  int32_t xsize;            /* --xsize */
  int32_t notrunclabels;    /* --notrunclabels */
  int32_t fasta_width;      /* --fasta_width (default 80; 0: one line) */
  int64_t minseqlength;     /* --minseqlength (default 1) */
  int64_t maxseqlength;     /* --maxseqlength (default 50 000) */
  int64_t maxhits;          /* --maxhits (0: all) */
  int32_t uc_allhits;       /* --uc_allhits */
  int32_t output_no_hits;   /* --output_no_hits */
  int32_t batch_queries;    /* queries per device call (default 65 536) */
  int32_t reserved;
} vsg_search_exact_opts;
typedef struct vsg_search_exact_outputs {
  const char * blast6out, * uc, * matched, * notmatched, * dbmatched, * dbnotmatched, * otutabout, * mothur_shared_out;
} vsg_search_exact_outputs;
typedef struct vsg_search_exact_stats {
  int64_t queries, matched;                     /* "Matching unique query sequences: matched of queries" */
  int64_t queries_abundance, matched_abundance; /* "Matching total query sequences" (printed with --sizein) */
  int64_t db_sequences, db_discarded_short, db_discarded_long, hits;
  double parse_s, device_s, write_s, wall_s;
} vsg_search_exact_stats;
void vsg_search_exact_opts_default(vsg_search_exact_opts * e, vsg_search_opts * s);
int vsg_search_exact_command(vsg_ctx * ctx, const char * query_path, const char * db_path, const vsg_search_exact_opts * e,
                             const vsg_search_opts * s, const vsg_search_exact_outputs * outputs, vsg_search_exact_stats * stats);

/* ---- the --usearch_global command: replaces usearch_global() (commands/usearch_global.cpp:150-373, 537-845) on one
 *      context (one GPU).  The database: a UDB file (vsg_udb_detect) is read by vsg_udb_open / vsg_udb_load, its mask and
 *      word length are the file's, its headers and sequences are printed as stored; any other file is read whole as db.read
 *      keeps it (FASTA or FASTQ, labels cut at the first blank unless notrunclabels, records outside [minseqlength,
 *      maxseqlength] discarded and counted), with dbmask dust DUST-masked on the device, with soft + hardmask lower case
 *      turned into 'N', and indexed at s->wordlength with lower case out of the words unless dbmask is none.  Abundances
 *      come from ";size=".  Queries (FASTA or FASTQ) stream in batches of batch_queries over a reader thread, the device
 *      and a writer thread, rows in input order (the reference's order with --threads 1).  Per batch on the device: upload,
 *      qmask (dust: vsg_seqset_dust, the minus strand masked on its own; soft + hardmask: 'N' on the host), the search with
 *      every hit kept (vsg_search_hits with maxhits 0, query_sizes from ";size=", --self label identities), then the CIGAR
 *      of every --uc row that is printed and is not "=" (vsg_align_pairs: plus-strand rows against the searched query set,
 *      minus-strand rows against its vsg_seqset_revcomp).  The writer is vsg_search_write's.  A query whose only hits are
 *      weak (weak_id below id) is matched, as search_joinhits keeps it.  Refused with VSG_EINVAL and no file left: no
 *      output, gzip or bzip2 input, qmask or dbmask dust with hardmask, a missing file, negative maxhits, non-NULL size or
 *      label arrays in s, and a --uc row whose alignment the 16-bit aligner defers (its CIGAR cannot come from the
 *      fallback callback).  Not offered: --alnout, --samout, --userout, --fastapairs, --qsegout, --tsegout, --lcaout,
 *      --biomout, --relabel*, --label_suffix, --sample, several GPUs (vsg_usearch_stream is the multi-GPU --blast6out
 *      stream).  s carries id, weak_id, maxaccepts, maxrejects, wordlength, strand_both and the filters; its size and label
 *      arrays are the command's own (pass them NULL).  vsg_usearch_global_opts_default fills the CLI's defaults (cli.cc):
 *      dbmask and qmask dust, minseqlength 32, maxseqlength 50 000, fasta_width 80, maxhits 0 (all), batch_queries 65 536,
 *      and vsg_search_opts_default's (maxaccepts 1, maxrejects 32, wordlength 8); the caller sets id.
 *      vsg_search_write needs no device: the output files of nq queries (headers as kept, sequences as printed, i.e. as
 *      masked, abundances) with their search rows (query i's are rows[first[i] .. first[i + 1]), every hit, in
 *      search_joinhits order) against ndb database records (headers, sequences as printed, abundances).  cigar_off[j]
 *      (one per row) places row j's NUL-terminated CIGAR in cigar_buf; it is read only for a printed --uc row whose matches
 *      differ from its alignment length.  --blast6out: at most maxhits rows per query (the "*" row with output_no_hits);
 *      --uc: an H row for the first of them (every one with uc_allhits; column 2 the target number, column 3 the query
 *      length, "=" when matches == alignment length, terminal gaps included, else the CIGAR), an N row for a query without
 *      hits; top_hits_only stops both at the first row whose id is below the first row's.  --matched / --notmatched: the
 *      queries with / without a hit.  --otutabout / --mothur_shared_out: each query's first row's target (core/otutable.cpp,
 *      as for --search_exact), unmatched targets added with 0.  --dbmatched: the targets of any row, abundance the query
 *      abundances summed with sizein, the row count without; --dbnotmatched: the others with their own abundance.
 *      *matched (optional): the queries with a hit.  A failed write leaves no file. ---- */
typedef struct vsg_usearch_global_opts {
  int32_t dbmask;           /* --dbmask: VSG_DBMASK_NONE / _SOFT / _DUST (default dust); ignored for a UDB database */
  int32_t qmask;            /* --qmask (default dust) */
  int32_t hardmask;         /* --hardmask (with soft: lower case becomes 'N'; refused with dust) */
  int32_t sizein;           /* --sizein: --dbmatched abundances sum the query abundances */
  int32_t sizeout;          /* --sizeout */
  int32_t xsize;            /* --xsize */
  int32_t notrunclabels;    /* --notrunclabels */
  int32_t fasta_width;      /* --fasta_width (default 80; 0: one line) */
  int64_t minseqlength;     /* --minseqlength (default 32) */
  int64_t maxseqlength;     /* --maxseqlength (default 50 000) */
  int64_t maxhits;          /* --maxhits (0: all) */
  int32_t uc_allhits;       /* --uc_allhits */
  int32_t output_no_hits;   /* --output_no_hits */
  int32_t top_hits_only;    /* --top_hits_only */
  int32_t batch_queries;    /* queries per device call (default 65 536) */
} vsg_usearch_global_opts;
typedef vsg_search_exact_outputs vsg_usearch_global_outputs;
typedef struct vsg_usearch_global_stats {
  int64_t queries, matched;                     /* "Matching unique query sequences: matched of queries" */
  int64_t queries_abundance, matched_abundance; /* "Matching total query sequences" (printed with --sizein) */
  int64_t db_sequences, db_discarded_short, db_discarded_long, hits;
  int64_t pairs, cells;                         /* the search's alignments and their DP cells */
  double parse_s, device_s, cigar_s, write_s, wall_s;
} vsg_usearch_global_stats;
void vsg_usearch_global_opts_default(vsg_usearch_global_opts * u, vsg_search_opts * s);
int vsg_usearch_global_command(vsg_ctx * ctx, const char * query_path, const char * db_path, const vsg_usearch_global_opts * u,
                               const vsg_search_opts * s, const vsg_usearch_global_outputs * outputs, vsg_usearch_global_stats * stats);
int vsg_search_write(int64_t nq, const char * const * query_headers, const char * qcat, const int64_t * qoff, const int32_t * qlen,
                     const int64_t * query_sizes, const vsg_search_result * rows, const int64_t * first, const char * cigar_buf,
                     const int64_t * cigar_off, int64_t ndb, const char * const * db_headers, const char * dbcat,
                     const int64_t * dboff, const int32_t * dblen, const int64_t * db_sizes, const vsg_usearch_global_opts * u,
                     const vsg_usearch_global_outputs * outputs, int64_t * matched);

/* ---- Chimera detection: the --uchime_ref, --uchime_denovo, --uchime2_denovo and --uchime3_denovo commands
 *      (core/chimera.cpp), with the output files of `vsearch ... --threads 1`.  Each query of 4 nt or more is cut into
 *      four pieces that are searched on the device (--id 0.55, maxaccepts 4, maxrejects 16); the whole query is aligned
 *      with the accepted targets, the two parents are selected on the device, and the parents are evaluated on the host.
 *      --uchime_ref: the queries (input_path) are FASTA, read and printed as they are (never DUST-masked; with --qmask
 *      soft or dust their lower case is left out of the k-mer search); the database (db_path) is FASTA (dbmask none,
 *      soft or dust, --hardmask with soft) or UDB.
 *      De novo (db_path NULL): the input is FASTA or FASTQ, read as db.read keeps it, DUST-masked (--qmask dust) or
 *      hardmasked, sorted by abundance, and each sequence is searched against the non-chimeras before it, as the
 *      reference's single thread does.  The sorted input is cut into abundance bands of at most band_cap sequences, none
 *      of which can be a parent of another under --abskew; a band is searched on the device against the index as it
 *      stood at its start, then replayed on the host in order (a query whose candidates change is finished again on its
 *      own: stats.recomputed).  --abskew 1 or less gives bands of one sequence: exact, but one round trip per sequence.
 *      The abundance of a sequence comes from ";size=".
 *      Refused with VSG_EINVAL (message in vsg_last_error, no output file left behind): no output file, --uchime_ref
 *      without a database or de novo with one, gzip or bzip2 input, FASTQ queries for --uchime_ref, --strand both,
 *      --hardmask with --qmask dust or --dbmask dust, a missing file, a pair the 16-bit aligner defers (its CIGAR would
 *      come from nowhere).
 *      --chimeras_denovo (VSG_CHIMERAS_DENOVO, db_path NULL) is the de novo command for long, high-quality reads
 *      (find_best_parents_long / eval_parents_long): a query is cut into chimeras_parts parts (0: one per 100 nt, 2 to
 *      100), its parents are the candidates with the longest indel-free stretches that match within chimeras_diff_pct
 *      percent, up to chimeras_parents_max of them, each at least chimeras_length_min long, and the query is chimeric when
 *      two or more parents cover it completely.  Its defaults: --abskew 1.0, --alignwidth 60.  Its sorted input is cut
 *      into bands of band_cap consecutive reads; a band's earlier members are searched as parents of its later ones on
 *      the speculation that they are non-chimeric, and the serial pass finishes again a query whose candidates that
 *      changes (stats.recomputed).  The uchimeout slot takes
 *      its --tabbedout file (a row per chimera only) and the uchimealns slot its --alnout file; --borderline is refused.
 *      The four chimeras_* fields must keep their defaults for the other commands. ---- */
#define VSG_UCHIME_REF 0
#define VSG_UCHIME_DENOVO 1
#define VSG_UCHIME_2_DENOVO 2
#define VSG_UCHIME_3_DENOVO 3
#define VSG_CHIMERAS_DENOVO 4
typedef struct vsg_uchime_opts {   /* vsg_uchime_opts_default(command, &o) sets the CLI's defaults */
  int32_t command;                 /* VSG_UCHIME_REF / _DENOVO / _2_DENOVO / _3_DENOVO, VSG_CHIMERAS_DENOVO */
  double abskew, dn, xn, mindiv, minh;   /* --abskew 2.0 (16.0 for --uchime3_denovo, 1.0 for --chimeras_denovo; de novo only), --dn 1.4, --xn 8.0, --mindiv 0.8, --minh 0.28 */
  int32_t mindiffs;                /* --mindiffs 3 */
  int32_t qmask, dbmask, hardmask; /* VSG_DBMASK_*: --qmask dust, --dbmask dust (--uchime_ref only); --hardmask */
  int32_t self, selfid;            /* --uchime_ref: --self (label), --selfid (a piece equal to the target); always on de novo */
  int32_t strand_both;             /* --strand both: refused */
  int32_t sizeout, xsize, fasta_score, notrunclabels, uchimeout5;
  int32_t fasta_width, alignwidth; /* 80, 80 (60 for --chimeras_denovo); < 1: one line */
  int64_t minseqlength, maxseqlength;   /* records kept (the database's for --uchime_ref, the input's de novo): 1 .. 50 000 */
  int64_t batch_queries;           /* --uchime_ref: queries per device batch (< 1: 8 192) */
  int64_t band_cap;                /* de novo: the most sequences in an abundance band (< 1: 1 024) */
  int32_t chimeras_parts;          /* --chimeras_parts: 0 = (length + 99) / 100, clamped to 2 .. 100; else 2 .. 100 */
  int32_t chimeras_parents_max;    /* --chimeras_parents_max 3: 2 .. 20 */
  int32_t chimeras_length_min;     /* --chimeras_length_min 10: at least 1 */
  double chimeras_diff_pct;        /* --chimeras_diff_pct 0.0: 0 .. 50 */
} vsg_uchime_opts;
typedef struct vsg_uchime_outputs {   /* NULL: not written */
  const char * chimeras, * nonchimeras, * borderline, * uchimeout, * uchimealns;
} vsg_uchime_outputs;
typedef struct vsg_uchime_stats {
  int64_t queries, chimeras, nonchimeras, borderline;   /* the reference's stderr summary */
  int64_t queries_abundance, chimeras_abundance, nonchimeras_abundance, borderline_abundance;
  int64_t db_sequences;            /* --uchime_ref: database sequences */
  int64_t candidates;              /* whole-query alignments (distinct accepted targets of the pieces) */
  int64_t part_pairs;              /* alignments of the part searches */
  int64_t bands, recomputed;       /* de novo: abundance bands; queries the serial pass finished again */
  double parse_s, search_s, align_s, parents_s, eval_s, serial_s, write_s, wall_s;
} vsg_uchime_stats;
void vsg_uchime_opts_default(int command, vsg_uchime_opts * o);
int vsg_uchime_command(vsg_ctx * ctx, const char * input_path, const char * db_path, const vsg_uchime_opts * o,
                       const vsg_uchime_outputs * out, vsg_uchime_stats * st);

#ifdef __cplusplus
}
#endif
#endif /* VSG_H */
