// vsg_internal.h — shared between the CUDA translation units of libvsg.so (not installed).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <cstdio>
#include <memory>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/vsg.h"

namespace vsg {

// ---------------------------------------------------------------------------------------------
// Scoring as the kernels see it (built once per context from vsg_scoring; the 16-bit clamping and
// the "defer everything" flag follow core/align_simd.cpp:1264-1277, 1316-1373).
// ---------------------------------------------------------------------------------------------
enum { Q_L = 0, T_L = 1, Q_I = 2, T_I = 3, Q_R = 4, T_R = 5 };

struct ScoreParams {
  int16_t S[16][16];  // substitution matrix over 4-bit codes (align_simd.cpp:1319-1342)
  int16_t go[6];      // gap open   {q_l,t_l,q_i,t_i,q_r,t_r}
  int16_t ge[6];      // gap extend {q_l,t_l,q_i,t_i,q_r,t_r}
  int16_t match, mismatch;
  int16_t score_min;  // SHRT_MIN + max(0, all six open+extend) (align_simd.cpp:1432-1444)
  int16_t n_mismatch;
  int32_t fallback;   // a value did not fit a 16-bit cell: every pair is deferred
  int32_t shift;      // anti-diagonal shift c of a SHIFTED scoring (align_ckpt.cuh): S - 2c, ge + c; 0 = the caller's own
};

// One symbol per byte in HBM: bits 0-3 = 4-bit IUPAC code (utils/maps.cpp:75-118),
// bit 4 = lower case (soft-masked).  That is everything the aligner (code) and the k-mer
// sampler (code is a single base? lower case?) need from the ASCII byte.
struct DevSeqs {
  const uint8_t * sym;
  const int64_t * off;
  const int32_t * len;
  int64_t n;
};

// A unit of forward-DP work for one warp: one query against two targets, one per 16-bit half of
// every packed register (thi == tlo when the query has an odd number of targets; the duplicate
// half's output slot is -1).
struct FastTask {
  uint32_t q;
  uint32_t tlo, thi;
  int32_t out_lo, out_hi;  // pair slots (index into the per-batch stats array), -1 = discard
  int32_t dmax;            // max(dlen_lo, dlen_hi)
  uint64_t dir_off;        // byte offset of this task's direction block
  uint64_t bnd_off;        // element offset (uint2) of the strip-boundary row, if strips > 1
};

struct ExactTask {
  uint32_t q, t;
  int32_t out;
  int32_t pad;
  uint64_t dir_off;  // qlen*dlen bytes, row-major, one byte per cell
  uint64_t he_off;   // 2*qlen int16
};

// PairDesc::kind: where the pair's forward pass left what its traceback reads
enum { PD_FAST = 0, PD_EXACT = 1, PD_CKPT = 2 };

// What the traceback kernel needs to find a pair's direction bits.
struct PairDesc {
  uint32_t q, t;
  uint64_t dir_off;
  int32_t kind;   // PD_FAST = fast layout, PD_EXACT = exact layout, PD_CKPT = checkpoints (align_ckpt.cuh): dir_off / aux_off are uint2 element offsets
  int32_t out;    // pair slot in the stats array
  int32_t R;      // fast: rows per lane
  int32_t half;   // fast: 0 = low nibble, 1 = high nibble; checkpoints: bit 0 = half, bit 1 = general alphabet
  int32_t dmax;   // fast: steps per strip = dmax + 31
  uint64_t cigar_off;  // scratch region for the reversed CIGAR (qlen+dlen+2 bytes)
  uint64_t aux_off;    // checkpoints: element offset of the task's column checkpoints
};

struct Error {
  static void set(const std::string & m);
};

#define VSG_CUDA_OK(call)                                                                 \
  do {                                                                                    \
    cudaError_t e__ = (call);                                                             \
    if (e__ != cudaSuccess) {                                                             \
      vsg::Error::set(std::string(#call) + ": " + cudaGetErrorString(e__));               \
      return VSG_ECUDA;                                                                   \
    }                                                                                     \
  } while (0)

// growable device / pinned buffers
struct DevBuf {
  void * p = nullptr;
  size_t cap = 0;
  int reserve(size_t bytes);
  void release();
};
struct PinBuf {
  void * p = nullptr;
  size_t cap = 0;
  int reserve(size_t bytes);
  void release();
};

void count_launch(int n = 1);

// ---------------------------------------------------------------------------------------------
// The k-mer ranker and its indexes (rank.cu)
// ---------------------------------------------------------------------------------------------
// the most candidates per query the ranker keeps in shared memory; longer lists go through rank_lists
constexpr int RANK_TOPHITS_MAX = 1024;

// The bounded ranker's results on the device, in ctx->rank_tmp: query i's candidates are seqno / count[i * tophits ...],
// n[i] of them, best first; status != 0 when a query was too long to rank.
struct RankTop {
  uint32_t * seqno;
  uint32_t * count;
  int32_t * n;
  int32_t * status;
};

const vsg_seqset * index_db(const vsg_index * ix);
int index_wordlength(const vsg_index * ix);
// the index's shards on its device (rank_steps.cuh)
struct ShardDev;
const ShardDev * index_shards(const vsg_index * ix, int & nshards);
// *out = the index's 4^k-word table on its device: per k-mer, the number of targets holding it (Dbindex::getmatchcount);
// built from the shards with c's stream on the first call and kept until vsg_index_destroy
int index_word_counts(vsg_ctx * c, const vsg_index * ix, const uint32_t ** out);

// What the ranker ranks against: a shard table on the device, the targets' lengths (only lens.len is read) and the
// query-side masking.  incr: the cluster driver's incremental index (rank_kernel<true, MODE>), whose candidates are
// dense target numbers.  timed: launches go into vsg_profile.rank_ms (the static index; the cluster ranker is untimed).
struct RankTargets {
  const ShardDev * shards = nullptr;
  int nshards = 0;
  DevSeqs lens{};
  int k = 0, mask_lower = 0, device = 0;
  bool incr = false, timed = false;
};
// the static index's targets, ranked with the query-side masking mask_lower
RankTargets index_targets(const vsg_index * ix, int mask_lower);
// enqueues the ranker over queries [q0, q0 + nq) on c's stream, timed into vsg_profile.rank_ms
int rank_enqueue(vsg_ctx * c, const vsg_index * ix, const vsg_seqset * queries, int64_t q0, int64_t nq,
                 int minwordmatches, int tophits, int mask_lower, RankTop & out);
// copies the results of rank_enqueue / cindex_rank_enqueue to the host, waits for them and checks their status
int rank_download(vsg_ctx * c, const RankTop & r, int64_t nq, int tophits, uint32_t * h_seqno, uint32_t * h_count,
                  int32_t * h_n, const char * caller);
// unbounded ranker (any tophits): query i's list is seqno / count[first[i] .. first[i + 1])
int rank_lists(vsg_ctx * c, const RankTargets & t, const vsg_seqset * queries, int64_t q0, int64_t nq, int minwordmatches,
               int64_t tophits, std::vector<int64_t> & first, std::vector<uint32_t> & seqno, std::vector<uint32_t> & count);
// n[i] = how many targets query q0 + i has at or above the reference's threshold
int rank_counts(vsg_ctx * c, const RankTargets & t, const vsg_seqset * queries, int64_t q0, int64_t nq, int minwordmatches,
                std::vector<int32_t> & n);

// the cluster driver's incremental index of the centroids; candidates are DENSE target numbers (cindex_seqnos maps
// them to sequence numbers)
struct CIndex;
int cindex_create(vsg_ctx * c, const vsg_seqset * set, int wordlength, int mask_lower, CIndex ** out);
void cindex_destroy(CIndex * ix);
int cindex_append(vsg_ctx * c, CIndex * ix, const uint32_t * seqnos, int n);
int cindex_rank_enqueue(vsg_ctx * c, CIndex * ix, const vsg_seqset * queries, int64_t q0, int64_t nq, int minwordmatches,
                        int tophits, RankTop & out);
// rank_lists against the centroids indexed so far (tophits above RANK_TOPHITS_MAX); candidates are dense numbers
int cindex_rank_lists(vsg_ctx * c, CIndex * ix, const vsg_seqset * queries, int64_t q0, int64_t nq, int minwordmatches,
                      int64_t tophits, std::vector<int64_t> & first, std::vector<uint32_t> & seqno, std::vector<uint32_t> & count);
const std::vector<uint32_t> & cindex_seqnos(const CIndex * ix);

// vsg_align_pairs with traceback on demand (align_ckpt.cuh, TbGate): leader_of[k] = index of pair k's group leader in
// this call, or -1; threshold = 100 * --id (+ margin); skipped pairs return aligned = matches = mismatches = 0xffff.
// ck_counts (optional, 3 entries): checkpoint tasks stored, score-only, re-run with stores
int align_pairs_gated(vsg_ctx * c, const vsg_seqset * queries, const vsg_seqset * targets,
                      int64_t npairs, const uint32_t * qidx, const uint32_t * tidx,
                      int16_t * score, uint16_t * aligned, uint16_t * matches,
                      uint16_t * mismatches, uint16_t * gaps, int32_t * trims,
                      char * cigar_buf, int64_t cigar_cap, int64_t * cigar_off,
                      const int32_t * leader_of, double gate_threshold, int gate_iddef, int64_t * ck_counts = nullptr);

// vsg_search_hits with the rows kept on the host: query i's are rows[first[i] .. first[i + 1]) (search.cu)
int search_hits_host(vsg_ctx * c, const vsg_index * ix, const vsg_seqset * db, const vsg_seqset * queries, int64_t q0,
                     int64_t nq, const vsg_search_opts * opts, int64_t maxhits, std::vector<vsg_search_result> & rows,
                     std::vector<int64_t> & first, int64_t * work);
// vsg_group_search_hits with the rows kept on the host (group.cu)
int group_search_rows(vsg_group * g, const char * qcat, const int64_t * qoff, const int32_t * qlen, int64_t nq, int dust_queries,
                      const vsg_search_opts * opts, int64_t maxhits, std::vector<vsg_search_result> & rows,
                      std::vector<int64_t> & first, int64_t * work);
// vsg_sintax of host queries sharded over the group's devices; query i gets input number opts->query_number0 + i
int group_sintax(vsg_group * g, const char * qcat, const int64_t * qoff, const int32_t * qlen, int64_t nq,
                 const vsg_sintax_opts * opts, vsg_sintax_result * out);
// vsg_orient of host queries sharded over the group's devices (group.cu)
int group_orient(vsg_group * g, const char * qcat, const int64_t * qoff, const int32_t * qlen, int64_t nq, int query_mask_lower,
                 vsg_orient_result * out);
// VSG_EINVAL (message prefixed with caller) for --sintax_random or a cutoff outside 0..1 (sintax.cu)
int sintax_check_opts(const vsg_sintax_opts * o, const char * caller);
// the --tabbedout rows of vsg_sintax_rows, appended to `out` (sintax.cu)
int sintax_rows_string(const vsg_sintax_result * res, int64_t nq, const char * const * qheads, const char * const * theads,
                       const vsg_sintax_opts * opts, std::string & out);
// rows / first to the caller's buffers of vsg_search_hits / vsg_group_search_hits: *nhits = rows needed, VSG_ECAP
// (first filled, hits untouched) when they exceed cap
int hits_out(const std::vector<vsg_search_result> & rows, const std::vector<int64_t> & first, const char * caller,
             vsg_search_result * hits, int64_t cap, int64_t * first_out, int64_t * nhits);

// VSG_EINVAL (message prefixed with caller) for a word length outside 3..15 or an unknown dbmask (makeudb.cu)
int makeudb_check_opts(const vsg_makeudb_opts * o, const char * caller);

// every record of a FASTA or FASTQ file as db.read keeps it (stream.cu): the format from the first byte, gzip and bzip2
// refused, core/fasta.cpp's symbol rules, labels cut at the first blank unless notrunclabels, records outside
// [minlen, maxlen] discarded and counted (minlen < 1: no lower bound).  Errors are VSG_EINVAL, prefixed with caller.
struct FastxFile {
  std::vector<char> cat;             // sequences back to back, as read (case kept), then a NUL
  std::vector<int64_t> off;
  std::vector<int32_t> len;
  std::vector<std::string> head;
  int64_t stripped = 0, discarded_short = 0, discarded_long = 0;
};
int read_fastx_file(const char * caller, const char * path, bool notrunclabels, int64_t minlen, int64_t maxlen, FastxFile & out);
// The reference's label and FASTA writers as the commands use them (cluster_cmd.cu).
// header_find_attribute: the first "(^|;)size=[0-9]+(;|$)" of the label; [start, end) covers "size=<digits>"
bool find_size(const std::string & h, int & start, int & end);
// fastx_get_abundance / header_get_size: 1 without an annotation; zero or out of range is an error (false, err set)
bool abundance_of(const std::string & h, int64_t & out, std::string & err);
// header_fprint_strip with only --xsize among the stripped attributes; returns whether the last character written is ';'
bool header_fprint_strip(std::string & out, const std::string & h, bool strip_size);
// fasta_print_general with the options the commands offer: --relabel prefix (used when ordinal > 0, NULL: none),
// --xsize, --sizeout (";size=" when abundance > 0), ";clusterid=" (clusterid >= 0), fasta_width (< 1: one line)
struct FastaFormat {
  const char * relabel;
  bool xsize, sizeout;
  int fasta_width;
};
// prefix: text before the label (NULL: none); seqs > 0: ";seqs=" (before ";clusterid="); seq NULL: no sequence line
void fasta_print_general(std::string & out, const FastaFormat & f, const std::string & head, const char * seq, int64_t len,
                         int64_t abundance, int64_t ordinal, int64_t clusterid, const char * prefix = nullptr, int64_t seqs = 0);
// reverse_complement (utils/reverse_complement.cpp) with the reference's complement map (utils/maps.cpp): IUPAC codes
// to their complements in the same case, U to A, anything else to N
struct Complement {
  char map[256];
  Complement()
  {
    for (char & m : map) { m = 'N'; }
    char const * const from = "ACGTURYKMBVDHSWNacgturykmbvdhswn";
    char const * const to = "TGCAAYRMKVBHDSWNtgcaayrmkvbhdswn";
    for (int i = 0; from[i] != '\0'; i++) { map[static_cast<unsigned char>(from[i])] = to[i]; }
  }
};
// the files a call creates, removed again unless the call succeeds
struct OutFiles {
  std::vector<std::string> made;
  bool ok = false;
  ~OutFiles() { if (!ok) { for (auto const & p : made) { std::remove(p.c_str()); } } }
  // opens path for writing, to be removed again unless the call succeeds; NULL when it cannot be opened
  std::FILE * open(const std::string & path)
  {
    std::FILE * f = std::fopen(path.c_str(), "wb");
    if (f != nullptr) { made.push_back(path); }
    return f;
  }
  bool write(const std::string & path, const std::string & data)
  {
    std::FILE * f = std::fopen(path.c_str(), "wb");
    if (f == nullptr) { return false; }
    made.push_back(path);
    bool const good = std::fwrite(data.data(), 1, data.size(), f) == data.size();
    return std::fclose(f) == 0 && good;
  }
};
// results_show_blast6out_one (core/results.cpp:221-271): the --blast6out rows of one query's n hits, or with n == 0 and
// output_no_hits its "*" row; returns the rows written (stream.cu)
int64_t blast6_rows(std::string & out, const std::string & qhead, const vsg_search_result * r, int64_t n,
                    const char * const * target_labels, bool output_no_hits);

// vsg_search_exact with the rows kept on the host: query i's are rows[first[i] .. first[i + 1]) (exact.cu)
int search_exact_host(vsg_ctx * c, const vsg_exact_index * ix, const vsg_seqset * queries, int64_t q0, int64_t nq,
                      const vsg_search_opts * opts, int64_t maxhits, std::vector<vsg_search_result> & rows,
                      std::vector<int64_t> & first);

// owning handle of a sequence set
struct SeqsetDeleter { void operator()(vsg_seqset * s) const { vsg_seqset_destroy(s); } };
using SeqsetPtr = std::unique_ptr<vsg_seqset, SeqsetDeleter>;

// the reverse complements of src's sequences [q0, q0 + n), as a compact set
int seqset_revcomp(vsg_ctx * c, const vsg_seqset * src, int64_t q0, int64_t n, SeqsetPtr & out);
// both strands of every sequence of src, sequence s at 2s and its reverse complement at 2s+1
int seqset_both_strands(vsg_ctx * c, const vsg_seqset * src, SeqsetPtr & out);

// ---- what the search commands share (search_out.cu) ----
// DUST on the device, then the printed sequences `cat` (the set's, plus a NUL) take the device's case: dust_core
// upper-cases, then lowers the masked symbols; the letters stay the input's
int dust_case(vsg_ctx * ctx, vsg_seqset * set, std::vector<char> & cat);
// --hardmask with --qmask / --dbmask soft (hardmask / hardmask_all, core/mask.cpp): lower case becomes 'N'
void hardmask(std::vector<char> & cat);
// A search command's database: the records as printed (file), their abundances from ";size=", the header pointers, the
// device set as searched and, for --self, label identities (label_id[t] = the first record with t's header).
struct SearchDb {
  FastxFile file;
  std::vector<int64_t> size;
  std::vector<const char *> heads;
  SeqsetPtr set;
  std::vector<int64_t> label_id;
  std::unordered_map<std::string, int64_t> label_ids;
};
// size, heads and (self) the label identities of db.file's records
int search_db_labels(const char * caller, bool self, SearchDb & db);
// db.read(..., upcase = 0) under [minlen, maxlen], lower case to 'N' for dbmask soft + hardmask, search_db_labels, the
// device set, and with `dust` DUST on the device with the printed case (dust_case)
int search_db_read(vsg_ctx * ctx, const char * caller, const char * path, bool notrunclabels, int64_t minlen, int64_t maxlen,
                   int dbmask, bool hardmask_soft, bool dust, bool self, SearchDb & db);
// o = s with a batch's query abundances (from heads' ";size="), the database's, and for --self the queries' label identities
int search_batch_opts(const char * caller, const std::vector<std::string> & heads, const SearchDb & db, const vsg_search_opts & s,
                      std::vector<int64_t> & size, std::vector<int64_t> & label, vsg_search_opts & o);

// The output files of a search command (search_output_results and the end of usearch_global / search_exact): fed
// batches of queries with their rows in input order (batch), then the end-of-run files (finish).  Where the two commands
// differ is a parameter.
struct SearchWriterOpts {
  int64_t maxhits = 0;            // 0: all
  bool top_hits_only = false, uc_allhits = false, output_no_hits = false, sizein = false, xsize = false;
  bool weak_dbmatched = false;    // a weak hit marks its target too (usearch_global.cpp:368-372; search_exact: accepted only)
  bool dbnotmatched_size = false; // --dbnotmatched prints the target's abundance (usearch_global.cpp:828), not 0 (search_exact)
  FastaFormat fmt{nullptr, false, false, 80};
};
SearchWriterOpts usearch_global_writer_opts(const vsg_usearch_global_opts & u);
// one batch: query i's rows are rows[first[i] .. first[i + 1]); a printed --uc row j that is not "=" reads its CIGAR at
// cigar_buf + cigar_off[j]
struct SearchRows {
  int64_t nq;
  const std::string * head;
  const char * cat;
  const int64_t * off;
  const int32_t * len;
  const int64_t * size;
  const vsg_search_result * rows;
  const int64_t * first;
  const char * cigar_buf;
  const int64_t * cigar_off;
};
struct OtuTable;
class SearchWriter {
 public:
  SearchWriter(const SearchWriterOpts & o, const vsg_search_exact_outputs & out, const std::vector<std::string> & dbhead,
               const char * dbcat, const int64_t * dboff, const int32_t * dblen, const int64_t * dbsize);
  ~SearchWriter();
  // the rows of a query's n hits that --blast6out / --uc show: min(maxhits, n), cut by --top_hits_only
  int64_t shown(const vsg_search_result * r, int64_t n) const;
  // of those, the rows --uc prints
  int64_t uc_rows(int64_t shown) const;
  // appends the batch's rows to outs[0..3] = blast6out, uc, matched, notmatched, and accumulates the rest
  void batch(const SearchRows & b, std::string * outs);
  // --otutabout, --mothur_shared_out, --dbmatched, --dbnotmatched through files; false (error set) on a failed write
  bool finish(const char * caller, OutFiles & files);
  int64_t queries = 0, matched = 0, queries_abundance = 0, matched_abundance = 0, hits = 0, blast6 = 0;
 private:
  const char * const * dbhead_ptrs();
  SearchWriterOpts o_;
  vsg_search_exact_outputs out_;
  const std::vector<std::string> & dbhead_;
  const char * dbcat_;
  const int64_t * dboff_;
  const int32_t * dblen_;
  const int64_t * dbsize_;
  std::vector<uint64_t> dbmatched_;
  std::vector<const char *> dbheads_;
  std::unique_ptr<OtuTable> otu_;
};

// The CIGARs of pairs (q[j], t[j]) on strand[j], two vsg_align_pairs calls: plus-strand pairs align queries' q against
// targets' t, minus-strand pairs the reverse complement of queries' q (vsg_seqset_revcomp of the whole set).  Pair j's
// NUL-terminated CIGAR is appended to buf at offs[j]; deferred = the first pair the 16-bit aligner defers
// (VSG_SCORE_SENTINEL; its offs stays -1), or -1.
int strand_cigars(vsg_ctx * c, const vsg_seqset * queries, const vsg_seqset * targets, const std::vector<uint32_t> & q,
                  const std::vector<uint32_t> & t, const std::vector<uint8_t> & strand, std::vector<char> & buf,
                  std::vector<int64_t> & offs, int64_t & deferred);

}  // namespace vsg

struct vsg_seqset {
  vsg::DevSeqs d{};
  std::vector<int32_t> h_len;       // host copy of lengths
  std::vector<int64_t> h_off;       // host copy of offsets
  std::vector<uint8_t> h_nonacgt;   // 1 if the sequence holds a symbol outside ACGTU
  vsg::DevBuf b_sym, b_off, b_len;
  int device = 0;
  int64_t total = 0;
};

// a UDB database in host memory: read from a file (vsg_udb_open, udb.cu) or made from sequences (vsg_udb_make, makeudb.cu)
struct vsg_udb {
  vsg_udb_info info{};
  std::vector<uint32_t> kmercount;   // 4^k
  std::vector<uint32_t> kmerindex;   // info.index_entries
  std::vector<char> headers;         // header block (NUL-terminated strings)
  std::vector<uint32_t> header_off;  // seqcount + 1
  std::vector<char> cat;             // sequences back to back, one NUL at the very end
  std::vector<int64_t> off;
  std::vector<int32_t> len;
};

struct vsg_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  vsg_scoring scoring{};
  vsg::ScoreParams sp{};
  vsg::ScoreParams sp2{};      // the shifted scoring the checkpoint kernels run with (align_ckpt.cuh)
  bool ckpt_enabled = true;    // false when the shifted scoring does not fit (shifted_params): direction-bit kernels only
  bool fast_disabled = false;  // VSG_DISABLE_FAST=1 (tests force the exact kernel)
  // scratch
  vsg::DevBuf dir, bnd, he, cigar_scratch, cigar_dense, stats, tasks_fast, tasks_exact, pairs,
      cigar_len, cigar_offs, cub_tmp, rank_tmp, rank_scratch, pre_flags, gate, rerun_count;
  vsg::PinBuf h_tasks, h_stats;
  size_t dir_budget = (size_t)64 << 30;
  cudaEvent_t ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  // cumulative profile since the last vsg_profile_reset (kernel times from cudaEvents on `stream`)
  int64_t prof_cells = 0, prof_fast = 0, prof_exact = 0, prof_fwd_launches = 0, prof_tb_skipped = 0, prof_tb_redone = 0;
  float prof_fwd_ms = 0.f, prof_tb_ms = 0.f, prof_rank_ms = 0.f;
  bool rank_pending = false;
  std::vector<cudaEvent_t> ev_pool;  // 3 per chunk of an align call
  vsg_fallback_fn fallback = nullptr;  // host-side aligner for SHRT_MAX pairs
  void * fallback_user = nullptr;
  std::vector<vsg_ctx *> children;  // per-host-thread contexts of vsg_search_batch
  std::shared_ptr<void> search_scratch;  // host buffers of vsg_search_batch's driver, kept between calls
};
