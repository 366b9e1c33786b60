/* oracle/sintax_shim.cpp — TEST INFRASTRUCTURE ONLY.
 *
 * A C-ABI window (for ctypes) onto the UNMODIFIED reference's SINTAX bootstraps, linked against the reference objects
 * that oracle/Makefile compiles into oracle/_ref/libvsearch_ref.a (oracle/sintax.mk builds
 * oracle/_ref/libvsref_sintax.so).  It calls the reference's own
 *   Database::add / Dbindex::prepare / add_all_sequences  (src/core/db.hpp, src/core/dbindex.hpp)
 *   unique_count(..., Masking::none)                      (src/core/unique.hpp)
 *   reverse_complement                                    (src/utils/reverse_complement.hpp)
 *   SplitMix64, random_substream_seed, random_bounded     (src/utils/random.hpp)
 *   sintax_search_topscores                               (src/commands/sintax.cpp:299, non-static, declared here)
 * and repeats only the loop of sintax_query that strings them together (commands/sintax.cpp:405-507), so that the
 * per-bootstrap winners of the device path can be pinned against the reference's own counting and tie breaking.
 */
#include "vsearch_api.h"
#include "core/searchcore.hpp"
#include "core/search_internal.hpp"
#include "core/minheap.hpp"
#include "core/unique.hpp"
#include "utils/random.hpp"
#include "utils/reverse_complement.hpp"

#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

auto sintax_search_topscores(struct searchinfo_s * searchinfo, SplitMix64 & rng, struct Parameters const & parameters) -> void;

namespace {

constexpr int subset_size = 32;
constexpr int bootstrap_count = 100;

struct SintaxDb {
  Parameters params;
  Database db;
  Dbindex dbindex;
};

}  // namespace

extern "C" {

/* the database as --sintax builds it from a FASTA file: sequences in the order given (the caller drops those under
   32 nt, as db.read does), the index at `wordlength`, lower case excluded iff mask_lower (--dbmask dust / soft) */
void * vsref_sintax_db_create(int n, const char * cat, const int64_t * off, const int * len, int wordlength, int mask_lower)
{
  SintaxDb * r = new SintaxDb();
  Parameters & p = r->params;
  p.opt_wordlength = wordlength;
  p.opt_threads = 1;
  p.opt_dbmask = mask_lower != 0 ? Masking::dust : Masking::none;
  r->db.init();
  for (int i = 0; i < n; i++) {
    std::string const head = "t" + std::to_string(i);
    std::string const seq(cat + off[i], static_cast<size_t>(len[i]));
    r->db.add(false, head.c_str(), seq.c_str(), nullptr, head.size(), seq.size(), 1);
  }
  r->dbindex.prepare(1, p.opt_dbmask, r->db, p);
  r->dbindex.add_all_sequences(p.opt_dbmask, r->db, p);
  return r;
}

void vsref_sintax_db_free(void * h)
{
  SintaxDb * r = static_cast<SintaxDb *>(h);
  r->dbindex.clear();
  r->db.clear();
  delete r;
}

/* the bootstraps of one query with input number query_number under base seed `seed`, laid out as vsg_sintax_result:
   out[0] = strand, out[1..2] = successful bootstraps per strand, out[3..4] = largest winning count per strand,
   out[5 + 100 * s + i] = winner i of strand s (-1 beyond the successful ones) */
void vsref_sintax(void * h, const char * query, int len, int64_t query_number, uint64_t seed, int strand_both, int32_t * out)
{
  SintaxDb * r = static_cast<SintaxDb *>(h);
  int const seqcount = static_cast<int>(r->db.getsequencecount());
  SplitMix64 rng(random_substream_seed(seed, static_cast<uint64_t>(query_number)));
  int boot_count[2] = {0, 0};
  unsigned int best_count[2] = {0, 0};
  for (int i = 0; i < 5 + 2 * bootstrap_count; i++) { out[i] = i < 5 ? 0 : -1; }
  std::vector<char> seq(static_cast<size_t>(len) + 1, 0);
  for (int s = 0; s < (strand_both != 0 ? 2 : 1); s++) {
    if (s == 0) { std::memcpy(seq.data(), query, static_cast<size_t>(len)); }
    else { reverse_complement(seq.data(), query, len); }
    searchinfo_s si;
    search_thread_init(&si, seqcount, 1, r->params, r->dbindex, r->db);
    unsigned int kmersamplecount = 0;
    unsigned int const * kmersample = nullptr;
    unique_count(si.uh, static_cast<int>(r->dbindex.wordlength), len, seq.data(), &kmersamplecount, &kmersample, Masking::none);
    if (kmersamplecount >= subset_size) {
      std::vector<unsigned char> drawn(kmersamplecount);
      for (int b = 0; b < bootstrap_count; b++) {
        unsigned int subset[subset_size];
        int subsamples = 0;
        std::fill(drawn.begin(), drawn.end(), 0);
        for (int j = 0; j < subset_size; j++) {
          uint64_t const x = random_bounded(rng, kmersamplecount);
          if (drawn[x] == 0) { subset[subsamples++] = kmersample[x]; drawn[x] = 1; }
        }
        si.kmersamplecount = static_cast<unsigned int>(subsamples);
        si.kmersample = subset;
        sintax_search_topscores(&si, rng, r->params);
        if (!minheap_isempty(si.m)) {
          elem_t const e = minheap_poplast(si.m);
          out[5 + bootstrap_count * s + boot_count[s]++] = static_cast<int32_t>(e.seqno);
          if (e.count > best_count[s]) { best_count[s] = e.count; }
        }
      }
    }
    si.kmersample = nullptr;
    search_thread_exit(&si);
  }
  int strand = 0;
  if (strand_both != 0) {
    if (best_count[1] > best_count[0]) { strand = 1; }
    else if (best_count[1] == best_count[0] && boot_count[1] > boot_count[0]) { strand = 1; }
  }
  out[0] = strand;
  out[1] = boot_count[0]; out[2] = boot_count[1];
  out[3] = static_cast<int32_t>(best_count[0]); out[4] = static_cast<int32_t>(best_count[1]);
}

}  // extern "C"
