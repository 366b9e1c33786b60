// search_out.cu — what the search commands (--search_exact, --usearch_global) share around the device search: the
// database as they read, mask and print it, the per-query options of a batch, the writer of their output files, and
// the by-strand CIGAR step that --usearch_global and the clustering commands run for their --uc rows.
//
// Replaces, host side,
//   db.read / dust_all / hardmask_all               (core/db.cpp, core/mask.cpp)             search_db_read
//   search_output_results, the end of usearch_global (commands/usearch_global.cpp:150-373, 760-845) and of
//   search_exact (commands/search_exact.cpp:211-424, 800-890), otutable_* (core/otutable.cpp:178-392)
//                                                                                              SearchWriter, vsg_search_write
#include "vsg_internal.h"

#include <algorithm>
#include <climits>
#include <cstdio>
#include <cstring>
#include <map>
#include <set>
#include <string>
#include <vector>

using namespace vsg;

namespace {

// "(^|;)<name>=([^;]*)($|;)" as regexec finds it: the leftmost, at h[at] (the name's first character); the value is
// h[start, start + len)
bool find_attribute(const std::string & h, const char * name, size_t & at, size_t & start, size_t & len)
{
  size_t const nl = std::strlen(name);
  for (size_t p = 0; p + nl < h.size(); p++) {
    if ((p == 0 || h[p - 1] == ';') && h.compare(p, nl, name) == 0 && h[p + nl] == '=') {
      at = p;
      start = p + nl + 1;
      size_t const e = h.find(';', start);
      len = (e == std::string::npos ? h.size() : e) - start;
      return true;
    }
  }
  return false;
}

}  // namespace

// otutable_add / otutable_print_otutabout / otutable_print_mothur_shared_out (core/otutable.cpp:178-392)
struct vsg::OtuTable {
  std::set<std::string> otus, samples;
  std::map<std::pair<std::string, std::string>, uint64_t> count;   // (otu, sample)
  std::map<std::string, std::string> tax;

  void add(const std::string * query, const std::string * target, int64_t abundance)
  {
    std::string sample, otu;
    if (query != nullptr) {
      size_t p = 0, s = 0, l = 0, p2 = 0, s2 = 0, l2 = 0;
      bool const a = find_attribute(*query, "sample", p, s, l), b = find_attribute(*query, "barcodelabel", p2, s2, l2);
      if (a || b) {
        if (!a || (b && p2 < p)) { s = s2; l = l2; }   // the leftmost of the two
        sample = query->substr(s, l);
      } else {
        sample = query->substr(0, std::strspn(query->c_str(), "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz_0123456789"));
      }
      samples.insert(sample);
    }
    if (target != nullptr) {
      size_t p = 0, s = 0, l = 0;
      otu = find_attribute(*target, "otu", p, s, l) ? target->substr(s, l) : target->substr(0, std::strcspn(target->c_str(), ";"));
      if (find_attribute(*target, "tax", p, s, l)) { tax[otu] = target->substr(s, l); }
      otus.insert(otu);
    }
    if (query != nullptr && target != nullptr && abundance != 0) { count[{otu, sample}] += static_cast<uint64_t>(abundance); }
  }
  std::string otutabout() const
  {
    std::string out = "#OTU ID";
    for (auto const & s : samples) { out += '\t'; out += s; }
    if (!tax.empty()) { out += "\ttaxonomy"; }
    out += '\n';
    for (auto const & o : otus) {
      out += o;
      for (auto const & s : samples) {
        auto const it = count.find({o, s});
        out += '\t'; out += std::to_string(it == count.end() ? 0 : it->second);
      }
      if (!tax.empty()) {
        out += '\t';
        auto const it = tax.find(o);
        if (it != tax.end()) { out += it->second; }
      }
      out += '\n';
    }
    return out;
  }
  std::string mothur_shared_out() const
  {
    std::string out = "label\tGroup\tnumOtus";
    for (auto const & o : otus) { out += '\t'; out += o; }
    out += '\n';
    for (auto const & s : samples) {
      out += "vsearch\t"; out += s; out += '\t'; out += std::to_string(otus.size());
      for (auto const & o : otus) {
        auto const it = count.find({o, s});
        out += '\t'; out += std::to_string(it == count.end() ? 0 : it->second);
      }
      out += '\n';
    }
    return out;
  }
};

int vsg::dust_case(vsg_ctx * ctx, vsg_seqset * set, std::vector<char> & cat)
{
  int rc = vsg_seqset_dust(ctx, set);
  if (rc != VSG_OK) { return rc; }
  std::vector<uint8_t> sym(cat.size());
  if ((rc = vsg_seqset_symbols(ctx, set, sym.data(), static_cast<int64_t>(sym.size()))) != VSG_OK) { return rc; }
  for (size_t i = 0; i + 1 < cat.size(); i++) {
    unsigned char const ch = static_cast<unsigned char>(cat[i]);
    cat[i] = static_cast<char>((sym[i] & 0x10) != 0 ? (ch | 0x20) : (ch >= 'a' && ch <= 'z' ? ch & ~0x20 : ch));
  }
  return VSG_OK;
}

void vsg::hardmask(std::vector<char> & cat)
{
  for (size_t i = 0; i + 1 < cat.size(); i++) { if (cat[i] >= 'a' && cat[i] <= 'z') { cat[i] = 'N'; } }
}

int vsg::search_db_labels(const char * caller, bool self, SearchDb & db)
{
  size_t const n = db.file.head.size();
  if (n > 0x7fffffffULL) { Error::set(std::string(caller) + ": too many database sequences"); return VSG_EINVAL; }
  db.size.resize(n);
  db.heads.resize(n);
  for (size_t i = 0; i < n; i++) {
    std::string err;
    if (!abundance_of(db.file.head[i], db.size[i], err)) {
      Error::set(std::string(caller) + ": " + err + " (" + db.file.head[i] + ")");
      return VSG_EINVAL;
    }
    db.heads[i] = db.file.head[i].c_str();
  }
  if (self) {
    db.label_id.resize(n);
    for (size_t i = 0; i < n; i++) { db.label_id[i] = db.label_ids.emplace(db.file.head[i], static_cast<int64_t>(i)).first->second; }
  }
  return VSG_OK;
}

int vsg::search_db_read(vsg_ctx * ctx, const char * caller, const char * path, bool notrunclabels, int64_t minlen, int64_t maxlen,
                        int dbmask, bool hardmask_soft, bool dust, bool self, SearchDb & db)
{
  int rc = read_fastx_file(caller, path, notrunclabels, minlen, maxlen, db.file);
  if (rc != VSG_OK) { return rc; }
  if (dbmask == VSG_DBMASK_SOFT && hardmask_soft) { hardmask(db.file.cat); }
  if ((rc = search_db_labels(caller, self, db)) != VSG_OK) { return rc; }
  vsg_seqset * raw = nullptr;
  if ((rc = vsg_seqset_create(ctx, db.file.cat.data(), db.file.off.data(), db.file.len.data(), static_cast<int64_t>(db.heads.size()), 1,
                              &raw)) != VSG_OK) { return rc; }
  db.set.reset(raw);
  if (dust && (rc = dust_case(ctx, db.set.get(), db.file.cat)) != VSG_OK) { return rc; }
  return VSG_OK;
}

int vsg::search_batch_opts(const char * caller, const std::vector<std::string> & heads, const SearchDb & db, const vsg_search_opts & s,
                           std::vector<int64_t> & size, std::vector<int64_t> & label, vsg_search_opts & o)
{
  size_t const nq = heads.size();
  size.resize(nq);
  for (size_t q = 0; q < nq; q++) {
    std::string err;
    if (!abundance_of(heads[q], size[q], err)) { Error::set(std::string(caller) + ": " + err + " (" + heads[q] + ")"); return VSG_EINVAL; }
  }
  o = s;
  o.query_sizes = size.data();
  o.target_sizes = db.size.data();
  if (s.self != 0) {
    label.resize(nq);
    for (size_t q = 0; q < nq; q++) {
      auto const it = db.label_ids.find(heads[q]);
      label[q] = it == db.label_ids.end() ? -1 : it->second;
    }
    o.query_labels = label.data();
    o.target_labels = db.label_id.data();
  }
  return VSG_OK;
}

SearchWriter::SearchWriter(const SearchWriterOpts & o, const vsg_search_exact_outputs & out, const std::vector<std::string> & dbhead,
                           const char * dbcat, const int64_t * dboff, const int32_t * dblen, const int64_t * dbsize)
    : o_(o), out_(out), dbhead_(dbhead), dbcat_(dbcat), dboff_(dboff), dblen_(dblen), dbsize_(dbsize),
      dbmatched_(dbhead.size(), 0), otu_(new OtuTable())
{
}

SearchWriter::~SearchWriter() = default;

int64_t SearchWriter::shown(const vsg_search_result * r, int64_t n) const
{
  int64_t const report = std::min(o_.maxhits == 0 ? INT64_MAX : o_.maxhits, n);   // vsearch.cc:188-191
  if (!o_.top_hits_only) { return report; }
  int64_t k = 0;   // usearch_global.cpp:208-215
  while (k < report && !(r[k].id < r[0].id)) { k++; }
  return k;
}

int64_t SearchWriter::uc_rows(int64_t shown) const
{
  return o_.uc_allhits ? shown : std::min<int64_t>(shown, 1);
}

void SearchWriter::batch(const SearchRows & b, std::string * outs)
{
  char row[96];
  for (int64_t q = 0; q < b.nq; q++) {
    int64_t const n = b.first[q + 1] - b.first[q];
    vsg_search_result const * const r = b.rows + b.first[q];
    int64_t const report = std::min(o_.maxhits == 0 ? INT64_MAX : o_.maxhits, n);
    int64_t const show = shown(r, n);
    int64_t const qsize = b.size[q];
    std::string const & head = b.head[q];
    queries++;
    queries_abundance += qsize;
    hits += n;
    if (out_.blast6out != nullptr) { blast6 += blast6_rows(outs[0], head, r, show, dbhead_ptrs(), o_.output_no_hits); }
    if (out_.uc != nullptr) {   // results_show_uc_one (core/results.cpp:274-330)
      if (report == 0) { outs[1] += "N\t*\t*\t*\t.\t*\t*\t*\t"; outs[1] += head; outs[1] += "\t*\n"; }
      for (int64_t j = 0; j < uc_rows(show); j++) {
        outs[1].append(row, static_cast<size_t>(std::snprintf(row, sizeof row, "H\t%d\t%d\t%.1f\t%c\t0\t0\t", r[j].target, b.len[q],
                                                              r[j].id, r[j].strand != 0 ? '-' : '+')));
        if (r[j].matches == r[j].alignment_length) { outs[1] += '='; } else { outs[1] += b.cigar_buf + b.cigar_off[b.first[q] + j]; }
        outs[1] += '\t';
        header_fprint_strip(outs[1], head, o_.xsize);
        outs[1] += '\t';
        header_fprint_strip(outs[1], dbhead_[static_cast<size_t>(r[j].target)], o_.xsize);
        outs[1] += '\n';
      }
    }
    if (out_.otutabout != nullptr || out_.mothur_shared_out != nullptr) {
      otu_->add(&head, report > 0 ? &dbhead_[static_cast<size_t>(r[0].target)] : nullptr, qsize);
    }
    if (n > 0) {
      matched++;
      matched_abundance += qsize;
      if (out_.matched != nullptr) { fasta_print_general(outs[2], o_.fmt, head, b.cat + b.off[q], b.len[q], qsize, matched, -1); }
    } else if (out_.notmatched != nullptr) {
      fasta_print_general(outs[3], o_.fmt, head, b.cat + b.off[q], b.len[q], qsize, queries - matched, -1);
    }
    for (int64_t j = 0; j < n; j++) {
      if (r[j].accepted != 0 || o_.weak_dbmatched) {
        dbmatched_[static_cast<size_t>(r[j].target)] += static_cast<uint64_t>(o_.sizein ? qsize : 1);
      }
    }
  }
}

const char * const * SearchWriter::dbhead_ptrs()
{
  if (dbheads_.size() != dbhead_.size()) {
    dbheads_.resize(dbhead_.size());
    for (size_t i = 0; i < dbhead_.size(); i++) { dbheads_[i] = dbhead_[i].c_str(); }
  }
  return dbheads_.data();
}

bool SearchWriter::finish(const char * caller, OutFiles & files)
{
  size_t const ndb = dbhead_.size();
  auto write = [&](const char * path, const std::string & data) {
    if (path == nullptr || files.write(path, data)) { return true; }
    Error::set(std::string(caller) + ": cannot write " + path);
    return false;
  };
  if (out_.otutabout != nullptr || out_.mothur_shared_out != nullptr) {
    for (size_t i = 0; i < ndb; i++) { if (dbmatched_[i] == 0) { otu_->add(nullptr, &dbhead_[i], 0); } }
    if (!write(out_.otutabout, out_.otutabout != nullptr ? otu_->otutabout() : std::string()) ||
        !write(out_.mothur_shared_out, out_.mothur_shared_out != nullptr ? otu_->mothur_shared_out() : std::string())) {
      return false;
    }
  }
  if (out_.dbmatched != nullptr || out_.dbnotmatched != nullptr) {
    std::string dbm, dbn;
    int64_t nm = 0, nn = 0;
    for (size_t k = 0; k < ndb; k++) {
      if (dbmatched_[k] != 0) {
        if (out_.dbmatched != nullptr) {
          fasta_print_general(dbm, o_.fmt, dbhead_[k], dbcat_ + dboff_[k], dblen_[k], static_cast<int64_t>(dbmatched_[k]), ++nm, -1);
        }
      } else if (out_.dbnotmatched != nullptr) {
        fasta_print_general(dbn, o_.fmt, dbhead_[k], dbcat_ + dboff_[k], dblen_[k], o_.dbnotmatched_size ? dbsize_[k] : 0, ++nn, -1);
      }
    }
    if (!write(out_.dbmatched, dbm) || !write(out_.dbnotmatched, dbn)) { return false; }
  }
  return true;
}

SearchWriterOpts vsg::usearch_global_writer_opts(const vsg_usearch_global_opts & u)
{
  SearchWriterOpts w;
  w.maxhits = u.maxhits;
  w.top_hits_only = u.top_hits_only != 0;
  w.uc_allhits = u.uc_allhits != 0;
  w.output_no_hits = u.output_no_hits != 0;
  w.sizein = u.sizein != 0;
  w.xsize = u.xsize != 0;
  w.weak_dbmatched = true;
  w.dbnotmatched_size = true;
  w.fmt = FastaFormat{nullptr, u.xsize != 0, u.sizeout != 0, u.fasta_width};
  return w;
}

extern "C" int vsg_search_write(int64_t nq, const char * const * query_headers, const char * qcat, const int64_t * qoff, const int32_t * qlen,
                                const int64_t * query_sizes, const vsg_search_result * rows, const int64_t * first, const char * cigar_buf,
                                const int64_t * cigar_off, int64_t ndb, const char * const * db_headers, const char * dbcat,
                                const int64_t * dboff, const int32_t * dblen, const int64_t * db_sizes, const vsg_usearch_global_opts * u,
                                const vsg_usearch_global_outputs * outputs, int64_t * matched)
{
  char const * const caller = "vsg_search_write";
  if (u == nullptr || outputs == nullptr || first == nullptr || nq < 0 || ndb < 0 ||
      (nq > 0 && (query_headers == nullptr || qcat == nullptr || qoff == nullptr || qlen == nullptr || query_sizes == nullptr)) ||
      (ndb > 0 && (db_headers == nullptr || dbcat == nullptr || dboff == nullptr || dblen == nullptr || db_sizes == nullptr))) {
    Error::set("vsg_search_write: null argument");
    return VSG_EINVAL;
  }
  if (u->maxhits < 0) { Error::set("vsg_search_write: The argument to maxhits cannot be negative"); return VSG_EINVAL; }
  int64_t const nrows = nq > 0 ? first[nq] : 0;
  if ((nrows > 0 && rows == nullptr) || first[0] != 0) { Error::set("vsg_search_write: bad rows"); return VSG_EINVAL; }
  for (int64_t q = 0; q < nq; q++) {
    if (first[q + 1] < first[q]) { Error::set("vsg_search_write: first is not ascending"); return VSG_EINVAL; }
  }
  for (int64_t j = 0; j < nrows; j++) {
    if (rows[j].target < 0 || rows[j].target >= ndb) {
      Error::set("vsg_search_write: row " + std::to_string(j) + " names no database sequence");
      return VSG_EINVAL;
    }
  }
  std::vector<std::string> qhead(static_cast<size_t>(nq)), dbhead(static_cast<size_t>(ndb));
  for (int64_t i = 0; i < nq; i++) { qhead[static_cast<size_t>(i)] = query_headers[i]; }
  for (int64_t i = 0; i < ndb; i++) { dbhead[static_cast<size_t>(i)] = db_headers[i]; }
  SearchWriterOpts const w = usearch_global_writer_opts(*u);
  SearchWriter writer(w, *outputs, dbhead, dbcat, dboff, dblen, db_sizes);
  // CIGARs are read only for the printed --uc rows that are not "="
  if (outputs->uc != nullptr) {
    for (int64_t q = 0; q < nq; q++) {
      int64_t const rows_q = writer.uc_rows(writer.shown(rows + first[q], first[q + 1] - first[q]));
      for (int64_t j = first[q]; j < first[q] + rows_q; j++) {
        if (rows[j].matches != rows[j].alignment_length && (cigar_buf == nullptr || cigar_off == nullptr || cigar_off[j] < 0)) {
          Error::set("vsg_search_write: row " + std::to_string(j) + " is printed in --uc and needs its CIGAR");
          return VSG_EINVAL;
        }
      }
    }
  }
  SearchRows const b{nq, qhead.data(), qcat, qoff, qlen, query_sizes, rows, first, cigar_buf, cigar_off};
  std::string outs[4];
  writer.batch(b, outs);
  OutFiles files;
  char const * const paths[4] = {outputs->blast6out, outputs->uc, outputs->matched, outputs->notmatched};
  for (int i = 0; i < 4; i++) {
    if (paths[i] != nullptr && !files.write(paths[i], outs[i])) { Error::set(std::string(caller) + ": cannot write " + paths[i]); return VSG_EINVAL; }
  }
  if (!writer.finish(caller, files)) { return VSG_EINVAL; }
  files.ok = true;
  if (matched != nullptr) { *matched = writer.matched; }
  return VSG_OK;
}

int vsg::strand_cigars(vsg_ctx * c, const vsg_seqset * queries, const vsg_seqset * targets, const std::vector<uint32_t> & q,
                       const std::vector<uint32_t> & t, const std::vector<uint8_t> & strand, std::vector<char> & buf,
                       std::vector<int64_t> & offs, int64_t & deferred)
{
  deferred = -1;
  offs.assign(q.size(), -1);
  SeqsetPtr rc_set;
  for (uint8_t s = 0; s < 2; s++) {
    std::vector<size_t> pick;
    std::vector<uint32_t> qs, ts;
    int64_t cap = 0;
    for (size_t j = 0; j < q.size(); j++) {
      if (strand[j] != s) { continue; }
      pick.push_back(j);
      qs.push_back(q[j]);
      ts.push_back(t[j]);
      cap += queries->h_len[q[j]] + targets->h_len[t[j]] + 1;
    }
    if (pick.empty()) { continue; }
    int rc = VSG_OK;
    if (s == 1 && (rc = seqset_revcomp(c, queries, 0, static_cast<int64_t>(queries->h_len.size()), rc_set)) != VSG_OK) { return rc; }
    size_t const m = pick.size();
    std::vector<int16_t> score(m);
    std::vector<uint16_t> aligned(m), matches(m), mismatches(m), gaps(m);
    std::vector<char> cb(static_cast<size_t>(cap) + 1);
    std::vector<int64_t> bo(m + 1);
    if ((rc = vsg_align_pairs(c, s == 0 ? queries : rc_set.get(), targets, static_cast<int64_t>(m), qs.data(), ts.data(), score.data(),
                              aligned.data(), matches.data(), mismatches.data(), gaps.data(), nullptr, cb.data(), cap + 1, bo.data())) != VSG_OK) {
      return rc;
    }
    for (size_t k = 0; k < m; k++) {
      if (score[k] == VSG_SCORE_SENTINEL) {
        if (deferred < 0 || static_cast<int64_t>(pick[k]) < deferred) { deferred = static_cast<int64_t>(pick[k]); }
        continue;
      }
      offs[pick[k]] = static_cast<int64_t>(buf.size());
      buf.insert(buf.end(), cb.begin() + bo[k], cb.begin() + bo[k + 1]);
      if (buf.empty() || buf.back() != '\0') { buf.push_back('\0'); }
    }
  }
  return VSG_OK;
}
