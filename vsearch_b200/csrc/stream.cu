// stream.cu — the streaming command drivers (SURVEY.md §8 f1): the multi-GPU --usearch_global stream (FASTA in,
// --blast6out out), --sintax (--tabbedout out), --orient (FASTA or FASTQ in, up to four outputs), and the --search_exact
// and --usearch_global commands (one GPU, FASTA or FASTQ in, the writers of search_out.cu).
//
// Replaces, around vsg_group_search, the host loop of the reference's command
//   search_thread_run / search_query      (commands/usearch_global.cpp:376-534)   read a query under mutex_input,
//                                                                                  mask it, search it
//   search_output_results                 (commands/usearch_global.cpp:150-300)   under mutex_output
//   results_show_blast6out_one            (core/results.cpp:221-271)
// by a three-stage pipeline over batches: a reader thread parses the file, the calling thread keeps the GPUs busy
// (upload, DUST, ranking, alignment, accept/reject, hit table), a writer thread formats rows in input order.  At the
// device's rate (hundreds of thousands of queries per second) one query at a time under two mutexes is the
// bottleneck; here parsing batch n+1 and formatting batch n-1 overlap the search of batch n.
#include "vsg_internal.h"

#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <climits>
#include <cstdio>
#include <cstring>
#include <deque>
#include <iterator>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

using namespace vsg;

namespace {

struct StreamBatch {
  int64_t first = 0;                 // index of the batch's first query in the file
  std::vector<char> cat;             // sequences back to back
  std::vector<char> qual;            // FASTQ: the qualities at the sequences' offsets
  bool fastq = false;
  std::vector<int64_t> off;
  std::vector<int32_t> len;
  std::vector<std::string> head;
  std::vector<vsg_search_result> res;   // query q's rows are res[row_first[q] .. row_first[q + 1])
  std::vector<int64_t> row_first;
  std::vector<vsg_sintax_result> tax;   // --sintax: one record per query
  std::vector<vsg_orient_result> orient;   // --orient: one record per query
  std::vector<int64_t> size;               // the search commands: the abundance of each query
  std::vector<char> cigar;                 // --usearch_global: row j's CIGAR at cigar[cigar_off[j]] (-1: none needed)
  std::vector<int64_t> cigar_off;
  bool last = false;
};

// a bounded hand-over between two stages
class Channel {
 public:
  explicit Channel(size_t cap) : cap_(cap) {}
  void put(std::unique_ptr<StreamBatch> b)
  {
    std::unique_lock<std::mutex> lk(m_);
    cv_.wait(lk, [&] { return q_.size() < cap_ || closed_; });
    if (closed_) { return; }
    q_.push_back(std::move(b));
    cv_.notify_all();
  }
  std::unique_ptr<StreamBatch> get()
  {
    std::unique_lock<std::mutex> lk(m_);
    cv_.wait(lk, [&] { return !q_.empty() || closed_; });
    if (q_.empty()) { return nullptr; }
    std::unique_ptr<StreamBatch> b = std::move(q_.front());
    q_.pop_front();
    cv_.notify_all();
    return b;
  }
  void close()
  {
    std::lock_guard<std::mutex> lk(m_);
    closed_ = true;
    cv_.notify_all();
  }
 private:
  std::mutex m_;
  std::condition_variable cv_;
  std::deque<std::unique_ptr<StreamBatch>> q_;
  size_t cap_;
  bool closed_ = false;
};

double seconds_since(std::chrono::steady_clock::time_point t0)
{
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

// db.read's rules for the records it keeps (core/db.cpp, core/fasta.cpp, core/fastq.cpp), which --makeudb_usearch and the
// clustering commands apply (read_fastx_file); the search, --sintax and --orient streams read with the default (no rules).
//   symbols: FASTA sequence bytes by core/fasta.cpp's action table — the IUPAC letters kept, tab, VT, FF and CR dropped
//            silently, other control bytes, '-' and '.' an error naming the line, anything else stripped and counted;
//            control bytes in a header an error.  FASTQ sequence bytes: IUPAC letters only; quality bytes: 33..126.
//   minlen / maxlen: records shorter or longer are discarded and counted.
struct FastxRules {
  bool symbols = false;
  int64_t minlen = 0, maxlen = INT64_MAX;
  int64_t stripped = 0, discarded_short = 0, discarded_long = 0;
};

enum class Sym : unsigned char { keep, strip, drop, reject, unprintable };

bool iupac_letter(unsigned char ch)
{
  return ((ch >= 'A' && ch <= 'Z') || (ch >= 'a' && ch <= 'z')) && std::strchr("ABCDGHKMNRSTUVWY", ch & ~0x20) != nullptr;
}

Sym fasta_symbol(unsigned char ch)
{
  if (ch == '\t' || ch == 11 || ch == 12 || ch == '\r') { return Sym::drop; }
  if (ch < 32) { return Sym::unprintable; }
  if (ch == '-' || ch == '.') { return Sym::reject; }
  return iupac_letter(ch) ? Sym::keep : Sym::strip;
}

// FASTA or FASTQ records of a file, one batch at a time.  The format is that of the file's first byte, as fastx_open
// finds it (core/fastx.cpp): '@' is FASTQ, anything else FASTA; gzip and bzip2 files are recognised by their magic bytes
// and refused.  FASTA (core/fasta.cpp / fastx.cpp): a header runs to the end of its line and is cut at the first blank
// unless --notrunclabels; sequence lines are joined, white space dropped.  FASTQ (core/fastq.cpp:324-581): a header line
// that starts with '@', sequence lines up to the first line that starts with '+', a '+' line that is empty or repeats
// the header, quality lines until the next line that starts with '@' once the quality is as long as the sequence; a
// record that breaks one of these rules, ends early or has a quality of another length is an error.
class FastxReader {
 public:
  enum Kind { FASTA, FASTQ, GZIP, BZIP2 };
  FastxReader(std::FILE * f, bool notrunc, FastxRules * rules = nullptr) : f_(f), notrunc_(notrunc), rules_(rules), buf_(1 << 22)
  {
    end_ = std::fread(buf_.data(), 1, buf_.size(), f_);
    unsigned char const * const u = reinterpret_cast<unsigned char const *>(buf_.data());
    if (end_ >= 2 && u[0] == 0x1f && u[1] == 0x8b) { kind_ = GZIP; }
    else if (end_ >= 3 && u[0] == 'B' && u[1] == 'Z' && u[2] == 'h') { kind_ = BZIP2; }
    else if (end_ >= 1 && u[0] == '@') { kind_ = FASTQ; }
  }
  Kind kind() const { return kind_; }
  // false when the file is exhausted and nothing was read
  bool fill(StreamBatch & b, int want, std::string & err)
  {
    b.cat.clear(); b.qual.clear(); b.off.clear(); b.len.clear(); b.head.clear();
    b.fastq = kind_ == FASTQ;
    if (kind_ == FASTQ) {
      if (!fill_fastq(b, want, err)) { return false; }
    } else {
      fill_fasta(b, want, err);
      if (!err.empty()) { return false; }
    }
    b.cat.push_back('\0');
    return !b.head.empty();
  }
 private:
  void fill_fasta(StreamBatch & b, int want, std::string & err)
  {
    while (static_cast<int>(b.head.size()) < want) {
      if (!have_header_) {
        if (!next_line()) { break; }
        if (line_.empty()) { continue; }
        if (line_[0] != '>') { err = "FASTA: a sequence line before the first header"; return; }
        pending_ = header_of(line_);
        have_header_ = true;
        if (!check_header(pending_, err)) { return; }
      }
      // sequence lines up to the next header
      int64_t const o = static_cast<int64_t>(b.cat.size());
      bool more = false;
      while (next_line()) {
        if (!line_.empty() && line_[0] == '>') { more = true; break; }
        if (rules_ != nullptr && rules_->symbols) {
          if (!fasta_line(b, err)) { return; }
        } else {
          for (char ch : line_) { if (ch != ' ' && ch != '\t' && ch != '\r') { b.cat.push_back(ch); } }
        }
      }
      int64_t const l = static_cast<int64_t>(b.cat.size()) - o;
      if (l > 0x7fffffff) { err = "FASTA: a sequence longer than 2^31"; return; }
      if (keep(b, o, l)) { b.off.push_back(o); b.len.push_back(static_cast<int32_t>(l)); b.head.push_back(pending_); }
      if (more) {
        pending_ = header_of(line_); have_header_ = true;
        if (!check_header(pending_, err)) { return; }
      } else {
        have_header_ = false;
      }
      if (!more) { break; }
    }
  }
  bool fill_fastq(StreamBatch & b, int want, std::string & err)
  {
    while (static_cast<int>(b.head.size()) < want) {
      if (!have_header_ && !next_line()) { break; }
      have_header_ = false;
      records_++;
      auto fail = [&](const char * what) { err = "FASTQ record " + std::to_string(records_) + ": " + what; return false; };
      if (line_.empty() || line_[0] != '@') { return fail("the header line does not start with '@'"); }
      if (!newline_) { return fail("the file ends early"); }
      header_line_.swap(line_);
      std::string head = header_of(header_line_);
      if (!check_header(head, err)) { return false; }
      int64_t const o = static_cast<int64_t>(b.cat.size());
      bool const symbols = rules_ != nullptr && rules_->symbols;
      for (;;) {
        if (!next_line() || !newline_) { return fail("the file ends early"); }
        if (!line_.empty() && line_[0] == '+') { break; }
        if (symbols) {
          for (char ch : line_) {
            if (ch == '\r') { continue; }
            if (!iupac_letter(static_cast<unsigned char>(ch))) { return fail(illegal("sequence", ch).c_str()); }
            b.cat.push_back(ch);
          }
        } else {
          b.cat.insert(b.cat.end(), line_.begin(), line_.end());
        }
      }
      if (line_.size() > 1 && line_.compare(1, std::string::npos, header_line_, 1, std::string::npos) != 0) {
        return fail("the '+' line is neither empty nor the header");
      }
      int64_t const l = static_cast<int64_t>(b.cat.size()) - o;
      if (l > 0x7fffffff) { return fail("a sequence longer than 2^31"); }
      bool first = true;
      while (next_line()) {
        if (!first && !line_.empty() && line_[0] == '@' && static_cast<int64_t>(b.qual.size()) - o == l) { have_header_ = true; break; }
        first = false;
        if (symbols) {
          for (char ch : line_) {
            if (ch < 33 || ch > 126) { return fail(illegal("quality", ch).c_str()); }
          }
        }
        b.qual.insert(b.qual.end(), line_.begin(), line_.end());
        if (static_cast<int64_t>(b.qual.size()) - o > l) { break; }
      }
      if (static_cast<int64_t>(b.qual.size()) - o != l) { return fail("the quality is not as long as the sequence"); }
      if (keep(b, o, l)) { b.off.push_back(o); b.len.push_back(static_cast<int32_t>(l)); b.head.push_back(std::move(head)); }
      else { b.qual.resize(static_cast<size_t>(o)); }
    }
    return true;
  }
  // the rules' length limits: false (the record's bytes removed, the discard counted) for a record outside them
  bool keep(StreamBatch & b, int64_t o, int64_t l)
  {
    if (rules_ == nullptr) { return true; }
    if (l >= rules_->minlen && l <= rules_->maxlen) { return true; }
    (l < rules_->minlen ? rules_->discarded_short : rules_->discarded_long)++;
    b.cat.resize(static_cast<size_t>(o));
    return false;
  }
  // a FASTA sequence line under the rules' symbol table
  bool fasta_line(StreamBatch & b, std::string & err)
  {
    for (char ch : line_) {
      unsigned char const u = static_cast<unsigned char>(ch);
      switch (fasta_symbol(u)) {
        case Sym::keep: b.cat.push_back(ch); break;
        case Sym::strip: rules_->stripped++; break;
        case Sym::drop: break;
        case Sym::reject:
          err = std::string("Illegal character '") + ch + "' in sequence on line " + std::to_string(lineno_) + " of FASTA file";
          return false;
        case Sym::unprintable:
          err = "Illegal unprintable ASCII character no " + std::to_string(u) + " in sequence on line " + std::to_string(lineno_) +
                " of FASTA file";
          return false;
      }
    }
    return true;
  }
  // fastx_filter_header: no control byte but tab, no DEL, in the label as it is kept
  bool check_header(const std::string & head, std::string & err) const
  {
    if (rules_ == nullptr || !rules_->symbols) { return true; }
    for (char ch : head) {
      unsigned char const u = static_cast<unsigned char>(ch);
      if (u == 127 || (u > 0 && u < 32 && u != '\t')) {
        err = "Illegal character encountered in FASTA/FASTQ header: unprintable ASCII character no " + std::to_string(u) +
              " on line " + std::to_string(lineno_);
        return false;
      }
    }
    return true;
  }
  std::string illegal(const char * what, char ch) const
  {
    unsigned char const u = static_cast<unsigned char>(ch);
    std::string const sym = (u > 32 && u < 127) ? std::string("'") + ch + "'" : "(unprintable, no " + std::to_string(u) + ")";
    return std::string("Illegal ") + what + " character " + sym + " on line " + std::to_string(lineno_);
  }
  std::string header_of(const std::string & line) const
  {
    size_t e = line.size();
    if (!notrunc_) { for (size_t i = 1; i < line.size(); i++) { if (line[i] == ' ' || line[i] == '\t') { e = i; break; } } }
    return line.substr(1, e - 1);
  }
  bool next_line()
  {
    line_.clear();
    for (;;) {
      if (pos_ == end_) {
        end_ = std::fread(buf_.data(), 1, buf_.size(), f_);
        pos_ = 0;
        if (end_ == 0) {
          newline_ = false;
          bool const got = !line_.empty() || got_partial_();
          lineno_ += got ? 1 : 0;
          return got;
        }
      }
      char const * const s = buf_.data() + pos_;
      char const * const nl = static_cast<char const *>(std::memchr(s, '\n', end_ - pos_));
      if (nl == nullptr) { line_.append(s, end_ - pos_); pos_ = end_; partial_ = true; continue; }
      line_.append(s, static_cast<size_t>(nl - s));
      pos_ += static_cast<size_t>(nl - s) + 1;
      partial_ = false;
      newline_ = true;
      lineno_++;
      if (!line_.empty() && line_.back() == '\r') { line_.pop_back(); }
      return true;
    }
  }
  bool got_partial_() { bool const p = partial_; partial_ = false; return p; }
  std::FILE * f_;
  bool notrunc_;
  FastxRules * rules_;
  std::vector<char> buf_;
  size_t pos_ = 0, end_ = 0;
  bool partial_ = false, newline_ = false;   // newline_: the last line read ended with '\n'
  Kind kind_ = FASTA;
  int64_t records_ = 0;
  int64_t lineno_ = 0;   // the number of the line last read, from 1
  std::string line_, pending_, header_line_;
  bool have_header_ = false;   // line_ (FASTQ) or pending_ (FASTA) holds the next record's header
};

// The three stages over the batches of one FASTA or FASTQ file: the reader thread parses batches of batch_queries
// records, the calling thread runs work(batch) (the GPU stage), the writer thread has format(batch, outs, stats) fill
// one string per output path and appends each to its file (a null path: no file) in input order.  need_fastq: FASTA
// input is an error.  Returns the first error of work, of the output files or of the parser, with `caller` in its
// message.  opened (optional) receives every output path the call created.
template <class Work, class Format>
int run_stream(const char * caller, const char * query_path, std::vector<const char *> const & out_paths, bool notrunclabels,
               int batch_queries, bool need_fastq, vsg_stream_stats * stats, Work && work, Format && format,
               std::vector<std::string> * opened = nullptr)
{
  std::FILE * fin = std::fopen(query_path, "rb");
  if (fin == nullptr) { Error::set(std::string(caller) + ": cannot open " + query_path); return VSG_EINVAL; }
  FastxReader fr(fin, notrunclabels);
  char const * refused = nullptr;
  if (fr.kind() == FastxReader::GZIP) { refused = ": gzip-compressed input is not supported: "; }
  else if (fr.kind() == FastxReader::BZIP2) { refused = ": bzip2-compressed input is not supported: "; }
  else if (need_fastq && fr.kind() != FastxReader::FASTQ) { refused = ": cannot write FASTQ output with FASTA input: "; }
  if (refused != nullptr) { std::fclose(fin); Error::set(std::string(caller) + refused + query_path); return VSG_EINVAL; }
  std::vector<std::FILE *> fout(out_paths.size(), nullptr);
  for (size_t i = 0; i < out_paths.size(); i++) {
    if (out_paths[i] == nullptr) { continue; }
    fout[i] = std::fopen(out_paths[i], "wb");
    if (fout[i] != nullptr && opened != nullptr) { opened->push_back(out_paths[i]); }
    if (fout[i] == nullptr) {
      for (std::FILE * f : fout) { if (f != nullptr) { std::fclose(f); } }
      std::fclose(fin);
      Error::set(std::string(caller) + ": cannot write " + out_paths[i]);
      return VSG_EINVAL;
    }
  }

  auto const t_wall = std::chrono::steady_clock::now();
  vsg_stream_stats st{};
  Channel parsed(2), searched(2);
  std::string reader_err;
  std::thread reader([&] {
    int64_t first = 0;
    for (;;) {
      auto const t0 = std::chrono::steady_clock::now();
      std::unique_ptr<StreamBatch> b(new StreamBatch());
      bool const ok = fr.fill(*b, batch_queries, reader_err);
      st.parse_s += seconds_since(t0);
      if (!ok) { break; }
      b->first = first;
      first += static_cast<int64_t>(b->head.size());
      parsed.put(std::move(b));
    }
    std::unique_ptr<StreamBatch> e(new StreamBatch());
    e->last = true;
    parsed.put(std::move(e));
  });
  std::thread writer([&] {
    std::vector<std::string> outs(out_paths.size());
    for (;;) {
      std::unique_ptr<StreamBatch> b = searched.get();
      if (b == nullptr || b->last) { break; }
      auto const t0 = std::chrono::steady_clock::now();
      for (auto & o : outs) { o.clear(); }
      format(*b, outs, st);
      for (size_t i = 0; i < outs.size(); i++) {
        if (fout[i] != nullptr) { std::fwrite(outs[i].data(), 1, outs[i].size(), fout[i]); }
      }
      st.write_s += seconds_since(t0);
    }
  });

  int rc = VSG_OK;
  for (;;) {
    std::unique_ptr<StreamBatch> b = parsed.get();
    if (b == nullptr || b->last) { break; }
    auto const t0 = std::chrono::steady_clock::now();
    int64_t const nq = static_cast<int64_t>(b->head.size());
    rc = work(*b);
    st.search_s += seconds_since(t0);
    if (rc != VSG_OK) { break; }
    st.queries += nq; st.batches++;
    st.nucleotides += static_cast<int64_t>(b->cat.size()) - 1;
    searched.put(std::move(b));
  }
  if (rc != VSG_OK) { parsed.close(); }   // unblocks the reader
  {
    std::unique_ptr<StreamBatch> e(new StreamBatch());
    e->last = true;
    searched.put(std::move(e));
  }
  reader.join();
  writer.join();
  std::fclose(fin);
  for (std::FILE * f : fout) {
    if (f != nullptr && std::fclose(f) != 0 && rc == VSG_OK) { Error::set(std::string(caller) + ": write error"); rc = VSG_EINVAL; }
  }
  if (rc == VSG_OK && !reader_err.empty()) { Error::set(std::string(caller) + ": " + reader_err); rc = VSG_EINVAL; }
  st.wall_s = seconds_since(t_wall);
  if (stats != nullptr) { *stats = st; }
  return rc;
}

}  // namespace

int64_t vsg::blast6_rows(std::string & out, const std::string & qhead, const vsg_search_result * r, int64_t n,
                         const char * const * target_labels, bool output_no_hits)
{
  if (n == 0 && output_no_hits) {
    out += qhead; out += "\t*\t0.0\t0\t0\t0\t0\t0\t0\t0\t-1\t0\n";   // results.cpp:248-250
    return 1;
  }
  char row[256];
  for (int64_t j = 0; j < n; j++) {
    int const qstart = r[j].strand != 0 ? r[j].query_length : 1, qend = r[j].strand != 0 ? 1 : r[j].query_length;
    out += qhead; out += '\t'; out += target_labels[r[j].target];
    int const w = std::snprintf(row, sizeof row, "\t%.1f\t%d\t%d\t%d\t%d\t%d\t%d\t%d\t%d\t%d\n", r[j].id, r[j].internal_alignment_length,
                                r[j].mismatches, r[j].internal_gaps, qstart, qend, 1, r[j].target_length, -1, 0);
    out.append(row, static_cast<size_t>(w));
  }
  return n;
}

extern "C" int vsg_usearch_stream(vsg_group * g, const char * const * target_labels, const char * query_fasta,
                                  const vsg_search_opts * opts, int qmask_dust, int notrunclabels, int batch_queries,
                                  int64_t maxhits, int output_no_hits, const char * blast6out_path, vsg_stream_stats * stats)
{
  if (g == nullptr || target_labels == nullptr || query_fasta == nullptr || opts == nullptr || blast6out_path == nullptr) {
    Error::set("vsg_usearch_stream: null argument");
    return VSG_EINVAL;
  }
  if (batch_queries < 1) { batch_queries = 65536; }
  if (maxhits < 0) { maxhits = 0; }
  return run_stream("vsg_usearch_stream", query_fasta, {blast6out_path}, notrunclabels != 0, batch_queries, false, stats,
                    [&](StreamBatch & b) {
    // every row min(maxhits, hits) asks for, built on the host by the group search itself: no buffer to outgrow
    return group_search_rows(g, b.cat.data(), b.off.data(), b.len.data(), static_cast<int64_t>(b.head.size()), qmask_dust,
                             opts, maxhits, b.res, b.row_first, nullptr);
  }, [&](StreamBatch const & b, std::vector<std::string> & outs, vsg_stream_stats & st) {
    std::string & out = outs[0];
    size_t const nq = b.head.size();
    for (size_t q = 0; q < nq; q++) {
      int64_t const n = b.row_first[q + 1] - b.row_first[q];
      if (n > 0) { st.matched++; }
      st.rows += blast6_rows(out, b.head[q], b.res.data() + b.row_first[q], n, target_labels, output_no_hits != 0);
    }
  });
}

// The --sintax command (commands/sintax.cpp:519-604, 679-800) over the same pipeline: headers kept whole
// (--notrunclabels is forced for --sintax, cli.cc:4497-4520), record n of the file uses random substream n, and the
// rows of vsg_sintax_rows go out in input order (the reference's order with --threads 1).  stats: `matched` counts the
// classified queries, `rows` every query.
extern "C" int vsg_sintax_stream(vsg_group * g, const char * const * target_headers, const char * query_fasta,
                                 const vsg_sintax_opts * opts, int batch_queries, const char * tabbedout_path,
                                 vsg_stream_stats * stats)
{
  if (g == nullptr || target_headers == nullptr || query_fasta == nullptr || opts == nullptr || tabbedout_path == nullptr) {
    Error::set("vsg_sintax_stream: null argument");
    return VSG_EINVAL;
  }
  int const rc = sintax_check_opts(opts, "vsg_sintax_stream");
  if (rc != VSG_OK) { return rc; }
  if (batch_queries < 1) { batch_queries = 65536; }
  return run_stream("vsg_sintax_stream", query_fasta, {tabbedout_path}, true, batch_queries, false, stats, [&](StreamBatch & b) {
    vsg_sintax_opts o = *opts;
    o.query_number0 = b.first;
    b.tax.resize(b.head.size());
    return group_sintax(g, b.cat.data(), b.off.data(), b.len.data(), static_cast<int64_t>(b.head.size()), &o, b.tax.data());
  }, [&](StreamBatch const & b, std::vector<std::string> & outs, vsg_stream_stats & st) {
    std::vector<const char *> heads(b.head.size());
    for (size_t q = 0; q < heads.size(); q++) {
      heads[q] = b.head[q].c_str();
      vsg_sintax_result const & r = b.tax[q];
      if (r.nboot[r.strand] >= (VSG_SINTAX_BOOTSTRAPS + 1) / 2) { st.matched++; }
    }
    sintax_rows_string(b.tax.data(), static_cast<int64_t>(heads.size()), heads.data(), target_headers, opts, outs[0]);
    st.rows += static_cast<int64_t>(heads.size());
  });
}

namespace {

// fasta_print_general / fasta_print_sequence (core/fasta.cpp:423-450, 482-...) without header rewriting: lines of
// `width` symbols (width < 1: one line, also for an empty sequence)
void fasta_record(std::string & out, const std::string & head, const char * seq, int64_t len, int width)
{
  out += '>'; out += head; out += '\n';
  if (width < 1) { out.append(seq, static_cast<size_t>(len)); out += '\n'; return; }
  for (int64_t i = 0; i < len; i += width) {
    out.append(seq + i, static_cast<size_t>(std::min<int64_t>(width, len - i)));
    out += '\n';
  }
}

// fastq_print_general (core/fastq.cpp:681-785) without header rewriting
void fastq_record(std::string & out, const std::string & head, const char * seq, const char * qual, int64_t len)
{
  out += '@'; out += head; out += '\n';
  out.append(seq, static_cast<size_t>(len)); out += "\n+\n";
  out.append(qual, static_cast<size_t>(len)); out += '\n';
}

}  // namespace

// The --orient command (commands/orient.cpp:116-441) over the same pipeline; outs are fastaout, fastqout, notmatched,
// tabbedout in that order.
extern "C" int vsg_orient_stream(vsg_group * g, const char * query_path, int query_mask_lower, int notrunclabels, int fasta_width,
                                 int batch_queries, const char * fastaout, const char * fastqout, const char * notmatched,
                                 const char * tabbedout, vsg_stream_stats * stats, int64_t * nstrand)
{
  if (g == nullptr || query_path == nullptr) { Error::set("vsg_orient_stream: null argument"); return VSG_EINVAL; }
  if (fastaout == nullptr && fastqout == nullptr && notmatched == nullptr && tabbedout == nullptr) {
    Error::set("vsg_orient_stream: no output file (fastaout, fastqout, notmatched or tabbedout)");
    return VSG_EINVAL;
  }
  if (batch_queries < 1) { batch_queries = 65536; }
  static Complement const comp;
  int64_t count[3] = {0, 0, 0};
  int const rc = run_stream("vsg_orient_stream", query_path, {fastaout, fastqout, notmatched, tabbedout}, notrunclabels != 0,
                            batch_queries, fastqout != nullptr, stats, [&](StreamBatch & b) {
    b.orient.resize(b.head.size());
    return group_orient(g, b.cat.data(), b.off.data(), b.len.data(), static_cast<int64_t>(b.head.size()), query_mask_lower,
                        b.orient.data());
  }, [&](StreamBatch const & b, std::vector<std::string> & outs, vsg_stream_stats & st) {
    std::string rseq, rqual;
    char row[64];
    for (size_t q = 0; q < b.head.size(); q++) {
      vsg_orient_result const & r = b.orient[q];
      const char * seq = b.cat.data() + b.off[q];
      const char * qual = b.fastq ? b.qual.data() + b.off[q] : nullptr;
      int64_t const len = b.len[q];
      count[r.strand]++;
      if (r.strand == 1) {
        rseq.resize(static_cast<size_t>(len));
        for (int64_t i = 0; i < len; i++) { rseq[static_cast<size_t>(i)] = comp.map[static_cast<unsigned char>(seq[len - 1 - i])]; }
        seq = rseq.data();
        if (qual != nullptr) { rqual.assign(std::reverse_iterator<const char *>(qual + len), std::reverse_iterator<const char *>(qual)); qual = rqual.data(); }
      }
      if (r.strand != 2) {
        st.matched++;
        if (fastaout != nullptr) { fasta_record(outs[0], b.head[q], seq, len, fasta_width); }
        if (fastqout != nullptr) { fastq_record(outs[1], b.head[q], seq, qual, len); }
      } else if (notmatched != nullptr) {
        if (b.fastq) { fastq_record(outs[2], b.head[q], seq, qual, len); } else { fasta_record(outs[2], b.head[q], seq, len, fasta_width); }
      }
      if (tabbedout != nullptr) {
        int const w = std::snprintf(row, sizeof row, "\t%c\t%u\t%u\n", "+-?"[r.strand], r.count_fwd, r.count_rev);
        outs[3] += b.head[q];
        outs[3].append(row, static_cast<size_t>(w));
      }
      st.rows++;
    }
  });
  if (nstrand != nullptr) { for (int s = 0; s < 3; s++) { nstrand[s] = count[s]; } }
  return rc;
}

// The whole of a FASTA or FASTQ file under db.read's rules (FastxRules): the records --makeudb_usearch and the clustering
// commands read into memory before they start.
int vsg::read_fastx_file(const char * caller, const char * path, bool notrunclabels, int64_t minlen, int64_t maxlen, FastxFile & out)
{
  std::FILE * fin = std::fopen(path, "rb");
  if (fin == nullptr) { Error::set(std::string(caller) + ": cannot open " + path); return VSG_EINVAL; }
  FastxRules rules;
  rules.symbols = true;
  rules.minlen = std::max<int64_t>(minlen, 0);
  rules.maxlen = maxlen;
  StreamBatch b;
  std::string err;
  {
    FastxReader fr(fin, notrunclabels, &rules);
    if (fr.kind() == FastxReader::GZIP) { err = "gzip-compressed input is not supported"; }
    else if (fr.kind() == FastxReader::BZIP2) { err = "bzip2-compressed input is not supported"; }
    else { fr.fill(b, INT32_MAX, err); }
  }
  std::fclose(fin);
  if (!err.empty()) { Error::set(std::string(caller) + ": " + err + " (" + path + ")"); return VSG_EINVAL; }
  if (b.cat.empty()) { b.cat.push_back('\0'); }
  out.cat = std::move(b.cat);
  out.off = std::move(b.off);
  out.len = std::move(b.len);
  out.head = std::move(b.head);
  out.stripped = rules.stripped;
  out.discarded_short = rules.discarded_short;
  out.discarded_long = rules.discarded_long;
  return VSG_OK;
}

// The --makeudb_usearch command (commands/makeudb_usearch.cpp:105-273): the whole file parsed under db.read's rules, the
// database made on the device (vsg_udb_make), the file written (vsg_udb_write).  The stages run one after another: the
// file's word index, which comes before its sequences, needs every sequence.
extern "C" int vsg_makeudb_usearch(vsg_ctx * c, const char * input_path, const vsg_makeudb_opts * opts, const char * output_path,
                                   vsg_makeudb_stats * stats)
{
  if (c == nullptr || input_path == nullptr || opts == nullptr) { Error::set("vsg_makeudb_usearch: null argument"); return VSG_EINVAL; }
  if (output_path == nullptr) { Error::set("vsg_makeudb_usearch: UDB output file must be specified"); return VSG_EINVAL; }
  int rc = makeudb_check_opts(opts, "vsg_makeudb_usearch");
  if (rc != VSG_OK) { return rc; }
  auto const t_wall = std::chrono::steady_clock::now();
  vsg_makeudb_stats st{};
  FastxFile b;
  rc = read_fastx_file("vsg_makeudb_usearch", input_path, opts->notrunclabels != 0, opts->minseqlength, opts->maxseqlength, b);
  if (rc != VSG_OK) { return rc; }
  int64_t const n = static_cast<int64_t>(b.head.size());
  std::vector<const char *> heads(static_cast<size_t>(n));
  for (int64_t i = 0; i < n; i++) { heads[static_cast<size_t>(i)] = b.head[static_cast<size_t>(i)].c_str(); }
  st.parse_s = seconds_since(t_wall);

  auto const t_dev = std::chrono::steady_clock::now();
  vsg_udb * u = nullptr;
  rc = vsg_udb_make(c, b.cat.data(), b.off.data(), b.len.data(), heads.data(), n, opts, &u);
  st.device_s = seconds_since(t_dev);
  if (rc != VSG_OK) { return rc; }
  auto const t_write = std::chrono::steady_clock::now();
  rc = vsg_udb_write(u, output_path);
  st.write_s = seconds_since(t_write);
  vsg_udb_info info{};
  vsg_udb_info_get(u, &info);
  vsg_udb_close(u);
  if (rc != VSG_OK) { return rc; }
  st.sequences = n;
  st.discarded_short = b.discarded_short;
  st.discarded_long = b.discarded_long;
  st.stripped = b.stripped;
  st.nucleotides = info.nucleotides;
  st.index_entries = info.index_entries;
  st.wall_s = seconds_since(t_wall);
  if (stats != nullptr) { *stats = st; }
  return VSG_OK;
}

extern "C" void vsg_search_exact_opts_default(vsg_search_exact_opts * e, vsg_search_opts * s)
{
  if (e != nullptr) {
    *e = vsg_search_exact_opts{};
    e->dbmask = VSG_DBMASK_DUST;
    e->qmask = VSG_DBMASK_DUST;
    e->fasta_width = 80;
    e->minseqlength = 1;
    e->maxseqlength = 50000;
    e->batch_queries = 65536;
  }
  if (s != nullptr) { vsg_search_opts_default(s); }
}


namespace {

// the refusals both search commands share (VSG_EINVAL, message prefixed with caller)
int search_command_check(const char * caller, int qmask, int dbmask, int hardmask, int64_t maxhits, const vsg_search_opts & s,
                         const vsg_search_exact_outputs & out)
{
  std::string const c(caller);
  if (out.blast6out == nullptr && out.uc == nullptr && out.matched == nullptr && out.notmatched == nullptr && out.dbmatched == nullptr &&
      out.dbnotmatched == nullptr && out.otutabout == nullptr && out.mothur_shared_out == nullptr) {
    Error::set(c + ": No output files specified");
    return VSG_EINVAL;
  }
  if (qmask < VSG_DBMASK_NONE || qmask > VSG_DBMASK_DUST || dbmask < VSG_DBMASK_NONE || dbmask > VSG_DBMASK_DUST) {
    Error::set(c + ": unknown qmask or dbmask");
    return VSG_EINVAL;
  }
  if (hardmask != 0 && (qmask == VSG_DBMASK_DUST || dbmask == VSG_DBMASK_DUST)) {
    Error::set(c + ": --qmask dust or --dbmask dust with --hardmask is not offered (DUST-masked symbols would become 'N')");
    return VSG_EINVAL;
  }
  if (maxhits < 0) { Error::set(c + ": The argument to maxhits cannot be negative"); return VSG_EINVAL; }
  if (s.query_sizes != nullptr || s.target_sizes != nullptr || s.query_labels != nullptr || s.target_labels != nullptr) {
    Error::set(c + ": the size and label arrays of the search options are the command's own: pass them NULL");
    return VSG_EINVAL;
  }
  return VSG_OK;
}

// a batch's queries on the device, masked: soft + hardmask turns lower case into 'N' on the host first; with `dust`,
// DUST on the device, and with print_case the printed sequences (b.cat) take its case
int batch_query_set(vsg_ctx * ctx, StreamBatch & b, int qmask, bool hardmask_soft, bool dust, bool print_case, SeqsetPtr & out)
{
  if (qmask == VSG_DBMASK_SOFT && hardmask_soft) { hardmask(b.cat); }
  vsg_seqset * raw = nullptr;
  int const rc = vsg_seqset_create(ctx, b.cat.data(), b.off.data(), b.len.data(), static_cast<int64_t>(b.head.size()), 1, &raw);
  if (rc != VSG_OK) { return rc; }
  out.reset(raw);
  if (!dust) { return VSG_OK; }
  return print_case ? dust_case(ctx, out.get(), b.cat) : vsg_seqset_dust(ctx, out.get());
}

SearchRows rows_of(StreamBatch const & b)
{
  return SearchRows{static_cast<int64_t>(b.head.size()), b.head.data(), b.cat.data(), b.off.data(), b.len.data(), b.size.data(),
                    b.res.data(), b.row_first.data(), b.cigar.data(), b.cigar_off.data()};
}

}  // namespace

// The --search_exact command (commands/search_exact.cpp:211-908): the database read whole, masked as printed and indexed
// (vsg_exact_index_create), the queries over run_stream's pipeline, the per-database and OTU-table files at the end.
extern "C" int vsg_search_exact_command(vsg_ctx * ctx, const char * query_path, const char * db_path, const vsg_search_exact_opts * e,
                                        const vsg_search_opts * s, const vsg_search_exact_outputs * outputs,
                                        vsg_search_exact_stats * stats)
{
  char const * const caller = "vsg_search_exact_command";
  if (ctx == nullptr || query_path == nullptr || db_path == nullptr || e == nullptr || s == nullptr || outputs == nullptr) {
    Error::set("vsg_search_exact_command: null argument");
    return VSG_EINVAL;
  }
  vsg_search_exact_outputs const & out = *outputs;
  int rc = search_command_check(caller, e->qmask, e->dbmask, e->hardmask, e->maxhits, *s, out);
  if (rc != VSG_OK) { return rc; }
  if (vsg_udb_detect(db_path) == 1) { Error::set(std::string(caller) + ": a UDB database is not offered: " + db_path); return VSG_EINVAL; }
  auto const t_wall = std::chrono::steady_clock::now();
  vsg_search_exact_stats st{};

  // the database: db.read(..., upcase = 0), its abundances, its mask as printed (DUST only for the files that print it)
  SearchDb db;
  bool const dust_db = (out.dbmatched != nullptr || out.dbnotmatched != nullptr) && e->dbmask == VSG_DBMASK_DUST;
  if ((rc = search_db_read(ctx, caller, db_path, e->notrunclabels != 0, e->minseqlength, e->maxseqlength, e->dbmask, e->hardmask != 0,
                           dust_db, s->self != 0, db)) != VSG_OK) { return rc; }
  st.parse_s = seconds_since(t_wall);
  auto const t_dev = std::chrono::steady_clock::now();
  vsg_exact_index * ixraw = nullptr;
  if ((rc = vsg_exact_index_create(ctx, db.set.get(), &ixraw)) != VSG_OK) { return rc; }
  std::unique_ptr<vsg_exact_index, void (*)(vsg_exact_index *)> ix(ixraw, vsg_exact_index_destroy);
  double const db_device_s = seconds_since(t_dev);

  bool const print_queries = out.matched != nullptr || out.notmatched != nullptr;
  SearchWriterOpts w;
  w.maxhits = e->maxhits;
  w.uc_allhits = e->uc_allhits != 0;
  w.output_no_hits = e->output_no_hits != 0;
  w.sizein = e->sizein != 0;
  w.xsize = e->xsize != 0;
  w.fmt = FastaFormat{nullptr, e->xsize != 0, e->sizeout != 0, e->fasta_width};
  SearchWriter writer(w, out, db.file.head, db.file.cat.data(), db.file.off.data(), db.file.len.data(), db.size.data());
  OutFiles files;
  vsg_stream_stats ss{};
  rc = run_stream(caller, query_path, {out.blast6out, out.uc, out.matched, out.notmatched}, e->notrunclabels != 0,
                  e->batch_queries < 1 ? 65536 : e->batch_queries, false, &ss, [&](StreamBatch & b) {
    vsg_search_opts o;
    std::vector<int64_t> qlabel;
    int r = search_batch_opts(caller, b.head, db, *s, b.size, qlabel, o);
    SeqsetPtr qset;
    if (r == VSG_OK) { r = batch_query_set(ctx, b, e->qmask, e->hardmask != 0, print_queries && e->qmask == VSG_DBMASK_DUST, true, qset); }
    if (r != VSG_OK) { return r; }
    return search_exact_host(ctx, ix.get(), qset.get(), 0, static_cast<int64_t>(b.head.size()), &o, 0, b.res, b.row_first);
  }, [&](StreamBatch const & b, std::vector<std::string> & outs, vsg_stream_stats &) { writer.batch(rows_of(b), outs.data()); },
  &files.made);
  if (rc != VSG_OK) { return rc; }

  auto const t_write = std::chrono::steady_clock::now();
  if (!writer.finish(caller, files)) { return VSG_EINVAL; }
  files.ok = true;
  st.queries = writer.queries;
  st.matched = writer.matched;
  st.queries_abundance = writer.queries_abundance;
  st.matched_abundance = writer.matched_abundance;
  st.hits = writer.hits;
  st.db_sequences = static_cast<int64_t>(db.heads.size());
  st.db_discarded_short = db.file.discarded_short;
  st.db_discarded_long = db.file.discarded_long;
  st.parse_s += ss.parse_s;
  st.device_s = db_device_s + ss.search_s;
  st.write_s = ss.write_s + seconds_since(t_write);
  st.wall_s = seconds_since(t_wall);
  if (stats != nullptr) { *stats = st; }
  return VSG_OK;
}

extern "C" void vsg_usearch_global_opts_default(vsg_usearch_global_opts * u, vsg_search_opts * s)
{
  if (u != nullptr) {
    *u = vsg_usearch_global_opts{};
    u->dbmask = VSG_DBMASK_DUST;
    u->qmask = VSG_DBMASK_DUST;
    u->fasta_width = 80;
    u->minseqlength = 32;   // cli.cc: 32 for --usearch_global (1 for --search_exact)
    u->maxseqlength = 50000;
    u->batch_queries = 65536;
  }
  if (s != nullptr) { vsg_search_opts_default(s); }
}

// The --usearch_global command (commands/usearch_global.cpp:150-373, 537-845): the database read whole (or a UDB file
// loaded), masked and indexed; the queries over run_stream's pipeline with the k-mer search (search_hits_host, every hit
// kept) and the CIGARs of the printed --uc rows on the device; the per-database and OTU-table files at the end.
extern "C" int vsg_usearch_global_command(vsg_ctx * ctx, const char * query_path, const char * db_path, const vsg_usearch_global_opts * u,
                                          const vsg_search_opts * s, const vsg_usearch_global_outputs * outputs,
                                          vsg_usearch_global_stats * stats)
{
  char const * const caller = "vsg_usearch_global_command";
  if (ctx == nullptr || query_path == nullptr || db_path == nullptr || u == nullptr || s == nullptr || outputs == nullptr) {
    Error::set("vsg_usearch_global_command: null argument");
    return VSG_EINVAL;
  }
  vsg_usearch_global_outputs const & out = *outputs;
  int rc = search_command_check(caller, u->qmask, u->dbmask, u->hardmask, u->maxhits, *s, out);
  if (rc != VSG_OK) { return rc; }
  auto const t_wall = std::chrono::steady_clock::now();
  vsg_usearch_global_stats st{};

  // the database and its index (usearch_global.cpp:561-589)
  SearchDb db;
  vsg_index * ixraw = nullptr;
  double db_device_s = 0.0;
  if (vsg_udb_detect(db_path) == 1) {   // udb_read: the file's sequences, headers, mask and word length
    vsg_udb * uraw = nullptr;
    if ((rc = vsg_udb_open(db_path, &uraw)) != VSG_OK) { return rc; }
    std::unique_ptr<vsg_udb, void (*)(vsg_udb *)> udb(uraw, vsg_udb_close);
    int64_t const n = static_cast<int64_t>(udb->len.size());
    db.file.cat = udb->cat;
    db.file.off = udb->off;
    db.file.len = udb->len;
    db.file.head.resize(static_cast<size_t>(n));
    for (int64_t i = 0; i < n; i++) { db.file.head[static_cast<size_t>(i)] = vsg_udb_header(udb.get(), i); }
    if ((rc = search_db_labels(caller, s->self != 0, db)) != VSG_OK) { return rc; }
    st.parse_s = seconds_since(t_wall);
    auto const t_dev = std::chrono::steady_clock::now();
    vsg_seqset * setraw = nullptr;
    if ((rc = vsg_udb_load(ctx, udb.get(), &setraw, &ixraw, nullptr)) != VSG_OK) { return rc; }
    db.set.reset(setraw);
    db_device_s = seconds_since(t_dev);
  } else {
    if ((rc = search_db_read(ctx, caller, db_path, u->notrunclabels != 0, u->minseqlength, u->maxseqlength, u->dbmask, u->hardmask != 0,
                             u->dbmask == VSG_DBMASK_DUST, s->self != 0, db)) != VSG_OK) { return rc; }
    st.parse_s = seconds_since(t_wall);
    auto const t_dev = std::chrono::steady_clock::now();
    if ((rc = vsg_index_create(ctx, db.set.get(), s->wordlength, u->dbmask != VSG_DBMASK_NONE ? 1 : 0, &ixraw)) != VSG_OK) { return rc; }
    db_device_s = seconds_since(t_dev);
  }
  std::unique_ptr<vsg_index, void (*)(vsg_index *)> ix(ixraw, vsg_index_destroy);

  bool const print_queries = out.matched != nullptr || out.notmatched != nullptr;
  SearchWriter writer(usearch_global_writer_opts(*u), out, db.file.head, db.file.cat.data(), db.file.off.data(), db.file.len.data(),
                      db.size.data());
  OutFiles files;
  vsg_stream_stats ss{};
  double cigar_s = 0.0;
  rc = run_stream(caller, query_path, {out.blast6out, out.uc, out.matched, out.notmatched}, u->notrunclabels != 0,
                  u->batch_queries < 1 ? 65536 : u->batch_queries, false, &ss, [&](StreamBatch & b) {
    int64_t const nq = static_cast<int64_t>(b.head.size());
    vsg_search_opts o;
    std::vector<int64_t> qlabel;
    int r = search_batch_opts(caller, b.head, db, *s, b.size, qlabel, o);
    SeqsetPtr qset;
    if (r == VSG_OK) { r = batch_query_set(ctx, b, u->qmask, u->hardmask != 0, u->qmask == VSG_DBMASK_DUST, print_queries, qset); }
    if (r != VSG_OK) { return r; }
    // search_query: the query's k-mers skip lower case unless qmask none; the minus strand is DUST-masked on its own
    o.mask_lower = u->qmask != VSG_DBMASK_NONE ? 1 : 0;
    o.qmask_dust = u->qmask == VSG_DBMASK_DUST ? 1 : 0;
    int64_t work[4] = {0, 0, 0, 0};
    if ((r = search_hits_host(ctx, ix.get(), db.set.get(), qset.get(), 0, nq, &o, 0, b.res, b.row_first, work)) != VSG_OK) { return r; }
    st.pairs += work[2];
    st.cells += work[3];

    // the CIGARs of the --uc rows the writer prints that are not "="
    auto const t_cigar = std::chrono::steady_clock::now();
    b.cigar.assign(1, '\0');
    b.cigar_off.assign(b.res.size(), -1);
    if (out.uc != nullptr) {
      std::vector<uint32_t> pq, pt;
      std::vector<uint8_t> ps;
      std::vector<int64_t> prow;
      for (int64_t q = 0; q < nq; q++) {
        int64_t const f = b.row_first[static_cast<size_t>(q)];
        vsg_search_result const * const h = b.res.data() + f;
        int64_t const k = writer.uc_rows(writer.shown(h, b.row_first[static_cast<size_t>(q) + 1] - f));
        for (int64_t j = 0; j < k; j++) {
          if (h[j].matches == h[j].alignment_length) { continue; }
          pq.push_back(static_cast<uint32_t>(q));
          pt.push_back(static_cast<uint32_t>(h[j].target));
          ps.push_back(h[j].strand != 0 ? 1 : 0);
          prow.push_back(f + j);
        }
      }
      std::vector<int64_t> offs;
      int64_t deferred = -1;
      if (!pq.empty() && (r = strand_cigars(ctx, qset.get(), db.set.get(), pq, pt, ps, b.cigar, offs, deferred)) != VSG_OK) { return r; }
      if (deferred >= 0) {
        Error::set(std::string(caller) + ": the 16-bit aligner defers the alignment of " + b.head[pq[static_cast<size_t>(deferred)]] +
                   " with " + db.file.head[pt[static_cast<size_t>(deferred)]] + ": its CIGAR for --uc cannot come from the fallback callback");
        return VSG_EINVAL;
      }
      for (size_t k = 0; k < offs.size(); k++) { b.cigar_off[static_cast<size_t>(prow[k])] = offs[k]; }
    }
    cigar_s += seconds_since(t_cigar);
    return VSG_OK;
  }, [&](StreamBatch const & b, std::vector<std::string> & outs, vsg_stream_stats &) { writer.batch(rows_of(b), outs.data()); },
  &files.made);
  if (rc != VSG_OK) { return rc; }

  auto const t_write = std::chrono::steady_clock::now();
  if (!writer.finish(caller, files)) { return VSG_EINVAL; }
  files.ok = true;
  st.queries = writer.queries;
  st.matched = writer.matched;
  st.queries_abundance = writer.queries_abundance;
  st.matched_abundance = writer.matched_abundance;
  st.hits = writer.hits;
  st.db_sequences = static_cast<int64_t>(db.heads.size());
  st.db_discarded_short = db.file.discarded_short;
  st.db_discarded_long = db.file.discarded_long;
  st.parse_s += ss.parse_s;
  st.device_s = db_device_s + ss.search_s - cigar_s;
  st.cigar_s = cigar_s;
  st.write_s = ss.write_s + seconds_since(t_write);
  st.wall_s = seconds_since(t_wall);
  if (stats != nullptr) { *stats = st; }
  return VSG_OK;
}
