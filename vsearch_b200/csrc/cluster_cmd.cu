// cluster_cmd.cu — the clustering commands --cluster_fast, --cluster_size, --cluster_smallmem and --cluster_unoise, from a
// FASTA or FASTQ file to the --uc, --centroids and --clusters files.
//
// Replaces cluster() (reference core/cluster.cpp:1140-1430), which all four commands call
// (commands/cluster_{fast,size,smallmem,unoise}.cpp); they differ only in the sort order, the --minsize filter of
// --cluster_unoise, its acceptance rule and the "=" rule of --uc.  In order:
//   db.read(..., upcase = 0)                 (core/db.cpp:229-300)          read_fastx_file, abundance, --minsize
//   dust_all / hardmask_all                  (core/mask.cpp)                on the device / on the host
//   sortbylength / sortbyabundance           (core/db.cpp:433-485)          on the host
//   cluster_core_parallel / _serial          (core/cluster.cpp:877-1115)    vsg_cluster_fast
//   the CIGAR each H record carries                                          vsg_align_pairs, both strands
//   results_show_uc_one, the C records, fasta_print_general, the --clusters files
//                                            (core/results.cpp:274-327, core/cluster.cpp:1258-1423, core/fasta.cpp:482-...)
//                                                                            vsg_cluster_write (host only)
// The device holds only the clustering; parsing, sorting and writing are host work around it.
#include "vsg_internal.h"

#include <algorithm>
#include <cerrno>
#include <charconv>
#include <chrono>
#include <cinttypes>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <string>
#include <unordered_map>
#include <vector>

using namespace vsg;

namespace {

double seconds_since(std::chrono::steady_clock::time_point t0)
{
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

// align_trim (core/searchcore.cpp:357-463): the alignment length without its terminal gap runs
int64_t internal_length(const char * cigar, int64_t aligned)
{
  int64_t const n = static_cast<int64_t>(std::strlen(cigar));
  int64_t q_left = 0, t_left = 0, q_right = 0, t_right = 0;
  if (n > 0) {
    int64_t run = 1, i = 0;
    if (cigar[0] >= '0' && cigar[0] <= '9') { run = std::strtoll(cigar, nullptr, 10); while (cigar[i] >= '0' && cigar[i] <= '9') { i++; } }
    if (cigar[i] == 'D') { q_left = run; } else if (cigar[i] == 'I') { t_left = run; }
    char const op = cigar[n - 1];
    if (op != 'M') {
      int64_t p = n - 1;
      while (p > 0 && cigar[p - 1] <= '9') { p--; }
      run = p < n - 1 ? std::strtoll(cigar + p, nullptr, 10) : 1;
      if (op == 'D') { q_right = run; } else { t_right = run; }
    }
  }
  if (q_left >= aligned) { q_right = 0; }
  if (t_left >= aligned) { t_right = 0; }
  return aligned - q_left - t_left - q_right - t_right;
}

}  // namespace

// header_find_attribute (core/attributes.cpp): the first "(^|;)size=[0-9]+(;|$)" of the label; [start, end) covers
// "size=<digits>"
bool vsg::find_size(const std::string & h, int & start, int & end)
{
  static char const text[] = "size=";
  int const tl = 5;
  int const len = static_cast<int>(h.size());
  int offset = 0;
  while (offset < len - tl) {
    char const * const p = std::strstr(h.c_str() + offset, text);
    if (p == nullptr) { break; }
    offset = static_cast<int>(p - h.c_str());
    if (offset > 0 && h[static_cast<size_t>(offset - 1)] != ';') { offset += tl + 1; continue; }
    int const digits = static_cast<int>(std::strspn(h.c_str() + offset + tl, "0123456789"));
    if (digits == 0) { offset += tl + 1; continue; }
    if (offset + tl + digits < len && h[static_cast<size_t>(offset + tl + digits)] != ';') { offset += tl + digits + 2; continue; }
    start = offset;
    end = offset + tl + digits;
    return true;
  }
  return false;
}

// fastx_get_abundance / header_get_size: 1 without an annotation; zero or out of range is an error
bool vsg::abundance_of(const std::string & h, int64_t & out, std::string & err)
{
  int start = 0, end = 0;
  out = 1;
  if (!find_size(h, start, end)) { return true; }
  errno = 0;
  long long const v = std::strtoll(h.c_str() + start + 5, nullptr, 10);
  if (errno == ERANGE) { err = "Invalid (range error) abundance annotation in FASTA file header"; return false; }
  if (v == 0) { err = "Invalid (zero) abundance annotation in FASTA file header"; return false; }
  out = v;
  return true;
}

// header_fprint_strip (core/attributes.cpp) with only --xsize among the stripped attributes; returns whether the last
// character written is ';'
bool vsg::header_fprint_strip(std::string & out, const std::string & h, bool strip_size)
{
  int const len = static_cast<int>(h.size());
  int start = 0, end = 0;
  int last = -1;
  if (!strip_size || !find_size(h, start, end)) {
    out += h;
    last = len - 1;
  } else {
    if (start > 1) { out.append(h, 0, static_cast<size_t>(start - 1)); last = start - 2; }
    if (len > end + 1) { out.append(h, static_cast<size_t>(end), std::string::npos); last = len - 1; }
  }
  return last >= 0 && h[static_cast<size_t>(last)] == ';';
}

// fasta_print_general (core/fasta.cpp:482-...) with the options the commands offer: a prefix, --relabel (ordinal > 0),
// --xsize / --sizeout, ";seqs=" (seqs > 0), ";clusterid=" (clusterid >= 0), fasta_width, no sequence line (seq NULL)
void vsg::fasta_print_general(std::string & out, const FastaFormat & c, const std::string & head, const char * seq, int64_t len,
                              int64_t abundance, int64_t ordinal, int64_t clusterid, const char * prefix, int64_t seqs)
{
  out += '>';
  if (prefix != nullptr) { out += prefix; }
  bool trailing = false;
  if (c.relabel != nullptr && ordinal > 0) {
    out += c.relabel;
    out += std::to_string(ordinal);
  } else {
    trailing = header_fprint_strip(out, head, c.xsize || (c.sizeout && abundance > 0));
  }
  auto sep = [&] { if (trailing) { trailing = false; } else { out += ';'; } };
  if (seqs > 0) { sep(); out += "seqs="; out += std::to_string(seqs); }
  if (clusterid >= 0) { sep(); out += "clusterid="; out += std::to_string(clusterid); }
  if (c.sizeout && abundance > 0) { sep(); out += "size="; out += std::to_string(abundance); }
  out += '\n';
  if (seq == nullptr) { return; }
  if (c.fasta_width < 1) { out.append(seq, static_cast<size_t>(len)); out += '\n'; return; }
  for (int64_t i = 0; i < len; i += c.fasta_width) {
    out.append(seq + i, static_cast<size_t>(std::min<int64_t>(c.fasta_width, len - i)));
    out += '\n';
  }
}

extern "C" void vsg_cluster_cmd_opts_default(int command, vsg_cluster_cmd_opts * c, vsg_search_opts * s)
{
  if (c != nullptr) {
    *c = vsg_cluster_cmd_opts{};
    c->command = command;
    c->threads = 1;
    c->qmask = VSG_DBMASK_DUST;
    c->fasta_width = 80;
    c->minseqlength = 32;
    c->maxseqlength = 50000;
    c->minsize = command == VSG_CLUSTER_UNOISE ? 8 : 1;
  }
  if (s != nullptr) {
    vsg_search_opts_default(s);
    s->wordlength = 8;
    s->maxrejects = command == VSG_CLUSTER_FAST ? 8 : 32;
    if (command == VSG_CLUSTER_UNOISE) {   // --id is not given: weak_id stays 0.90 (cli.cc, vsearch.cc:206)
      s->id = -1.0;
      s->weak_id = 0.90;
    }
  }
}

namespace {

// the checks and the order both writers share: every result a cluster assignment, the cluster abundances (the sum of
// the members' abundances with --sizein, the member count without, cluster.cpp:1258-1265) and the records by cluster
// (clusterout_sort: cluster abundance descending first), the centroid first in each (cluster.cpp:1290-1320)
int cluster_order(const char * caller, int64_t n, const int64_t * abundances, const vsg_cluster_result * results,
                  const vsg_cluster_cmd_opts * c, std::vector<int64_t> & abundance, std::vector<int64_t> & order)
{
  int64_t nclusters = 0;
  for (int64_t i = 0; i < n; i++) {
    vsg_cluster_result const & r = results[i];
    if (r.cluster < 0 || r.cluster > i || r.centroid >= n || (r.centroid >= 0 && results[r.centroid].cluster != r.cluster)) {
      Error::set(std::string(caller) + ": result " + std::to_string(i) + " is not a cluster assignment");
      return VSG_EINVAL;
    }
    nclusters = std::max<int64_t>(nclusters, r.cluster + 1);
  }
  abundance.assign(static_cast<size_t>(nclusters), 0);
  for (int64_t i = 0; i < n; i++) { abundance[static_cast<size_t>(results[i].cluster)] += c->sizein != 0 ? abundances[i] : 1; }
  order.resize(static_cast<size_t>(n));
  std::iota(order.begin(), order.end(), int64_t{0});
  std::sort(order.begin(), order.end(), [&](int64_t a, int64_t b) {
    int32_t const ca = results[a].cluster, cb = results[b].cluster;
    if (c->clusterout_sort != 0 && abundance[static_cast<size_t>(ca)] != abundance[static_cast<size_t>(cb)]) {
      return abundance[static_cast<size_t>(ca)] > abundance[static_cast<size_t>(cb)];
    }
    if (ca != cb) { return ca < cb; }
    return a < b;
  });
  return VSG_OK;
}

}  // namespace

extern "C" int vsg_cluster_write(int64_t n, const char * const * headers, const char * cat, const int64_t * off, const int32_t * len,
                                 const int64_t * abundances, const vsg_cluster_result * results, const char * cigar_buf,
                                 const int64_t * cigar_off, const vsg_cluster_cmd_opts * c, const char * uc, const char * centroids,
                                 const char * clusters_prefix, int64_t * singletons)
{
  if (c == nullptr || n < 0 || (n > 0 && (headers == nullptr || cat == nullptr || off == nullptr || len == nullptr ||
                                          abundances == nullptr || results == nullptr || cigar_buf == nullptr || cigar_off == nullptr))) {
    Error::set("vsg_cluster_write: null argument");
    return VSG_EINVAL;
  }
  std::vector<std::string> head(headers, headers + n);
  std::vector<int64_t> abundance, order;
  int const rc = cluster_order("vsg_cluster_write", n, abundances, results, c, abundance, order);
  if (rc != VSG_OK) { return rc; }
  if (singletons != nullptr) { *singletons = std::count(abundance.begin(), abundance.end(), int64_t{1}); }

  std::string out_uc, out_cent;
  if (uc != nullptr) {
    char row[96];
    for (int64_t i = 0; i < n; i++) {
      vsg_cluster_result const & r = results[i];
      if (r.centroid < 0) {
        out_uc.append(row, static_cast<size_t>(std::snprintf(row, sizeof row, "S\t%d\t%d\t*\t*\t*\t*\t*\t", r.cluster, len[i])));
        header_fprint_strip(out_uc, head[static_cast<size_t>(i)], c->xsize != 0);
        out_uc += "\t*\n";
        continue;
      }
      char const * const cigar = cigar_buf + cigar_off[i];
      int64_t const columns = c->command == VSG_CLUSTER_FAST ? internal_length(cigar, r.alignment_length) : r.alignment_length;
      out_uc.append(row, static_cast<size_t>(std::snprintf(row, sizeof row, "H\t%d\t%d\t%.1f\t%c\t0\t0\t", r.cluster, len[i], r.id,
                                                          r.strand != 0 ? '-' : '+')));
      if (r.matches == columns) { out_uc += '='; } else { out_uc += cigar; }
      out_uc += '\t';
      header_fprint_strip(out_uc, head[static_cast<size_t>(i)], c->xsize != 0);
      out_uc += '\t';
      header_fprint_strip(out_uc, head[static_cast<size_t>(r.centroid)], c->xsize != 0);
      out_uc += '\n';
    }
  }

  OutFiles files;
  FastaFormat const fmt{c->relabel, c->xsize != 0, c->sizeout != 0, c->fasta_width};
  std::string out_cluster;
  int64_t ordinal = 0;
  char row[96];
  for (size_t k = 0; k < order.size(); k++) {
    int64_t const i = order[k];
    int32_t const cl = results[i].cluster;
    bool const first = k == 0 || results[order[k - 1]].cluster != cl;
    if (first) {
      int64_t const ab = abundance[static_cast<size_t>(cl)];
      if (centroids != nullptr) {
        fasta_print_general(out_cent, fmt, head[static_cast<size_t>(i)], cat + off[i], len[i], ab, cl + 1, c->clusterout_id != 0 ? cl : -1);
      }
      if (uc != nullptr) {
        out_uc.append(row, static_cast<size_t>(std::snprintf(row, sizeof row, "C\t%d\t%" PRId64 "\t*\t*\t*\t*\t*\t", cl, ab)));
        header_fprint_strip(out_uc, head[static_cast<size_t>(i)], c->xsize != 0);
        out_uc += "\t*\n";
      }
      out_cluster.clear();
    }
    if (clusters_prefix != nullptr) {
      // fasta_print_db_relabel: the member's own abundance, its ordinal in the cluster
      ordinal = first ? 1 : ordinal + 1;
      fasta_print_general(out_cluster, fmt, head[static_cast<size_t>(i)], cat + off[i], len[i], abundances[i], ordinal, -1);
      bool const last = k + 1 == order.size() || results[order[k + 1]].cluster != cl;
      if (last && !files.write(std::string(clusters_prefix) + std::to_string(cl), out_cluster)) {
        Error::set(std::string("vsg_cluster_write: unable to write clusters file ") + clusters_prefix + std::to_string(cl));
        return VSG_EINVAL;
      }
    }
  }
  if (uc != nullptr && !files.write(uc, out_uc)) { Error::set(std::string("vsg_cluster_write: cannot write ") + uc); return VSG_EINVAL; }
  if (centroids != nullptr && !files.write(centroids, out_cent)) {
    Error::set(std::string("vsg_cluster_write: cannot write ") + centroids);
    return VSG_EINVAL;
  }
  files.ok = true;
  return VSG_OK;
}

namespace {

// one --msaout row (compute_and_print_msa, core/msa.cpp): the member's symbols (`seq`, already oriented) in the
// columns its CIGAR gives against the centroid's insertion blocks `ins`; false when the two do not agree
bool msa_row(std::string & row, const char * cigar, const char * seq, int64_t slen, const int32_t * ins, int64_t clen)
{
  int64_t q = 0, t = 0;
  bool inserted = false;
  auto block = [&]() { if (!inserted) { row.append(static_cast<size_t>(ins[q]), '-'); } };
  for (char const * p = cigar; *p != '\0';) {
    int64_t run = 1;
    if (*p >= '0' && *p <= '9') { run = std::strtoll(p, const_cast<char **>(&p), 10); }
    char const op = *p++;
    if (op == 'D') {
      if (q > clen || run > ins[q] || t + run > slen) { return false; }
      row.append(seq + t, static_cast<size_t>(run));
      row.append(static_cast<size_t>(ins[q] - run), '-');
      t += run;
      inserted = true;
    } else if (op == 'M' || op == 'I') {
      if (q + run > clen || (op == 'M' && t + run > slen)) { return false; }
      for (int64_t k = 0; k < run; k++) {
        block();
        row += op == 'M' ? seq[t++] : '-';
        q++;
        inserted = false;
      }
    } else {
      return false;
    }
  }
  if (q != clen || t != slen) { return false; }
  block();
  return true;
}

}  // namespace

extern "C" int vsg_cluster_msa_write(int64_t n, const char * const * headers, const char * cat, const int64_t * off, const int32_t * len,
                                     const int64_t * abundances, const vsg_cluster_result * results, const char * cigar_buf,
                                     const int64_t * cigar_off, const int32_t * insertions, const int64_t * col_first,
                                     const uint64_t * profile, const char * consensus, const vsg_cluster_cmd_opts * c,
                                     const char * msaout, const char * consout, const char * profile_path)
{
  char const * const caller = "vsg_cluster_msa_write";
  if (c == nullptr || n < 0 || (n > 0 && (headers == nullptr || cat == nullptr || off == nullptr || len == nullptr || abundances == nullptr ||
                                          results == nullptr || cigar_buf == nullptr || cigar_off == nullptr || insertions == nullptr ||
                                          col_first == nullptr || profile == nullptr || consensus == nullptr))) {
    Error::set("vsg_cluster_msa_write: null argument");
    return VSG_EINVAL;
  }
  std::vector<int64_t> abundance, order;
  int const rc = cluster_order(caller, n, abundances, results, c, abundance, order);
  if (rc != VSG_OK) { return rc; }
  int64_t const nclusters = static_cast<int64_t>(abundance.size());
  // each cluster's insertion blocks, in cluster-number order; its width must be the centroid plus its blocks
  std::vector<int64_t> ifirst(static_cast<size_t>(nclusters) + 1, 0);
  for (int64_t i = 0; i < n; i++) {
    if (results[i].centroid < 0) { ifirst[static_cast<size_t>(results[i].cluster) + 1] = len[i] + 1; }
  }
  for (int64_t cl = 0; cl < nclusters; cl++) {
    int64_t const nb = ifirst[static_cast<size_t>(cl) + 1];
    ifirst[static_cast<size_t>(cl) + 1] += ifirst[static_cast<size_t>(cl)];
    int64_t w = nb - 1;
    for (int64_t p = 0; p < nb; p++) { w += insertions[ifirst[static_cast<size_t>(cl)] + p]; }
    if (nb == 0 || col_first[cl + 1] - col_first[cl] != w) {
      Error::set("vsg_cluster_msa_write: the columns of cluster " + std::to_string(cl) + " do not match its insertions");
      return VSG_EINVAL;
    }
  }

  OutFiles files;
  std::FILE * fp[3] = {nullptr, nullptr, nullptr};
  char const * const path[3] = {msaout, consout, profile_path};
  auto close_all = [&]() {
    bool ok = true;
    for (std::FILE *& f : fp) { if (f != nullptr) { ok = std::fclose(f) == 0 && ok; f = nullptr; } }
    return ok;
  };
  for (int k = 0; k < 3; k++) {
    if (path[k] != nullptr && (fp[k] = files.open(path[k])) == nullptr) {
      close_all();
      Error::set(std::string("vsg_cluster_msa_write: cannot write ") + path[k]);
      return VSG_EINVAL;
    }
  }
  FastaFormat const fmt{c->relabel, c->xsize != 0, c->sizeout != 0, c->fasta_width};
  static Complement const comp;
  std::string out, row, rc_seq;
  char num[24];
  for (size_t k = 0; k < order.size();) {
    int32_t const cl = results[order[k]].cluster;
    size_t k1 = k;
    while (k1 < order.size() && results[order[k1]].cluster == cl) { k1++; }
    int64_t const cent = order[k];
    std::string const head(headers[cent]);
    int64_t const width = col_first[cl + 1] - col_first[cl];
    int32_t const * const ins = insertions + ifirst[static_cast<size_t>(cl)];
    char const * const cons = consensus + col_first[cl];
    uint64_t const * const prof = profile + col_first[cl] * 6;
    int64_t const members = static_cast<int64_t>(k1 - k);
    int64_t const ab = abundance[static_cast<size_t>(cl)];
    int64_t const clusterid = c->clusterout_id != 0 ? cl : -1;
    if (fp[0] != nullptr) {
      out.assign(1, '\n');
      for (size_t m = k; m < k1; m++) {
        int64_t const i = order[m];
        row.clear();
        if (m == k) {
          for (int64_t p = 0; p < len[i]; p++) { row.append(static_cast<size_t>(ins[p]), '-'); row += cat[off[i] + p]; }
          row.append(static_cast<size_t>(ins[len[i]]), '-');
        } else {
          char const * seq = cat + off[i];
          if (results[i].strand != 0) {
            rc_seq.resize(static_cast<size_t>(len[i]));
            for (int64_t p = 0; p < len[i]; p++) { rc_seq[static_cast<size_t>(p)] = comp.map[static_cast<unsigned char>(seq[len[i] - 1 - p])]; }
            seq = rc_seq.data();
          }
          if (!msa_row(row, cigar_buf + cigar_off[i], seq, len[i], ins, len[cent])) {
            close_all();
            Error::set("vsg_cluster_msa_write: the CIGAR of record " + std::to_string(i) + " does not match its cluster's insertions");
            return VSG_EINVAL;
          }
        }
        if (static_cast<int64_t>(row.size()) != width) {
          close_all();
          Error::set("vsg_cluster_msa_write: the row of record " + std::to_string(i) + " does not fill its cluster's columns");
          return VSG_EINVAL;
        }
        fasta_print_general(out, fmt, headers[i], row.data(), width, abundances[i], 0, -1, m == k ? "*" : nullptr);
      }
      fasta_print_general(out, fmt, "consensus", cons, width, 0, 0, -1);
      if (std::fwrite(out.data(), 1, out.size(), fp[0]) != out.size()) { break; }
    }
    if (fp[1] != nullptr) {
      row.clear();
      for (int64_t p = 0; p < width; p++) { if (cons[p] != '+' && cons[p] != '-') { row += cons[p]; } }
      out.clear();
      fasta_print_general(out, fmt, head, row.data(), static_cast<int64_t>(row.size()), ab, cl + 1, clusterid, "centroid=", members);
      if (std::fwrite(out.data(), 1, out.size(), fp[1]) != out.size()) { break; }
    }
    if (fp[2] != nullptr) {
      // print_alignment_profile: A, C, G, T, then gap before N
      out.clear();
      fasta_print_general(out, fmt, head, nullptr, 0, ab, cl + 1, clusterid, "centroid=", members);
      for (int64_t p = 0; p < width; p++) {
        out += std::to_string(p);
        out += '\t';
        out += cons[p];
        for (int const s : {0, 1, 2, 3, 5, 4}) {
          out += '\t';
          out.append(num, static_cast<size_t>(std::to_chars(num, num + sizeof num, prof[p * 6 + s]).ptr - num));
        }
        out += '\n';
      }
      out += '\n';
      if (std::fwrite(out.data(), 1, out.size(), fp[2]) != out.size()) { break; }
    }
    k = k1;
  }
  bool const ok = !(fp[0] != nullptr && std::ferror(fp[0])) && !(fp[1] != nullptr && std::ferror(fp[1])) &&
                  !(fp[2] != nullptr && std::ferror(fp[2]));
  if (!close_all() || !ok) { Error::set("vsg_cluster_msa_write: a write failed"); return VSG_EINVAL; }
  files.ok = true;
  return VSG_OK;
}

extern "C" int vsg_cluster_command(vsg_ctx * ctx, const char * input_path, const vsg_cluster_cmd_opts * c, const vsg_search_opts * s,
                                   const char * uc, const char * centroids, const char * clusters_prefix, vsg_cluster_cmd_stats * stats)
{
  vsg_cluster_cmd_outputs const outputs{uc, centroids, clusters_prefix, nullptr, nullptr, nullptr};
  return vsg_cluster_command_outputs(ctx, input_path, c, s, &outputs, stats);
}

extern "C" int vsg_cluster_command_outputs(vsg_ctx * ctx, const char * input_path, const vsg_cluster_cmd_opts * c, const vsg_search_opts * s,
                                           const vsg_cluster_cmd_outputs * outputs, vsg_cluster_cmd_stats * stats)
{
  char const * const caller = "vsg_cluster_command";
  if (outputs == nullptr) { Error::set("vsg_cluster_command: null argument"); return VSG_EINVAL; }
  char const * const uc = outputs->uc, * const centroids = outputs->centroids, * const clusters_prefix = outputs->clusters_prefix;
  bool const msa = outputs->msaout != nullptr || outputs->consout != nullptr || outputs->profile != nullptr;
  static const bool trace = std::getenv("VSG_TRACE") != nullptr;
  double msa_device_s = 0, msa_write_s = 0;
  if (ctx == nullptr || input_path == nullptr || c == nullptr || s == nullptr) { Error::set("vsg_cluster_command: null argument"); return VSG_EINVAL; }
  if (c->command < VSG_CLUSTER_FAST || c->command > VSG_CLUSTER_UNOISE) { Error::set("vsg_cluster_command: unknown command"); return VSG_EINVAL; }
  if (c->qmask < VSG_DBMASK_NONE || c->qmask > VSG_DBMASK_DUST) { Error::set("vsg_cluster_command: unknown qmask"); return VSG_EINVAL; }
  if (c->qmask == VSG_DBMASK_DUST && c->hardmask != 0) {
    Error::set("vsg_cluster_command: --qmask dust with --hardmask is not offered (DUST-masked symbols would become 'N')");
    return VSG_EINVAL;
  }
  if (s->wordlength < 3 || s->wordlength > 10) {
    Error::set("vsg_cluster_command: the device's cluster index supports --wordlength 3..10");
    return VSG_EINVAL;
  }
  if (c->threads < 1) { Error::set("vsg_cluster_command: threads must be at least 1"); return VSG_EINVAL; }
  if (s->query_sizes != nullptr || s->target_sizes != nullptr || s->query_labels != nullptr || s->target_labels != nullptr) {
    Error::set("vsg_cluster_command: the size and label arrays of the search options are the command's own: pass them NULL");
    return VSG_EINVAL;
  }
  auto const t_wall = std::chrono::steady_clock::now();
  vsg_cluster_cmd_stats st{};

  // read: db.read(..., upcase = 0) with the --minsize filter of --cluster_unoise (core/db.cpp:262-294)
  FastxFile in;
  int rc = read_fastx_file(caller, input_path, c->notrunclabels != 0, c->minseqlength, c->maxseqlength, in);
  if (rc != VSG_OK) { return rc; }
  std::vector<int64_t> keep, ab;
  keep.reserve(in.head.size());
  ab.reserve(in.head.size());
  for (size_t i = 0; i < in.head.size(); i++) {
    int64_t a = 1;
    std::string err;
    if (!abundance_of(in.head[i], a, err)) { Error::set(std::string(caller) + ": " + err + " (" + in.head[i] + ")"); return VSG_EINVAL; }
    if (c->command == VSG_CLUSTER_UNOISE && a < c->minsize) { st.discarded_minsize++; continue; }
    keep.push_back(static_cast<int64_t>(i));
    ab.push_back(a);
  }
  int64_t const n = static_cast<int64_t>(keep.size());
  if (n > 0x7fffffff) { Error::set("vsg_cluster_command: too many sequences"); return VSG_EINVAL; }
  st.parse_s = seconds_since(t_wall);

  // sort (core/db.cpp:433-485); order[k] = the position in `keep` of the k-th record processed
  auto const t_sort = std::chrono::steady_clock::now();
  std::vector<int64_t> order(static_cast<size_t>(n));
  std::iota(order.begin(), order.end(), int64_t{0});
  auto len_of = [&](int64_t k) { return in.len[static_cast<size_t>(keep[static_cast<size_t>(k)])]; };
  auto head_of = [&](int64_t k) -> const std::string & { return in.head[static_cast<size_t>(keep[static_cast<size_t>(k)])]; };
  if (c->command == VSG_CLUSTER_FAST) {
    std::sort(order.begin(), order.end(), [&](int64_t a, int64_t b) {
      if (len_of(a) != len_of(b)) { return len_of(a) > len_of(b); }
      if (ab[static_cast<size_t>(a)] != ab[static_cast<size_t>(b)]) { return ab[static_cast<size_t>(a)] > ab[static_cast<size_t>(b)]; }
      int const o = std::strcmp(head_of(a).c_str(), head_of(b).c_str());
      return o != 0 ? o < 0 : a < b;
    });
  } else if (c->command != VSG_CLUSTER_SMALLMEM) {
    std::sort(order.begin(), order.end(), [&](int64_t a, int64_t b) {
      if (ab[static_cast<size_t>(a)] != ab[static_cast<size_t>(b)]) { return ab[static_cast<size_t>(a)] > ab[static_cast<size_t>(b)]; }
      int const o = std::strcmp(head_of(a).c_str(), head_of(b).c_str());
      return o != 0 ? o < 0 : a < b;
    });
  } else if (c->usersort == 0) {
    for (int64_t k = 1; k < n; k++) {
      if (len_of(k) > len_of(k - 1)) {
        Error::set("vsg_cluster_command: Sequences not sorted by length and --usersort not specified.");
        return VSG_EINVAL;
      }
    }
  }
  // the records in processing order: sequences as printed (soft + hardmask: lower case to 'N', hardmask_all)
  std::vector<char> cat;
  std::vector<int64_t> off(static_cast<size_t>(n)), abundance(static_cast<size_t>(n));
  std::vector<int32_t> len(static_cast<size_t>(n));
  std::vector<const char *> heads(static_cast<size_t>(n));
  for (int64_t k = 0; k < n; k++) {
    int64_t const r = keep[static_cast<size_t>(order[static_cast<size_t>(k)])];
    off[static_cast<size_t>(k)] = static_cast<int64_t>(cat.size());
    len[static_cast<size_t>(k)] = in.len[static_cast<size_t>(r)];
    abundance[static_cast<size_t>(k)] = ab[static_cast<size_t>(order[static_cast<size_t>(k)])];
    heads[static_cast<size_t>(k)] = in.head[static_cast<size_t>(r)].c_str();
    cat.insert(cat.end(), in.cat.begin() + in.off[static_cast<size_t>(r)], in.cat.begin() + in.off[static_cast<size_t>(r)] + in.len[static_cast<size_t>(r)]);
    st.nucleotides += in.len[static_cast<size_t>(r)];
  }
  if (c->qmask == VSG_DBMASK_SOFT && c->hardmask != 0) {
    for (char & ch : cat) { if ((static_cast<unsigned char>(ch) & 0x20) != 0) { ch = 'N'; } }
  }
  cat.push_back('\0');
  st.sort_s = seconds_since(t_sort);

  std::vector<vsg_cluster_result> res(static_cast<size_t>(n));
  std::vector<int32_t> msa_ins;
  std::vector<int64_t> msa_first(1, 0);
  std::vector<uint64_t> msa_prof;
  std::vector<char> msa_cons;
  std::vector<char> cigars(1, '\0');
  std::vector<int64_t> cigar_off(static_cast<size_t>(n), 0);
  if (n > 0) {
    // device: the set, its mask, the clustering
    auto const t_dev = std::chrono::steady_clock::now();
    vsg_seqset * raw = nullptr;
    if ((rc = vsg_seqset_create(ctx, cat.data(), off.data(), len.data(), n, 1, &raw)) != VSG_OK) { return rc; }
    SeqsetPtr set(raw);
    if (c->qmask == VSG_DBMASK_DUST && (rc = vsg_seqset_dust(ctx, set.get())) != VSG_OK) { return rc; }
    vsg_search_opts o = *s;
    o.mask_lower = c->qmask != VSG_DBMASK_NONE ? 1 : 0;
    o.unoise = c->command == VSG_CLUSTER_UNOISE ? 1 : 0;
    o.target_sizes = abundance.data();
    std::vector<int64_t> label_id;
    if (o.self != 0) {
      std::unordered_map<std::string, int64_t> ids;
      label_id.resize(static_cast<size_t>(n));
      for (int64_t k = 0; k < n; k++) { label_id[static_cast<size_t>(k)] = ids.emplace(heads[static_cast<size_t>(k)], k).first->second; }
      o.target_labels = label_id.data();
    }
    int64_t nclusters = 0, work[2] = {0, 0};
    if ((rc = vsg_cluster_fast(ctx, set.get(), &o, c->threads, res.data(), &nclusters, work)) != VSG_OK) { return rc; }
    st.pairs = work[0];
    st.cells = work[1];
    st.device_s = seconds_since(t_dev);

    // the CIGARs of the H records: plus-strand members against the set, minus-strand ones as reverse complements
    auto const t_cigar = std::chrono::steady_clock::now();
    std::vector<uint32_t> q, t;
    std::vector<uint8_t> strand;
    for (int64_t k = 0; k < n; k++) {
      vsg_cluster_result const & r = res[static_cast<size_t>(k)];
      if (r.centroid < 0) { continue; }
      q.push_back(static_cast<uint32_t>(k));
      t.push_back(static_cast<uint32_t>(r.centroid));
      strand.push_back(r.strand != 0 ? 1 : 0);
    }
    std::vector<int64_t> offs;
    int64_t deferred = -1;
    if (!q.empty() && (rc = strand_cigars(ctx, set.get(), set.get(), q, t, strand, cigars, offs, deferred)) != VSG_OK) { return rc; }
    if (deferred >= 0) {
      Error::set(std::string("vsg_cluster_command: the 16-bit aligner defers the alignment of ") + heads[q[static_cast<size_t>(deferred)]] +
                 " with its centroid " + heads[t[static_cast<size_t>(deferred)]] + ": its CIGAR for --uc cannot come from the fallback callback");
      return VSG_EINVAL;
    }
    for (size_t j = 0; j < q.size(); j++) { cigar_off[q[j]] = offs[j]; }
    // the printed case is the device's (DUST), the letters the input's: 'U' and IUPAC codes print as read
    if (c->qmask == VSG_DBMASK_DUST) {
      std::vector<uint8_t> sym(cat.size());
      if ((rc = vsg_seqset_symbols(ctx, set.get(), sym.data(), static_cast<int64_t>(sym.size()))) != VSG_OK) { return rc; }
      for (size_t i = 0; i + 1 < cat.size(); i++) {
        unsigned char const ch = static_cast<unsigned char>(cat[i]);
        cat[i] = static_cast<char>((sym[i] & 0x10) != 0 ? (ch | 0x20) : (ch >= 'a' && ch <= 'z' ? ch & ~0x20 : ch));
      }
    }
    st.cigar_s = seconds_since(t_cigar);
    st.clusters = nclusters;

    // the profile and consensus of every cluster: a first call sizes the columns (VSG_ECAP)
    if (msa) {
      auto const t_msa = std::chrono::steady_clock::now();
      std::vector<uint64_t> weight(static_cast<size_t>(n));
      int64_t nins = 0;
      for (int64_t k = 0; k < n; k++) {
        weight[static_cast<size_t>(k)] = c->sizein != 0 ? static_cast<uint64_t>(abundance[static_cast<size_t>(k)]) : 1;
        if (res[static_cast<size_t>(k)].centroid < 0) { nins += len[static_cast<size_t>(k)] + 1; }
      }
      msa_ins.resize(static_cast<size_t>(nins));
      msa_first.resize(static_cast<size_t>(nclusters) + 1);
      int64_t ncols = 0;
      rc = vsg_cluster_msa(ctx, set.get(), n, res.data(), weight.data(), cigars.data(), cigar_off.data(), msa_ins.data(),
                           msa_first.data(), nullptr, nullptr, 0, &ncols);
      if (rc == VSG_ECAP) {
        msa_prof.resize(static_cast<size_t>(ncols) * 6);
        msa_cons.resize(static_cast<size_t>(ncols));
        rc = vsg_cluster_msa(ctx, set.get(), n, res.data(), weight.data(), cigars.data(), cigar_off.data(), msa_ins.data(),
                             msa_first.data(), msa_prof.data(), msa_cons.data(), ncols, &ncols);
      }
      if (rc != VSG_OK) { return rc; }
      msa_device_s = seconds_since(t_msa);
    }
  }

  auto const t_write = std::chrono::steady_clock::now();
  // the consensus files first: if the cluster files then fail, these are removed too
  if (msa) {
    rc = vsg_cluster_msa_write(n, heads.data(), cat.data(), off.data(), len.data(), abundance.data(), res.data(), cigars.data(),
                               cigar_off.data(), msa_ins.data(), msa_first.data(), msa_prof.data(), msa_cons.data(), c,
                               outputs->msaout, outputs->consout, outputs->profile);
    if (rc != VSG_OK) { return rc; }
    msa_write_s = seconds_since(t_write);
  }
  rc = vsg_cluster_write(n, heads.data(), cat.data(), off.data(), len.data(), abundance.data(), res.data(), cigars.data(),
                         cigar_off.data(), c, uc, centroids, clusters_prefix, &st.singletons);
  if (rc != VSG_OK) {
    for (char const * p : {outputs->msaout, outputs->consout, outputs->profile}) { if (p != nullptr) { std::remove(p); } }
    return rc;
  }
  st.write_s = seconds_since(t_write);
  if (trace && msa) {
    std::fprintf(stderr, "[vsg] cluster_command: msa device %.3f s, msa write %.3f s, %zu columns\n", msa_device_s, msa_write_s,
                 msa_cons.size());
  }
  st.sequences = n;
  st.discarded_short = in.discarded_short;
  st.discarded_long = in.discarded_long;
  st.wall_s = seconds_since(t_wall);
  if (stats != nullptr) { *stats = st; }
  return VSG_OK;
}
