// udb.cu — UDB database files (SURVEY.md §8 f3): the sequences, headers and the stored word index of a file written
// by `vsearch --makeudb_usearch`, and a device-resident database made from it.
//
// Replaces
//   udb_detect_isudb   (reference core/udb.cpp:120-175)   first word == 'UDBF'
//   udb_read           (core/udb.cpp:196-578)             file -> Database + Dbindex
// The file (little endian, the only byte order the reference supports, udb.cpp:89-91) is
//   50 words   header: [0]=0x55444246 [2]=32 [4]=wordlength [6]=dbaccel [13]=seqcount [17]=0x0000746e [49]=0x55444266
//   4^k words  kmercount[]: number of sequences holding each word
//   1 word     0x55444233
//   sum words  kmerindex[]: per word, the ascending numbers of those sequences
//   8 words    [0]=0x55444234 [1]=0x005e0db3 [2]=seqcount [3..4]=nucleotides [5..6]=header characters [7]=0x005e0db4
//   seqcount   offsets of the NUL-terminated headers inside the header block
//   headers, seqcount sequence lengths, the sequences back to back (ASCII, case = masking as it was when the file was made)
// and every check udb_read makes is made here (same order, same "Invalid UDB file" outcome, as an error code).
//
// The reader is host code (no CUDA call): tests run it without a GPU.  vsg_udb_load uploads the sequences and builds
// the DEVICE index from them at the file's word length — 6 ms for 100 000 x 1 500 nt, less than reading the stored
// lists would take — and then proves it equal to the stored one: per word, the number of sequences holding it must
// equal kmercount[].  That comparison also decides what the reference cannot know from the file alone, whether the
// index was built with masked (lower-case) symbols excluded (--dbmask dust/soft) or not (--dbmask none): the index is
// built with lower case excluded first and, if the counts differ, with it included; a file whose counts match neither
// is rejected.  (Both candidates come from the same sequences and the first is a subset of the second word by word,
// so equal counts mean equal lists.)
#include "vsg_internal.h"

#include <sys/stat.h>

#include <cstdio>
#include <cstring>
#include <limits>

using namespace vsg;

namespace vsg {
int index_create_counts(vsg_ctx * c, const vsg_seqset * db, int wordlength, int mask_lower, uint32_t * d_totals, vsg_index ** out);
}

namespace {

constexpr uint32_t UDB_MAGIC = 0x55444246u;   // "FBDU" on disk, udb.cpp:127

struct File {
  std::FILE * f = nullptr;
  ~File() { if (f != nullptr) { std::fclose(f); } }
};

bool read_exact(std::FILE * f, void * buf, uint64_t n, uint64_t & pos)
{
  // blocks of 16 MiB as largeread does (udb.cpp:82-117); fread itself has no such limit, the bound keeps one
  // call's size_t arithmetic away from 32-bit edges
  uint64_t done = 0;
  while (done < n) {
    uint64_t const rem = std::min<uint64_t>(n - done, 4096ull * 4096ull);
    if (std::fread(static_cast<char *>(buf) + done, 1, static_cast<size_t>(rem), f) != rem) { return false; }
    done += rem;
  }
  pos += n;
  return true;
}

int invalid(const char * what)
{
  Error::set(std::string("vsg_udb_open: Invalid UDB file (") + what + ")");
  return VSG_EINVAL;
}

}  // namespace

extern "C" int vsg_udb_detect(const char * path)
{
  if (path == nullptr) { Error::set("vsg_udb_detect: null argument"); return VSG_EINVAL; }
  struct stat fs;
  if (stat(path, &fs) != 0) { Error::set(std::string("vsg_udb_detect: unable to get status for input file (") + path + ")"); return VSG_EINVAL; }
  if (S_ISFIFO(fs.st_mode)) { return 0; }   // pipes are never UDB files (udb.cpp:136-142)
  File in;
  in.f = std::fopen(path, "rb");
  if (in.f == nullptr) { Error::set(std::string("vsg_udb_detect: cannot open ") + path); return VSG_EINVAL; }
  uint32_t magic = 0;
  size_t const got = std::fread(&magic, 1, sizeof magic, in.f);
  return (got == sizeof magic && magic == UDB_MAGIC) ? 1 : 0;
}

extern "C" int vsg_udb_open(const char * path, vsg_udb ** out)
{
  if (path == nullptr || out == nullptr) { Error::set("vsg_udb_open: null argument"); return VSG_EINVAL; }
  *out = nullptr;
  struct stat fs;
  if (stat(path, &fs) != 0) { Error::set(std::string("vsg_udb_open: unable to get status for input file (") + path + ")"); return VSG_EINVAL; }
  if (S_ISFIFO(fs.st_mode)) { Error::set("vsg_udb_open: cannot read UDB file from a pipe"); return VSG_EINVAL; }
  uint64_t const filesize = static_cast<uint64_t>(fs.st_size);
  File in;
  in.f = std::fopen(path, "rb");
  if (in.f == nullptr) { Error::set("vsg_udb_open: unable to open UDB file for reading"); return VSG_EINVAL; }
  std::unique_ptr<vsg_udb> u(new (std::nothrow) vsg_udb());
  if (!u) { Error::set("out of host memory"); return VSG_ENOMEM; }
  uint64_t pos = 0;
  uint32_t buffer[50];

  // header (udb.cpp:256-268)
  if (!read_exact(in.f, buffer, 4 * 50, pos)) { return invalid("truncated header"); }
  if (buffer[0] != UDB_MAGIC || buffer[2] != 32 || buffer[4] < 3 || buffer[4] > 15 || buffer[13] == 0 ||
      buffer[17] != 0x0000746eu || buffer[49] != 0x55444266u) { return invalid("header"); }
  uint32_t const k = buffer[4];
  uint32_t const seqcount = buffer[13];
  u->info.wordlength = static_cast<int32_t>(k);
  u->info.dbaccel = static_cast<int32_t>(buffer[6]);
  u->info.sequences = seqcount;
  if (seqcount > filesize / 4) { return invalid("sequence count"); }   // udb.cpp:279-282

  // word match counts (udb.cpp:296-321)
  uint64_t const hashsize = 1ull << (2 * k);
  if (4 * hashsize > filesize) { return invalid("word count table"); }
  u->kmercount.resize(static_cast<size_t>(hashsize));
  if (!read_exact(in.f, u->kmercount.data(), 4 * hashsize, pos)) { return invalid("truncated word counts"); }
  uint64_t indexsize = 0;
  for (uint64_t i = 0; i < hashsize; i++) {
    indexsize += u->kmercount[static_cast<size_t>(i)];   // cannot wrap: 2^30 terms below 2^32
  }
  if (indexsize > filesize / 4) { return invalid("word counts exceed the file"); }
  u->info.index_entries = static_cast<int64_t>(indexsize);

  // signature, then the sequence numbers of every word (udb.cpp:323-350)
  if (!read_exact(in.f, buffer, 4, pos) || buffer[0] != 0x55444233u) { return invalid("index signature"); }
  u->kmerindex.resize(static_cast<size_t>(indexsize));
  if (!read_exact(in.f, u->kmerindex.data(), 4 * indexsize, pos)) { return invalid("truncated word index"); }
  for (uint64_t i = 0; i < indexsize; i++) {
    if (u->kmerindex[static_cast<size_t>(i)] >= seqcount) { return invalid("sequence number in the word index"); }
  }

  // second header (udb.cpp:352-365)
  if (!read_exact(in.f, buffer, 4 * 8, pos)) { return invalid("truncated second header"); }
  if (buffer[0] != 0x55444234u || buffer[1] != 0x005e0db3u || buffer[2] != seqcount || buffer[7] != 0x005e0db4u) { return invalid("second header"); }
  uint64_t const nucleotides = (static_cast<uint64_t>(buffer[4]) << 32) | buffer[3];
  uint64_t const headerchars = (static_cast<uint64_t>(buffer[6]) << 32) | buffer[5];
  if (nucleotides > filesize || headerchars > filesize) { return invalid("sizes in the second header"); }
  u->info.nucleotides = static_cast<int64_t>(nucleotides);
  u->info.header_chars = static_cast<int64_t>(headerchars);

  // header index (udb.cpp:375-403): strictly increasing offsets inside the header block
  u->header_off.resize(static_cast<size_t>(seqcount) + 1);
  if (!read_exact(in.f, u->header_off.data(), 4ull * seqcount, pos)) { return invalid("truncated header index"); }
  u->header_off[seqcount] = static_cast<uint32_t>(headerchars);
  uint32_t last = 0;
  int64_t longestheader = 0;
  for (uint32_t i = 0; i < seqcount; i++) {
    uint32_t const cur = u->header_off[i];
    if (cur < last || cur >= headerchars) { return invalid("header offset"); }
    if (u->header_off[i + 1] <= cur) { return invalid("header offsets do not increase"); }
    int64_t const hl = static_cast<int64_t>(u->header_off[i + 1]) - cur - 1;
    if (hl > std::numeric_limits<int>::max() - 16) { Error::set("vsg_udb_open: UDB file contains a header too long"); return VSG_EINVAL; }
    longestheader = std::max(longestheader, hl);
    last = cur;
  }
  u->info.longest_header = longestheader;

  // headers (udb.cpp:408)
  u->headers.resize(static_cast<size_t>(headerchars) + 1);
  if (!read_exact(in.f, u->headers.data(), headerchars, pos)) { return invalid("truncated headers"); }
  u->headers[static_cast<size_t>(headerchars)] = '\0';
  for (uint32_t i = 0; i < seqcount; i++) {
    // every header must end inside its own slot (the reference trusts the NUL; a missing one would run into the next header)
    u->headers[u->header_off[i + 1] - 1] = '\0';
  }

  // sequence lengths (udb.cpp:417-452)
  std::vector<uint32_t> lens(seqcount);
  if (!read_exact(in.f, lens.data(), 4ull * seqcount, pos)) { return invalid("truncated sequence lengths"); }
  u->off.resize(seqcount);
  u->len.resize(seqcount);
  uint64_t sum = 0;
  uint32_t shortest = std::numeric_limits<uint32_t>::max(), longest = 0;
  for (uint32_t i = 0; i < seqcount; i++) {
    uint32_t const l = lens[i];
    if (static_cast<int64_t>(l) > std::numeric_limits<int>::max() - 16) { Error::set("vsg_udb_open: UDB file contains a sequence too long"); return VSG_EINVAL; }
    u->off[i] = static_cast<int64_t>(sum);
    u->len[i] = static_cast<int32_t>(l);
    shortest = std::min(shortest, l);
    longest = std::max(longest, l);
    sum += l;
    if (sum > nucleotides) { return invalid("sequence lengths exceed the nucleotide count"); }
  }
  if (sum != nucleotides) { return invalid("sequence lengths do not add up"); }
  u->info.shortest = static_cast<int32_t>(shortest);
  u->info.longest = static_cast<int32_t>(longest);

  // sequences (udb.cpp:455-462)
  u->cat.resize(static_cast<size_t>(nucleotides) + 1);
  if (!read_exact(in.f, u->cat.data(), nucleotides, pos)) { return invalid("truncated sequences"); }
  u->cat[static_cast<size_t>(nucleotides)] = '\0';
  if (pos != filesize) { Error::set("vsg_udb_open: Incorrect UDB file size"); return VSG_EINVAL; }
  *out = u.release();
  return VSG_OK;
}

extern "C" void vsg_udb_close(vsg_udb * u) { delete u; }

extern "C" int vsg_udb_info_get(const vsg_udb * u, vsg_udb_info * out)
{
  if (u == nullptr || out == nullptr) { Error::set("vsg_udb_info_get: null argument"); return VSG_EINVAL; }
  *out = u->info;
  return VSG_OK;
}

extern "C" int vsg_udb_sequences(const vsg_udb * u, const char ** cat, const int64_t ** off, const int32_t ** len)
{
  if (u == nullptr || cat == nullptr || off == nullptr || len == nullptr) { Error::set("vsg_udb_sequences: null argument"); return VSG_EINVAL; }
  *cat = u->cat.data(); *off = u->off.data(); *len = u->len.data();
  return VSG_OK;
}

extern "C" const char * vsg_udb_header(const vsg_udb * u, int64_t i)
{
  if (u == nullptr || i < 0 || i >= u->info.sequences) { return nullptr; }
  return u->headers.data() + u->header_off[static_cast<size_t>(i)];
}

extern "C" int vsg_udb_words(const vsg_udb * u, const uint32_t ** kmercount, const uint32_t ** kmerindex)
{
  if (u == nullptr || kmercount == nullptr || kmerindex == nullptr) { Error::set("vsg_udb_words: null argument"); return VSG_EINVAL; }
  *kmercount = u->kmercount.data(); *kmerindex = u->kmerindex.data();
  return VSG_OK;
}

extern "C" int vsg_udb_load(vsg_ctx * c, const vsg_udb * u, vsg_seqset ** db, vsg_index ** index, int * mask_lower)
{
  if (c == nullptr || u == nullptr || db == nullptr || index == nullptr) { Error::set("vsg_udb_load: null argument"); return VSG_EINVAL; }
  *db = nullptr; *index = nullptr;
  VSG_CUDA_OK(cudaSetDevice(c->device));
  vsg_seqset * s = nullptr;
  int rc = vsg_seqset_create(c, u->cat.data(), u->off.data(), u->len.data(), u->info.sequences, 1, &s);
  if (rc != VSG_OK) { return rc; }
  size_t const hashsize = static_cast<size_t>(1) << (2 * u->info.wordlength);
  DevBuf totals;
  if ((rc = totals.reserve(sizeof(uint32_t) * hashsize)) != VSG_OK) { vsg_seqset_destroy(s); return rc; }
  std::vector<uint32_t> got(hashsize);
  vsg_index * ix = nullptr;
  bool match = false;
  for (int ml = 1; ml >= 0 && !match; ml--) {
    cudaError_t e = cudaMemsetAsync(totals.p, 0, sizeof(uint32_t) * hashsize, c->stream);
    if (e == cudaSuccess) {
      rc = index_create_counts(c, s, u->info.wordlength, ml, static_cast<uint32_t *>(totals.p), &ix);
      if (rc != VSG_OK) { break; }
      e = cudaMemcpyAsync(got.data(), totals.p, sizeof(uint32_t) * hashsize, cudaMemcpyDeviceToHost, c->stream);
    }
    if (e == cudaSuccess) { e = cudaStreamSynchronize(c->stream); }
    if (e != cudaSuccess) { Error::set(std::string("vsg_udb_load: ") + cudaGetErrorString(e)); rc = VSG_ECUDA; break; }
    match = std::memcmp(got.data(), u->kmercount.data(), sizeof(uint32_t) * hashsize) == 0;
    if (match) { if (mask_lower != nullptr) { *mask_lower = ml; } }
    else { vsg_index_destroy(ix); ix = nullptr; }
  }
  totals.release();
  if (rc == VSG_OK && !match) {
    Error::set("vsg_udb_load: the word index stored in the UDB file does not belong to its sequences (with or without masked symbols)");
    rc = VSG_EINVAL;
  }
  if (rc != VSG_OK) { if (ix != nullptr) { vsg_index_destroy(ix); } vsg_seqset_destroy(s); return rc; }
  *db = s; *index = ix;
  return VSG_OK;
}

extern "C" int vsg_group_create_udb(const int * devices, int ndev, const vsg_scoring * scoring, const vsg_udb * u, vsg_group ** out)
{
  if (devices == nullptr || ndev < 1 || scoring == nullptr || u == nullptr || out == nullptr) { Error::set("vsg_group_create_udb: bad argument"); return VSG_EINVAL; }
  *out = nullptr;
  // the masking convention of the stored index is found on the first device, then the group is made as from FASTA
  vsg_ctx * c = nullptr;
  int rc = vsg_ctx_create(devices[0], scoring, &c);
  if (rc != VSG_OK) { return rc; }
  vsg_seqset * s = nullptr; vsg_index * ix = nullptr;
  int ml = 0;
  rc = vsg_udb_load(c, u, &s, &ix, &ml);
  if (ix != nullptr) { vsg_index_destroy(ix); }
  if (s != nullptr) { vsg_seqset_destroy(s); }
  vsg_ctx_destroy(c);
  if (rc != VSG_OK) { return rc; }
  return vsg_group_create(devices, ndev, scoring, u->cat.data(), u->off.data(), u->len.data(), u->info.sequences, u->info.wordlength, ml, 0, out);
}
