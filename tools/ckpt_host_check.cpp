// CPU check of vsearch_b200/csrc/tb_ckpt.h (the traceback of the checkpoint aligner) against the oracle.
// A scalar model of nw_ckpt_kernel (align_ckpt.cuh) fills the checkpoint arrays in the DEVICE layout (32 lanes x
// R rows, wavefront steps, chunk-aligned column checkpoints, two targets per task as biased 16-bit halves) under
// the SHIFTED scoring the kernel runs with (S - 2c, ge + c); the host/device traceback then has to reproduce
// the oracle's score (after undoing the shift), statistics and CIGAR for both targets.
//   g++ -O2 -std=c++17 -I oracle tools/ckpt_host_check.cpp -Loracle -loracle -Wl,-rpath,$PWD/oracle -o /tmp/ckpt_host_check
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <random>
#include <string>
#include <vector>

#include "oracle.h"
#include "../vsearch_b200/csrc/tb_ckpt.h"

using namespace vsg::ckpt;

struct Score {
  int16_t S[16][16];
  int go[6], ge[6];
  int n_mismatch, match, mismatch, shift;
};

static bool ambiguous4(unsigned c) { return __builtin_popcount(c) != 1; }

static void build(const oracle_scoring & o, Score & p)
{
  for (int k = 0; k < 6; k++) { p.go[k] = static_cast<int>(o.v[2 + k]); p.ge[k] = static_cast<int>(o.v[8 + k]); }
  p.n_mismatch = o.n_mismatch;
  p.match = static_cast<int>(o.v[0]); p.mismatch = static_cast<int>(o.v[1]); p.shift = 0;
  for (unsigned i = 0; i < 16; i++) {
    for (unsigned j = 0; j < 16; j++) {
      int v;
      if (p.n_mismatch && (i == 15 || j == 15)) { v = static_cast<int>(o.v[1]); }
      else if (ambiguous4(i) || ambiguous4(j)) { v = 0; }
      else if (i == j) { v = static_cast<int>(o.v[0]); }
      else { v = static_cast<int>(o.v[1]); }
      p.S[i][j] = static_cast<int16_t>(v);
    }
  }
}

// the shifted scoring of align_ckpt.cuh (vsg_api.cu: shifted_params)
static Score shifted(const Score & p)
{
  Score q = p;
  int smax = 0;
  for (int i = 0; i < 16; i++) { for (int j = 0; j < 16; j++) { smax = std::max<int>(smax, p.S[i][j]); } }
  int const c = (smax + 1) / 2;
  q.shift = c;
  for (int i = 0; i < 16; i++) { for (int j = 0; j < 16; j++) { q.S[i][j] = static_cast<int16_t>(p.S[i][j] - 2 * c); } }
  for (int k = 0; k < 6; k++) { q.ge[k] = p.ge[k] + c; }
  q.match = p.match - 2 * c; q.mismatch = p.mismatch - 2 * c;
  return q;
}

// forward pass of one (query, target) in plain ints, checkpoints written into half `half` of the task arrays
static int forward(const Score & sp, const std::vector<uint8_t> & q, const std::vector<uint8_t> & t, int R, int half,
                   std::vector<U2> & rowck, std::vector<U2> & colck)
{
  int const Q = static_cast<int>(q.size()), D = static_cast<int>(t.size());
  auto put = [&](uint32_t & w, int v) {
    uint32_t const b = static_cast<uint32_t>(v + 0x8000) & 0xffffu;
    w = half ? ((w & 0x0000ffffu) | (b << 16)) : ((w & 0xffff0000u) | b);
  };
  auto QRq = [&](int i) { return i == Q - 1 ? sp.go[CQ_R] + sp.ge[CQ_R] : sp.go[CQ_I] + sp.ge[CQ_I]; };
  auto Rq = [&](int i) { return i == Q - 1 ? sp.ge[CQ_R] : sp.ge[CQ_I]; };
  auto QRt = [&](int j) { return j >= D - 1 ? sp.go[CT_R] + sp.ge[CT_R] : sp.go[CT_I] + sp.ge[CT_I]; };
  auto Rt = [&](int j) { return j >= D - 1 ? sp.ge[CT_R] : sp.ge[CT_I]; };
  auto Hleft = [&](int i) { return i < 0 ? 0 : -(sp.go[CT_L] + (i + 1) * sp.ge[CT_L]); };
  auto Htop = [&](int j) { return j < 0 ? 0 : -(sp.go[CQ_L] + (j + 1) * sp.ge[CQ_L]); };
  std::vector<int> hprev(Q), ein(Q);
  for (int i = 0; i < Q; i++) { hprev[i] = Hleft(i); ein[i] = Hleft(i) - QRq(i); }
  int score = 0;
  for (int j = 0; j < D; j++) {
    int hdiag = Htop(j - 1), f_in = Htop(j) - QRt(j);
    for (int i = 0; i < Q; i++) {
      int const tt = hdiag + sp.S[t[j] & 15][q[i] & 15];
      int const m1 = tt > f_in ? tt : f_in;
      int const h = m1 > ein[i] ? m1 : ein[i];
      int const hf = h - QRt(j), f = f_in - Rt(j);
      int const he = h - QRq(i), e = ein[i] - Rq(i);
      hdiag = hprev[i];
      hprev[i] = h;
      ein[i] = e > he ? e : he;
      f_in = f > hf ? f : hf;
      int const l = i / R, r = i % R;
      if (r == R - 1) {   // leaves lane l's last row: what lane l hands down at step j + l
        U2 & ck = rowck[row_index(j + l, l)];
        put(ck.x, h); put(ck.y, f_in);
      }
      if ((j + l + 1) % CHUNK == 0) {   // the lane's state at the end of a 32-step chunk
        U2 & ck = colck[col_index((j + l + 1) / CHUNK, l, r, R)];
        put(ck.x, h); put(ck.y, ein[i]);
      }
    }
    score = hprev[Q - 1];
  }
  return score;
}

// fast_path_ok (vsg_api.cu): every intermediate of a (qpad x d) problem stays inside the 16-bit range
static bool path_ok(const Score & p, int qpad, int d)
{
  int64_t G = 0, Rm = 0, smax = 0, smin = 0;
  for (int k = 0; k < 6; k++) {
    if (p.go[k] < 0 || p.ge[k] < 0) { return false; }
    G = std::max<int64_t>(G, p.go[k] + p.ge[k]);
    Rm = std::max<int64_t>(Rm, p.ge[k]);
  }
  for (int i = 0; i < 16; i++) {
    for (int j = 0; j < 16; j++) { smax = std::max<int64_t>(smax, p.S[i][j]); smin = std::min<int64_t>(smin, p.S[i][j]); }
  }
  int64_t const lb = -(G + static_cast<int64_t>(qpad) * Rm) - G - static_cast<int64_t>(d + 4) * Rm - 2 * G + smin;
  int64_t const ub = smax * std::min<int64_t>(qpad, d + 4) + smax;
  return lb > -32700 && ub < 32700;
}

// the longest target (at most cap) the planner sends to the checkpoint kernels with R rows per lane: inside the
// bound of the scoring and of its shift (plan_pairs); 0 when there is none
static int ckpt_bound(const Score & p0, const Score & p, int R, int cap)
{
  int d = 0;
  for (int step = 1 << 16; step > 0; step >>= 1) {
    int const t = d + step;
    if (t <= cap && path_ok(p0, 32 * R, t) && path_ok(p, 32 * R, t)) { d = t; }
  }
  return d;
}

static std::string cigar_of(const std::string & rev)
{
  std::string out;
  size_t k = rev.size();
  while (k > 0) {
    size_t m = k;
    while (m > 0 && rev[m - 1] == rev[k - 1]) { m--; }
    size_t const run = k - m;
    if (run > 1) { out += std::to_string(run); }
    out += rev[k - 1];
    k = m;
  }
  return out;
}

int main(int argc, char ** argv)
{
  int const n = argc > 1 ? std::atoi(argv[1]) : 400;
  std::string const mode = argc > 3 ? argv[3] : "mixed";
  int const longest = argc > 2 ? std::atoi(argv[2]) : (mode == "mixed" ? 300 : 65535);
  if ((mode != "mixed" && mode != "long" && mode != "limits") || longest < 1) {
    std::fprintf(stderr, "usage: ckpt_host_check [cases [longest target [mixed|long|limits]]]\n");
    return 2;
  }
  std::mt19937 rng(12345);
  const char * acgt = "ACGT";
  const char * iupac = "ACGTUNRYSWKMBDHVacgtn";
  int bad = 0, checked = 0, longest_seen = 0, shifted_min = 0, score_max = 0;
  for (int k = 0; k < n; k++) {
    oracle_scoring sc;
    oracle_default_scoring(&sc);
    if (mode == "mixed" && k % 3 == 2) {
      sc.v[0] = 1 + rng() % 4; sc.v[1] = -static_cast<int64_t>(1 + rng() % 6);
      for (int z = 0; z < 6; z++) { sc.v[2 + z] = rng() % 22; sc.v[8 + z] = rng() % 4; }
    }
    if (mode == "limits") {
      if (k % 3 == 0) {
        sc.v[0] = 2; sc.v[1] = -80;
        for (int z = 0; z < 6; z++) { sc.v[2 + z] = 20; sc.v[8 + z] = 40; }
      } else {
        sc.v[0] = k % 3 == 1 ? 60 : 64; sc.v[1] = -4;
      }
    }
    sc.n_mismatch = mode != "limits" && (k % 7 == 6);
    Score sp0; build(sc, sp0);
    Score const sp = shifted(sp0);
    const char * A = (mode != "limits" && k % 5 == 4) ? iupac : acgt;
    size_t const na = std::strlen(A);
    int const R = 1 + rng() % 16;
    int const Q = mode == "limits" ? 32 * R : 1 + static_cast<int>(rng() % (32 * R));   // single strip
    std::string qs(Q, 'A');
    for (auto & ch : qs) { ch = A[rng() % na]; }
    std::string ts[2];
    if (mode == "mixed") {
      for (int h = 0; h < 2; h++) {
        int const D = 1 + rng() % longest;
        ts[h].assign(D, 'A');
        for (int x = 0; x < D; x++) { ts[h][x] = (k % 2 == 0 && x < Q && rng() % 10 != 0) ? qs[x] : A[rng() % na]; }
      }
    } else {
      int const dck = ckpt_bound(sp0, sp, R, longest);
      if (dck < 1) { continue; }
      for (int h = 0; h < 2; h++) {
        int D = dck - static_cast<int>(rng() % 3);
        if (mode == "long" && h == 1 && k % 3 == 0) { D = 1 + rng() % 64; }
        D = std::max(D, 1);
        // a relative of the query: 5 % substitutions
        std::string m = qs;
        for (auto & ch : m) { if (rng() % 20 == 0) { ch = A[rng() % na]; } }
        std::string t(D, 'A');
        for (auto & ch : t) { ch = A[rng() % na]; }
        bool const unrelated = mode == "limits" && k % 3 == 0;   // harsh penalties: the lowest scores
        if (!unrelated) {
          if (D <= Q) { t = m.substr(static_cast<size_t>(rng() % (Q - D + 1)), static_cast<size_t>(D)); }
          else {
            int const where = (k + h) % 3;   // 0: query at the start, 1: at the end, 2: in the middle
            int const at = where == 0 ? 0 : (where == 1 ? D - Q : (D - Q) / 2);
            t.replace(static_cast<size_t>(at), static_cast<size_t>(Q), m);
          }
        }
        ts[h] = t;
      }
    }
    int const dmax = static_cast<int>(std::max(ts[0].size(), ts[1].size()));
    longest_seen = std::max(longest_seen, dmax);
    std::vector<U2> rowck(row_elems(dmax), U2{0xdeaddeadu, 0xdeaddeadu});
    std::vector<U2> colck(col_elems(dmax, R), U2{0xdeaddeadu, 0xdeaddeadu});
    std::vector<uint8_t> q4(Q);
    for (int i = 0; i < Q; i++) { q4[i] = oracle_map_4bit(static_cast<unsigned char>(qs[i])); }
    for (int h = 0; h < 2; h++) {
      int const D = static_cast<int>(ts[h].size());
      std::vector<uint8_t> t4(D);
      for (int x = 0; x < D; x++) { t4[x] = oracle_map_4bit(static_cast<unsigned char>(ts[h][x])); }
      int const score = forward(sp, q4, t4, R, h, rowck, colck);
      // (the second target's forward pass runs before the first one's traceback in a kernel too)
      if (h == 0) { continue; }
      shifted_min = std::min(shifted_min, score);
      for (int hh = 0; hh < 2; hh++) {
        int const DD = static_cast<int>(ts[hh].size());
        std::vector<uint8_t> tt(DD);
        for (int x = 0; x < DD; x++) { tt[x] = oracle_map_4bit(static_cast<unsigned char>(ts[hh][x])); }
        int general = 0;
        for (int x = 0; x < Q; x++) { general |= __builtin_popcount(q4[x] & 15) != 1; }
        for (int x = 0; x < DD; x++) { general |= __builtin_popcount(tt[x] & 15) != 1; }
        PairView pv{rowck.data(), colck.data(), R, hh, Q, DD, general, q4.data(), tt.data()};
        TbOut out{};
        std::string rev;
        HostBits bits;
        HostRows rows{rowck.data()};
        auto emit = [&](char o, int cnt) { rev.append(static_cast<size_t>(cnt), o); };
        if (R <= 8) { if (general) { traceback<8, true>(sp, pv, bits, rows, out, emit); } else { traceback<8, false>(sp, pv, bits, rows, out, emit); } }
        else { if (general) { traceback<16, true>(sp, pv, bits, rows, out, emit); } else { traceback<16, false>(sp, pv, bits, rows, out, emit); } }
        int16_t os; uint16_t oa, om, omi, og;
        std::vector<char> cig(Q + DD + 64);
        if (oracle_nw16(&sc, qs.data(), Q, ts[hh].data(), DD, &os, &oa, &om, &omi, &og, cig.data(), cig.size()) != 0) { std::fprintf(stderr, "oracle_nw16 failed\n"); return 2; }
        if (os == ORACLE_SENTINEL) { continue; }
        checked++;
        score_max = std::max<int>(score_max, os);
        std::string const got = cigar_of(rev);
        bool ok = got == cig.data() && out.aligned == oa && out.matches == om && out.mismatches == omi && out.gaps == og;
        {
          // terminal runs as the driver's align_trim wants them (VSG_STAT_TRIM_LEFT/RIGHT): D positive, I negative
          std::string const c(cig.data());
          auto run_at = [&](size_t pos, int & len, char & o) {
            len = 0;
            while (pos < c.size() && c[pos] >= '0' && c[pos] <= '9') { len = len * 10 + (c[pos] - '0'); pos++; }
            if (len == 0) { len = 1; }
            o = c[pos];
          };
          int l0 = 0, l1 = 0; char o0 = 0, o1 = 0;
          run_at(0, l0, o0);
          size_t last = c.size() - 1;               // the op letter of the last run
          size_t st = last;
          while (st > 0 && c[st - 1] >= '0' && c[st - 1] <= '9') { st--; }
          run_at(st, l1, o1);
          int const want_left = o0 == 'D' ? l0 : (o0 == 'I' ? -l0 : 0);
          int const want_right = o1 == 'D' ? l1 : (o1 == 'I' ? -l1 : 0);
          ok = ok && out.trim_left == want_left && out.trim_right == want_right;
        }
        if (hh == 1) { ok = ok && score + sp.shift * (Q + DD) == os; }
        if (!ok) {
          if (++bad <= 5) {
            std::fprintf(stderr, "MISMATCH case %d half %d R %d Q %d D %d: %s vs %s  (%d %d %d %d | %d %d %d %d)\n", k, hh, R, Q, DD,
                         got.c_str(), cig.data(), out.aligned, out.matches, out.mismatches, out.gaps, oa, om, omi, og);
          }
        }
      }
    }
  }
  std::printf("%d pairs checked, %d mismatches (longest target %d, lowest shifted score %d, highest score %d)\n", checked, bad,
              longest_seen, shifted_min, score_max);
  return bad != 0;
}
