// tb_ckpt.h — the traceback that goes with nw_ckpt_kernel (align_ckpt.cuh): backtrack16
// (align_simd.cpp:1132-1245) over direction bits that are REGENERATED, tile by tile, from the forward
// pass's checkpoints instead of being read from a stored direction matrix.
//
// A tile = the cells lane b (rows [b*R, b*R+R)) computes during one 32-step chunk k of the wavefront,
// i.e. columns [32k - b, 32k - b + 31] clipped to the matrix.  Its inputs are exactly what the kernel
// checkpointed: H/E of the lane's rows at the end of chunk k-1 (column checkpoint k), and H/F leaving
// lane b-1's last row at every step (row checkpoints); first-row / first-column tiles use the boundary
// formulas (align_simd.cpp:852-857, 1895-1910).  Regenerating a tile replays onestep
// (align_simd.cpp:765-780) in plain ints; the walk then follows backtrack16's priorities.  Only the part
// of a tile between its top-left corner and the cell the path enters it at is recomputed.
//
// Host/device: the same function runs inside traceback_ckpt kernels and, compiled for the CPU, in
// tools/ckpt_host_check.cpp, which checks it against the oracle (tests/test_ckpt_cpu.py) over
// checkpoints laid out exactly as the kernel writes them.
#pragma once

#include <stdint.h>

#ifdef __CUDACC__
#define VSG_CKPT_HD __host__ __device__ __forceinline__
#else
#define VSG_CKPT_HD inline
#endif
#ifdef __CUDA_ARCH__
#define VSG_CKPT_UNROLL _Pragma("unroll")
#define VSG_CKPT_NOUNROLL _Pragma("unroll 1")
#else
#define VSG_CKPT_UNROLL
#define VSG_CKPT_NOUNROLL
#endif

namespace vsg {
namespace ckpt {

constexpr int CHUNK = 32;   // steps per chunk = distance between column checkpoints (in steps)
constexpr int RMAX = 16;    // rows per lane

struct U2 { uint32_t x, y; };  // layout of CUDA's uint2

// ---- checkpoint layout of one task (U2 / uint2 elements; .x/.y = the two values, low half = first target) ----
// The forward kernel writes it, the traceback reads it, and the host model of tools/ckpt_host_check.cpp writes it
// for the host traceback: all three use these functions.
// row checkpoints: element of (step s, lane l) — four consecutive steps of a lane share a 32-byte sector
VSG_CKPT_HD size_t row_index(int s, int l) { return (static_cast<size_t>(s >> 2) * 32 + l) * 4 + (s & 3); }
VSG_CKPT_HD size_t row_elems(int dmax) { return static_cast<size_t>((dmax + 31 + 3) >> 2) * 128; }
// column checkpoints: state (H, E entering the next column) of lane l's row r after step 32k - 1, k >= 1
VSG_CKPT_HD size_t col_index(int k, int l, int r, int R) { return (static_cast<size_t>(k - 1) * R + r) * 32 + l; }
VSG_CKPT_HD size_t col_elems(int dmax, int R) { return static_cast<size_t>((dmax + 31 + CHUNK - 1) / CHUNK) * R * 32; }

struct PairView {
  const U2 * rowck;   // the task's row checkpoints
  const U2 * colck;   // the task's column checkpoints
  int R, half, Q, D;
  int general;        // a symbol outside ACGT in either sequence: scores come from the 16x16 matrix
  const uint8_t * q;  // symbols, 4-bit code in the low nibble
  const uint8_t * t;
};

struct ckpt_true { static constexpr bool value = true; };
struct ckpt_false { static constexpr bool value = false; };

struct TbOut { int aligned, matches, mismatches, gaps, trim_left, trim_right; };  // VSG_STAT_* meanings

enum { CQ_L = 0, CT_L = 1, CQ_I = 2, CT_I = 3, CQ_R = 4, CT_R = 5 };

// Bits: storage of one regenerated tile — set(column, word, value) / get(column, word); word w of a column
// holds the 4-bit directions of rows 8w .. 8w+7.  The device keeps it in shared memory (one bank per thread),
// the host in a plain array.
struct HostBits {
  uint32_t w[CHUNK][RMAX / 8];
  void set(int bj, int k, uint32_t v) { w[bj][k] = v; }
  uint32_t get(int bj, int k) const { return w[bj][k]; }
  // slot (bj, 0) <- word wi of the target's aligned symbol window (see Walk::round); asynchronous on the device
  void stage_word(int bj, const uint8_t * t, int D, int mis, int wi);
  void wait() {}
};

// Rows: access to the row checkpoints of one lane for a tile's steps.  stage(l, s0, s1) announces the range
// [s0, s1] of steps about to be read (at most 34 of them: a tile's columns plus the diagonal input); the device
// version copies the sectors into shared memory with cp.async so that all of a tile's loads are in flight
// together instead of one dependent load per column; the host version reads memory directly.
struct HostRows {
  const U2 * rowck;
  int lane = 0;
  void stage(int l, int, int) { lane = l; }
  void wait() {}
  U2 get(int s) const { return rowck[row_index(s, lane)]; }
};

// ---- packed pairs of biased 16-bit values (the forward kernel's representation) --------------------------------
VSG_CKPT_HD uint32_t pk16(uint32_t lo, uint32_t hi) { return (lo & 0xffffu) | (hi << 16); }
// low half of a below the low half of b
VSG_CKPT_HD uint32_t lo_lo(uint32_t a, uint32_t b)
{
#ifdef __CUDA_ARCH__
  return __byte_perm(a, b, 0x5410);
#else
  return (a & 0xffffu) | (b << 16);
#endif
}
// low half of a below the high half of b
VSG_CKPT_HD uint32_t lo_hi(uint32_t a, uint32_t b)
{
#ifdef __CUDA_ARCH__
  return __byte_perm(a, b, 0x7610);
#else
  return (a & 0xffffu) | (b & 0xffff0000u);
#endif
}
// per-half unsigned max(a, b); where b > a strictly (the reference's compares, align_simd.cpp:765-780) the flag constant
// of that half is added to its word: clo to wlo for the low halves, chi to whi for the high ones.  On the device this is
// one VIMNMX.U16x2 with two predicate outputs and two predicated adds (the PTX below is the idiom ptxas fuses).
VSG_CKPT_HD uint32_t pmax_flag2(uint32_t a, uint32_t b, uint32_t & wlo, uint32_t clo, uint32_t & whi, uint32_t chi)
{
#ifdef __CUDA_ARCH__
  uint32_t m;
  asm("{.reg .pred plo, phi;\n\t.reg .u16 m0, m1, a0, a1;\n\t"
      "max.u16x2 %0, %3, %4;\n\t"
      "mov.b32 {m0, m1}, %0;\n\tmov.b32 {a0, a1}, %3;\n\t"
      "setp.eq.u16 plo, m0, a0;\n\tsetp.eq.u16 phi, m1, a1;\n\t"
      "@!plo add.u32 %1, %1, %5;\n\t@!phi add.u32 %2, %2, %6;}"
      : "=&r"(m), "+r"(wlo), "+r"(whi) : "r"(a), "r"(b), "r"(clo), "r"(chi));
  return m;
#else
  uint32_t const al = a & 0xffffu, bl = b & 0xffffu, ah = a >> 16, bh = b >> 16;
  if (bl > al) { wlo += clo; }
  if (bh > ah) { whi += chi; }
  return (bl > al ? bl : al) | ((bh > ah ? bh : ah) << 16);
#endif
}
// the same with both halves' flags in one word
VSG_CKPT_HD uint32_t pmax_flag1(uint32_t a, uint32_t b, uint32_t & w, uint32_t clo, uint32_t chi)
{
#ifdef __CUDA_ARCH__
  uint32_t m;
  asm("{.reg .pred plo, phi;\n\t.reg .u16 m0, m1, a0, a1;\n\t"
      "max.u16x2 %0, %2, %3;\n\t"
      "mov.b32 {m0, m1}, %0;\n\tmov.b32 {a0, a1}, %2;\n\t"
      "setp.eq.u16 plo, m0, a0;\n\tsetp.eq.u16 phi, m1, a1;\n\t"
      "@!plo add.u32 %1, %1, %4;\n\t@!phi add.u32 %1, %1, %5;}"
      : "=&r"(m), "+r"(w) : "r"(a), "r"(b), "r"(clo), "r"(chi));
  return m;
#else
  uint32_t const al = a & 0xffffu, bl = b & 0xffffu, ah = a >> 16, bh = b >> 16;
  if (bl > al) { w += clo; }
  if (bh > ah) { w += chi; }
  return (bl > al ? bl : al) | ((bh > ah ? bh : ah) << 16);
#endif
}
// per-half min(m, 1)
VSG_CKPT_HD uint32_t pmin1(uint32_t m)
{
#ifdef __CUDA_ARCH__
  return __vminu2(m, 0x00010001u);
#else
  return ((m & 0xffffu) ? 1u : 0u) | ((m >> 16) ? 0x10000u : 0u);
#endif
}

// four consecutive symbol bytes as one word: word w of the 4-byte-aligned window the sequence lies in (the device reads
// an aligned 32-bit word, which may reach up to three bytes before / past the sequence: the symbol buffers are padded,
// vsg_api.cu; the host model assembles the bytes it is allowed to touch)
VSG_CKPT_HD uint32_t sym_word(const uint8_t * t, int D, int mis, int w)
{
#ifdef __CUDA_ARCH__
  (void)D;
  return __ldg(reinterpret_cast<const uint32_t *>(t - mis) + w);
#else
  uint32_t x = 0;
  for (int z = 0; z < 4; z++) {
    int const idx = 4 * w + z - mis;
    if (idx >= 0 && idx < D) { x |= static_cast<uint32_t>(t[idx]) << (8 * z); }
  }
  return x;
#endif
}

inline void HostBits::stage_word(int bj, const uint8_t * t, int D, int mis, int wi) { w[bj][0] = sym_word(t, D, mis, wi); }

// emit(op, n) receives the alignment's operations last to first as runs ('M', 'I' = column consumed alone,
// 'D' = row consumed alone; consecutive calls may carry the same op).  SP supplies S[16][16], go[6], ge[6], match,
// mismatch, n_mismatch — the SAME (shifted) scoring the forward kernel ran with: the direction bits do not depend on
// the shift.
//
// Regeneration of a tile runs on the checkpoints' own representation, two cells per instruction like the forward
// kernel: the tile's rows are split in two halves of RH = RT/2 rows; packed operation k of step c computes row k at
// the tile's column c in the low halfword and row RH + k at column c - 1 in the high halfword (the one-column skew
// is what row RH needs from row RH - 1).  Step 0's high halves and the last step's low halves lie outside the tile:
// the former are computed and discarded, the latter get harmless inputs.  All subtractions are plain 32-bit ones;
// the host's bound (vsg_api.cu: fast_path_ok on the shifted scoring) keeps every real intermediate non-negative,
// and the halves that can hold garbage (rows below the entry row: always the HIGH half of an operation whose low
// half is real, or both) can only borrow out of bit 31.
// GENERAL: a symbol outside ACGT in either sequence (scores from the 16x16 table instead of match / mismatch).
// One alignment's traceback as a resumable object: start(), then round() once per tile while running(), then
// finish().  The statistics-only kernel keeps one of these per thread and runs the rounds of a warp's 32 walks
// together (align_ckpt.cuh).
template <int RT, bool GENERAL>
struct Walk {
  PairView v;
  int i, j, b, i0;
  char op;
  int aligned, matches, mismatches, gaps;
  char last_run_op; int last_run; bool last_open;   // the run that ENDS the alignment
  char first_op; int first_run;                     // the run still open = the alignment's first

  VSG_CKPT_HD void start(const PairView & pv)
  {
    v = pv;
    i = v.Q - 1; j = v.D - 1;
    b = i / v.R; i0 = b * v.R;
    op = 0;
    aligned = 0; matches = 0; mismatches = 0; gaps = 0;
    last_run_op = 0; last_run = 0; last_open = true;
    first_op = 0; first_run = 0;
  }
  VSG_CKPT_HD bool running() const { return i >= 0 && j >= 0; }

  template <class Emit>
  VSG_CKPT_HD void push(Emit & emit, char nop, int n)
  {
    aligned += n;
    if (last_open) {
      if (last_run == 0 || nop == last_run_op) { last_run_op = nop; last_run += n; }
      else { last_open = false; }
    }
    if (nop == first_op) { first_run += n; } else { first_op = nop; first_run = n; }
    emit(nop, n);
    op = nop;
  }

  // regenerate the tile the path is about to enter and walk through it
  template <class SP, class Bits, class Rows, class Emit>
  VSG_CKPT_HD void round(const SP & sp, Bits & bits, Rows & rows, Emit & emit)
  {
  constexpr int RH = RT / 2;
  constexpr uint32_t B = 0x8000u;
  int const R = v.R, Q = v.Q, D = v.D, sh = 16 * v.half;
  uint32_t const QRqi = sp.go[CQ_I] + sp.ge[CQ_I], Rqi = sp.ge[CQ_I], QRqr = sp.go[CQ_R] + sp.ge[CQ_R], Rqr = sp.ge[CQ_R];
  uint32_t const QRti = sp.go[CT_I] + sp.ge[CT_I], Rti = sp.ge[CT_I], QRtr = sp.go[CT_R] + sp.ge[CT_R], Rtr = sp.ge[CT_R];
  int const gotl = sp.go[CT_L], getl = sp.ge[CT_L], goql = sp.go[CQ_L], geql = sp.ge[CQ_L];
  // match / mismatch scoring of pure ACGT pairs: -S = sx - e * ds with e = 1 on a match (shifted scores are <= 0)
  uint32_t const sx = static_cast<uint32_t>(-static_cast<int>(sp.mismatch));
  uint32_t const sx2 = pk16(sx, sx);
  uint32_t const ds = static_cast<uint32_t>(static_cast<int>(sp.match) - static_cast<int>(sp.mismatch));
  auto half_of = [&](uint32_t w) { return (w >> sh) & 0xffffu; };   // stays biased

    // ---- regenerate the tile (lane b, chunk k) up to the cell (i, j) ----
    int const k = (j + b) / CHUNK;
    int const jlo = (CHUNK * k - b) > 0 ? (CHUNK * k - b) : 0;
    int const ni = i - i0 + 1, nj = j - jlo + 1;
    int const nk = ni < RH ? ni : RH;                 // packed operations per step
    int const nsteps = ni > RH ? nj + 1 : nj;         // the skewed high halves need one more step
    // the tile's row checkpoints: lane b-1 at steps (jlo-1)+(b-1) .. j+(b-1), the first one being the diagonal
    // input H(i0-1, jlo-1) of the tile's first cell
    if (b > 0) { rows.stage(b - 1, jlo + b - 2 > 0 ? jlo + b - 2 : 0, j + b - 1); }
    // only the query's last row has other query-gap penalties, and it can only be the tile's last row
    int const alast = (i == Q - 1) ? ni - 1 : -1;
    uint32_t hcol[RH], ecol[RH], X[RH], qrq[RH], rq[RH];
    // every global load of the set-up is issued before the first one is used
    U2 ckv[RT];
    uint32_t qv[RT];
    bool const from_ck = jlo != 0;
VSG_CKPT_UNROLL
    for (int a = 0; a < RT; a++) {
      int const ii = i0 + a < Q ? i0 + a : Q - 1;
      qv[a] = v.q[ii];
    }
    if (from_ck) {
VSG_CKPT_UNROLL
      for (int a = 0; a < RT; a++) { ckv[a] = v.colck[col_index(k, b, a < R ? a : R - 1, R)]; }
    } else {
VSG_CKPT_UNROLL
      for (int a = 0; a < RT; a++) { ckv[a] = U2{0u, 0u}; }
    }
    // the target's symbols come as aligned words of four, three words in flight
    int const tmis = static_cast<int>(reinterpret_cast<uintptr_t>(v.t) & 3u);
    int const twmax = (D - 1 + tmis) >> 2;
    // step 0 takes column jlo's symbol; after it the steps run in groups of four that share one 4-symbol word,
    // funnelled out of two words of the target's aligned symbol window.  The window's words are copied (cp.async on
    // the device: no registers, nothing waits) into slots of the tile's bit storage that are only written later:
    // word m of the window, first needed by the group of steps 4m+1 .. 4m+4, sits in column slot 4m+3, which the
    // regeneration fills at step 4m+3 (RT 16) or 4m+4 (RT 8) — after that group's words have been read.  A ninth
    // word (second word of the last group when the window is misaligned) stays in a register.
    int const tg = jlo + 1 + tmis;          // byte offset of step 1's symbol in the aligned window
    int const tsh = 8 * (tg & 3);
    int const twi = tg >> 2;
    uint32_t const t_first = v.t[jlo];
VSG_CKPT_UNROLL
    for (int m = 0; m < CHUNK / 4; m++) { bits.stage_word(4 * m + 3, v.t, D, tmis, twi + m < twmax ? twi + m : twmax); }
    uint32_t const tw_last = sym_word(v.t, D, tmis, twi + CHUNK / 4 < twmax ? twi + CHUNK / 4 : twmax);
    uint32_t sym4 = t_first;
    uint32_t qpack[RT / 8];
VSG_CKPT_UNROLL
    for (int w = 0; w < RT / 8; w++) { qpack[w] = 0; }
VSG_CKPT_UNROLL
    for (int a = 0; a < RT; a++) { qpack[a >> 3] |= (qv[a] & 15u) << (4 * (a & 7)); }
VSG_CKPT_UNROLL
    for (int kk = 0; kk < RH; kk++) {
      uint32_t hh[2], ee[2], xx[2];
VSG_CKPT_UNROLL
      for (int s = 0; s < 2; s++) {
        int const a = kk + s * RH;
        int const ii = i0 + a;
        bool const in = a < ni;
        xx[s] = in ? (qv[a] & 15u) : 0u;
        uint32_t const hb = B - static_cast<uint32_t>(gotl + (ii + 1) * getl);   // H(ii,-1)
        uint32_t const eb = hb - (ii == Q - 1 ? QRqr : QRqi);                     // E(ii,0)
        hh[s] = in ? (from_ck ? half_of(ckv[a].x) : hb) : B;
        ee[s] = in ? (from_ck ? half_of(ckv[a].y) : eb) : B;
      }
      hcol[kk] = pk16(hh[0], hh[1]); ecol[kk] = pk16(ee[0], ee[1]); X[kk] = pk16(xx[0], xx[1]);
      qrq[kk] = pk16(kk == alast ? QRqr : QRqi, kk + RH == alast ? QRqr : QRqi);
      rq[kk] = pk16(kk == alast ? Rqr : Rqi, kk + RH == alast ? Rqr : Rqi);
    }
    if (b > 0) { rows.wait(); } else { bits.wait(); }
    // H(i0-1, jlo-1): the diagonal input of the tile's first cell
    uint32_t hd;
    if (b == 0) { hd = jlo == 0 ? B : B - static_cast<uint32_t>(goql + jlo * geql); }
    else if (jlo == 0) { hd = B - static_cast<uint32_t>(gotl + i0 * getl); }
    else { hd = half_of(rows.get(jlo - 1 + b - 1).x); }
    // what row RH (first of the high halves) takes from row RH - 1: H two columns back (diagonal), F one column back
    uint32_t hmid_p = hcol[RH - 1], hmid_pp = B, fmid_p = B;
    uint32_t tprev = 0, qrt_prev = QRti, rt_prev = Rti;
    unsigned long long tsym2 = 0;   // ACGT pairs: the tile's column symbols as 2-bit codes, for the walk's match test
    uint32_t wprev = 0;   // RT == 8: the low rows' bits of the previous column wait for the high rows'
    U2 cknext = U2{0u, 0u};   // lane b-1's checkpoint of the next step: loaded one step ahead
    if (b > 0) { cknext = rows.get(jlo + b - 1); }
    auto step = [&](int c, auto first_tag) {
      constexpr bool FIRST = decltype(first_tag)::value;
      int const jj = jlo + c;
      uint32_t const qrt_lo = jj >= D - 1 ? QRtr : QRti, rt_lo = jj >= D - 1 ? Rtr : Rti;
      uint32_t const qrt2 = pk16(qrt_lo, qrt_prev), rt2 = pk16(rt_lo, rt_prev);
      qrt_prev = qrt_lo; rt_prev = rt_lo;
      uint32_t htop, fin;
      if (c == nj) { htop = B; fin = B; }   // past the tile: any in-range value
      else if (b == 0) { htop = B - static_cast<uint32_t>(goql + (jj + 1) * geql); fin = htop - qrt_lo; }
      else { htop = half_of(cknext.x); fin = half_of(cknext.y); }
      if (b > 0 && c + 1 < nj) { cknext = rows.get(jj + b); }
      uint32_t hdiag = lo_lo(hd, hmid_pp);
      uint32_t f = lo_lo(fin, fmid_p);
      hd = htop;
      uint32_t const tc = sym4 & 15u;
      sym4 >>= 8;
      if (!GENERAL && c < nj) { tsym2 |= static_cast<unsigned long long>((tc >> 1) - (tc >> 3)) << (2 * c); }
      uint32_t const T = tc | (tprev << 16);
      tprev = tc;
      uint32_t w0 = 0, w1 = 0;
      uint32_t hmid_new = B, fmid_new = B;
VSG_CKPT_UNROLL
      for (int kk = 0; kk < RH; kk++) {
        if (kk >= nk) { break; }
        uint32_t tt;
        if (!GENERAL) {
          tt = (hdiag - sx2) + pmin1(X[kk] & T) * ds;
        } else {
          uint32_t const sn_lo = static_cast<uint32_t>(-static_cast<int>(sp.S[T & 15u][X[kk] & 15u]));
          uint32_t const sn_hi = static_cast<uint32_t>(-static_cast<int>(sp.S[T >> 16][X[kk] >> 16]));
          tt = hdiag - pk16(sn_lo, sn_hi);
        }
        uint32_t const one = 1u << (4 * kk);
        uint32_t const e_in = ecol[kk];
        uint32_t m1, h, fn, en;
        if (RT == 8) {   // one word per column: rows 0-3 in the low half, rows 4-7 in the high half
          m1 = pmax_flag1(tt, f, w0, one, one << 16);                              // up:      F > h
          h = pmax_flag1(m1, e_in, w0, 2u * one, 2u * (one << 16));                // left:    E > h
          fn = pmax_flag1(h - qrt2, f - rt2, w0, 4u * one, 4u * (one << 16));      // extup:   F - R > H - QR
          en = pmax_flag1(h - qrq[kk], e_in - rq[kk], w0, 8u * one, 8u * (one << 16));   // extleft: E - R > H - QR
        } else {         // word 0: rows 0-7, word 1: rows 8-15
          m1 = pmax_flag2(tt, f, w0, one, w1, one);
          h = pmax_flag2(m1, e_in, w0, 2u * one, w1, 2u * one);
          fn = pmax_flag2(h - qrt2, f - rt2, w0, 4u * one, w1, 4u * one);
          en = pmax_flag2(h - qrq[kk], e_in - rq[kk], w0, 8u * one, w1, 8u * one);
        }
        hdiag = hcol[kk];
        hcol[kk] = FIRST ? lo_hi(h, hdiag) : h;       // step 0's high halves belong to no column
        ecol[kk] = FIRST ? lo_hi(en, e_in) : en;
        f = fn;
        if (kk == RH - 1) { hmid_new = h; fmid_new = fn; }
      }
      hmid_pp = hmid_p; hmid_p = hmid_new; fmid_p = fmid_new;
      if (RT == 8) {
        if (!FIRST) { bits.set(c - 1, 0, lo_hi(wprev, w0)); }
        wprev = w0;
      } else {
        if (c < nj) { bits.set(c, 0, w0); }
        if (!FIRST) { bits.set(c - 1, 1, w1); }
      }
    };
    step(0, ckpt_true{});
    for (int c = 1; c < nsteps;) {
      {
        int const m = (c - 1) >> 2;
        uint32_t const wa = bits.get(4 * m + 3, 0);
        uint32_t const wb = m + 1 < CHUNK / 4 ? bits.get(4 * m + 7, 0) : tw_last;
#ifdef __CUDA_ARCH__
        sym4 = __funnelshift_r(wa, wb, tsh);
#else
        sym4 = tsh == 0 ? wa : ((wa >> tsh) | (wb << (32 - tsh)));
#endif
      }
      int const ce = c + 4 < nsteps ? c + 4 : nsteps;
VSG_CKPT_NOUNROLL
      for (; c < ce; c++) { step(c, ckpt_false{}); }
    }
    if (RT == 8 && nsteps == nj) { bits.set(nj - 1, 0, wprev); }   // no high rows in this tile: the last column's word is still pending
    // ---- walk inside the tile (backtrack16's priorities, align_simd.cpp:1150-1210) ----
    auto nib = [&](int a, int bj) { return (bits.get(bj, RT > 8 ? (a >> 3) : 0) >> (4 * (a & 7))) & 15u; };
    while (i >= i0 && j >= jlo) {
      int const a = i - i0;
      uint32_t const d = nib(a, j - jlo);
      if ((op == 'I') && (d & 8u)) {
        // a gap run continues for as long as the cells say "extend": nothing else is looked at on the way
        int n = 1;
        j--;
        while (j >= jlo && (nib(a, j - jlo) & 8u)) { n++; j--; }
        push(emit, 'I', n);
        continue;
      }
      bool const ext_d = (op == 'D') && (d & 4u);
      bool const open_i = !ext_d && (d & 2u);
      bool const open_d = !ext_d && !open_i && (d & 1u);
      bool const is_i = open_i, is_d = ext_d || open_d;
      if ((open_i && op != 'I') || (open_d && op != 'D')) { gaps++; }
      if (!is_i && !is_d) {
        int const qa = static_cast<int>((qpack[RT > 8 ? (a >> 3) : 0] >> (4 * (a & 7))) & 15u);
        bool hit;
        if (!GENERAL) { hit = static_cast<uint32_t>((qa >> 1) - (qa >> 3)) == (static_cast<uint32_t>(tsym2 >> (2 * (j - jlo))) & 3u); }
        else { int const cc = v.t[j] & 15; hit = (qa & cc) != 0 && !(sp.n_mismatch && (qa == 15 || cc == 15)); }
        if (hit) { matches++; } else { mismatches++; }
      }
      if (!is_i) { i--; }
      if (!is_d) { j--; }
      push(emit, is_i ? 'I' : (is_d ? 'D' : 'M'), 1);
    }
    if (i < i0) { b--; i0 -= R; }
  }

  template <class Emit>
  VSG_CKPT_HD void finish(TbOut & out, Emit & emit)
  {
    if (i >= 0) { if (op != 'D') { gaps++; } push(emit, 'D', i + 1); i = -1; }
    if (j >= 0) { if (op != 'I') { gaps++; } push(emit, 'I', j + 1); j = -1; }
    out.aligned = aligned; out.matches = matches; out.mismatches = mismatches; out.gaps = gaps;
    out.trim_left = first_op == 'D' ? first_run : (first_op == 'I' ? -first_run : 0);
    out.trim_right = last_run_op == 'D' ? last_run : (last_run_op == 'I' ? -last_run : 0);
  }
};

template <int RT, bool GENERAL, class SP, class Bits, class Rows, class Emit>
VSG_CKPT_HD void traceback(const SP & sp, const PairView & v, Bits & bits, Rows & rows, TbOut & out, Emit && emit)
{
  Walk<RT, GENERAL> w;
  w.start(v);
  while (w.running()) { w.round(sp, bits, rows, emit); }
  w.finish(out, emit);
}

}  // namespace ckpt
}  // namespace vsg
