// align_ckpt.cuh — forward DP WITHOUT direction bits (sm_90a): the product's main aligner kernel.
//
// nw_ckpt_kernel<R, MODE, WRITE> is the warp wavefront of nw_fast_kernel (one warp = one query x two targets
// as packed 16-bit halves; lane l owns query rows [l*R, l*R+R) and visits column s - l at step s; DP
// state lives in registers, H/F of the row above arrive by SHFL.UP), but instead of the four direction
// bits per cell (align_simd.cpp:710-717) it keeps only what a traceback needs to REGENERATE the bits
// of the cells its path actually crosses (tb_ckpt.h):
//   row checkpoints    (H, F) leaving every lane's last row, every step   ->  8 B per lane-step
//   column checkpoints (H, E) of every row at the end of every 32-step chunk -> R * 8 B per lane-chunk
// The cell update (align_simd.cpp:752-781 without the compares) is then six instructions per packed
// cell pair, three on each of the SM's two integer pipes (tools/pipe_probe.cu: every one of them
// issues at 0.5 warp-instructions/clk/SMSP, the two pipes run in parallel):
//   t  = Hdiag - Sn                               IMAD.IADD   (FMA pipe)
//   h  = max3(t, F, E)                            VIMNMX3.U16x2          (ALU pipe)
//   F' = max(h - QRt, F - Rt)                     IMAD.IADD + VIADDMNMX.U16x2
//   E' = max(h - QRq, E - Rq)                     IMAD.IADD + VIADDMNMX.U16x2
// The subtractions are plain 32-bit ones, which is what lets ptxas put them on the FMA pipe; that
// needs every subtrahend to be a non-negative packed pair.  Substitution scores can be positive, so
// the host hands the kernel a SHIFTED scoring (vsg_api.cu: shifted_params): with c = ceil(smax / 2),
//   S2 = S - 2c <= 0,  ge2 = ge + c  (all six),  go unchanged
// is the same alignment problem with every cell of anti-diagonal i+j lowered by c*(i+j+2): all four
// direction bits of every cell are unchanged (they compare quantities of the same cell), the score
// is recovered as H2 + c*(Q+D).  Arithmetic is exact in the biased unsigned halfwords of
// align_kernels.cuh; the host bound (fast_path_ok) is evaluated for the shifted scoring too.
#pragma once

#include "align_kernels.cuh"
#include "tb_ckpt.h"   // the checkpoint layout and the traceback that reads it

namespace vsg {

static_assert(ckpt::RMAX == FAST_RMAX, "tb_ckpt.h and align_kernels.cuh disagree");
constexpr int CK_SO_STEPS = 8;   // steps per trip of the score-only steady loop
static_assert(ckpt::CHUNK % CK_SO_STEPS == 0, "score-only trip");

enum { CK_PROF = 0, CK_LUT = 1, CK_GEN = 2 };
__host__ __device__ constexpr size_t ck_dyn_smem(int R, int mode)
{
  return mode == CK_PROF ? static_cast<size_t>(FAST_WARPS) * 16 * ((R + 3) / 4) * 32 * 16 : 0;
}

// What a launch of the forward kernel writes besides the scores:
//   CK_STORE      row and column checkpoints of every task
//   CK_SCOREONLY  none (tasks whose pairs are all group followers of a gated search call: their walk is
//                 usually skipped, see TbGate below); a leaner steady loop without the staging of the stores
//   CK_RERUN      the checkpoints of those score-only tasks that turn out to need a walk after all (a half
//                 whose leader's verdict is not TB_VERDICT_ACCEPTED); every other warp returns after
//                 reading its task.  The scores are already in place and are not written again.
enum { CK_STORE = 0, CK_SCOREONLY = 1, CK_RERUN = 2 };

// stored in a group leader's VSG_STAT_CIGARLEN word by the phase-1 walk when the leader is accepted (TbGate)
constexpr int32_t TB_VERDICT_ACCEPTED = 0x5ca1ab1e;

template <int R, int MODE, int WRITE>
__global__ void __launch_bounds__(FAST_WARPS * 32)
nw_ckpt_kernel(const __grid_constant__ ScoreParams sp, DevSeqs qs, DevSeqs ts,
               const FastTask * __restrict__ tasks, int ntasks,
               uint2 * __restrict__ rowck, uint2 * __restrict__ colck, int32_t * __restrict__ stats,
               const int32_t * __restrict__ leader_of, int * __restrict__ rerun_count)
{
  constexpr bool PROF = (MODE == CK_PROF);
  constexpr bool GENERAL = (MODE == CK_GEN);
  constexpr bool STORE = (WRITE != CK_SCOREONLY);
  static_assert(!PROF || R <= 8, "the per-lane profile is for R <= 8");
  constexpr int RQ = (R + 3) / 4;
  constexpr int LUT_WORDS = GENERAL ? 4096 : (PROF ? 32 : 64 * 32);
  extern __shared__ uint4 prof_mem[];
  __shared__ uint32_t lut[LUT_WORDS];
  // column records of the warp's current and next chunk; every record is stored twice, RING entries
  // apart, so that the 32 records a lane reads during a chunk are contiguous.  ringX is the one word
  // every step needs (score-table offset of the column's symbol pair); ringA carries the rest for EDGE
  // steps (target-gap penalties, which change at a target's last column: align_simd.cpp:1741-1751)
  __shared__ uint32_t ringX[FAST_WARPS][2 * RING];
  __shared__ uint2 ringA[FAST_WARPS][2 * RING];

  int const lane = threadIdx.x & 31;
  int const wib = threadIdx.x >> 5;

  if (!PROF) {
    // negated (non-negative) substitution scores, both halves looked up at once
    for (int e = threadIdx.x; e < LUT_WORDS; e += blockDim.x) {
      if (GENERAL) {
        int const q = e >> 8, dlo = e & 15, dhi = (e >> 4) & 15;
        lut[e] = pk2(-sp.S[dlo][q], -sp.S[dhi][q]);
      } else {
        int const ent = e >> 5;  // replicated for the 32 lanes: word = ent*32 + lane
        int const q = 1 << (ent >> 4), dlo = 1 << (ent & 3), dhi = 1 << ((ent >> 2) & 3);
        lut[e] = pk2(-sp.S[dlo][q], -sp.S[dhi][q]);
      }
    }
    __syncthreads();
  }

  int const w = blockIdx.x * FAST_WARPS + wib;
  if (w >= ntasks) { return; }
  FastTask const tk = tasks[w];
  if (WRITE == CK_RERUN) {
    // every half of a score-only task is a follower (leader_of >= 0); it needs its walk unless its leader was accepted
    bool need = false;
    if (tk.out_lo >= 0) { need |= stats[static_cast<size_t>(leader_of[tk.out_lo]) * VSG_STAT_WORDS + VSG_STAT_CIGARLEN] != TB_VERDICT_ACCEPTED; }
    if (tk.out_hi >= 0) { need |= stats[static_cast<size_t>(leader_of[tk.out_hi]) * VSG_STAT_WORDS + VSG_STAT_CIGARLEN] != TB_VERDICT_ACCEPTED; }
    if (!need) { return; }
    if (rerun_count != nullptr && lane == 0) { atomicAdd(rerun_count, 1); }
  }

  int const Q = qs.len[tk.q];
  uint8_t const * __restrict__ qsym = qs.sym + qs.off[tk.q];
  int const Dlo = ts.len[tk.tlo], Dhi = ts.len[tk.thi];
  uint8_t const * __restrict__ dlo_p = ts.sym + ts.off[tk.tlo];
  uint8_t const * __restrict__ dhi_p = ts.sym + ts.off[tk.thi];
  int const dmax = tk.dmax;
  int const nsteps = dmax + 31;

  int const QRqi = sp.go[Q_I] + sp.ge[Q_I], Rqi = sp.ge[Q_I];
  int const QRqr = sp.go[Q_R] + sp.ge[Q_R], Rqr = sp.ge[Q_R];
  int const QRti = sp.go[T_I] + sp.ge[T_I], Rti = sp.ge[T_I];
  int const QRtr = sp.go[T_R] + sp.ge[T_R], Rtr = sp.ge[T_R];
  int const gotl = sp.go[T_L], getl = sp.ge[T_L];
  int const goql = sp.go[Q_L], geql = sp.ge[Q_L];

  int const llast = (Q - 1) / R;
  int const rlast = (Q - 1) % R;
  int score_lo = 0, score_hi = 0;

  uint32_t * const rX = ringX[wib];
  uint2 * const rA = ringA[wib];
  uint32_t const lut_s = static_cast<uint32_t>(__cvta_generic_to_shared(lut));
  uint32_t const rX_s = static_cast<uint32_t>(__cvta_generic_to_shared(rX));
  uint32_t const rA_s = static_cast<uint32_t>(__cvta_generic_to_shared(rA));
  uint4 * const myprof = prof_mem + static_cast<size_t>(wib) * 16 * RQ * 32 + lane;
  uint32_t const prof_s = static_cast<uint32_t>(__cvta_generic_to_shared(myprof));

  int const row0 = lane * R;
  // per-row state and constants: H of the previous column, E entering the current one, the row's
  // query-gap penalties (right-end values on the query's last row, align_simd.cpp:861-868 / 890-897)
  uint32_t Hl[R], E[R], nQRq[R], Rq[R], rowoff[PROF ? 1 : R];
#pragma unroll
  for (int r = 0; r < R; r++) {
    int const i = row0 + r;
    bool const last = (i == Q - 1);
    nQRq[r] = pk1(-(last ? QRqr : QRqi));   // per-half negation: the addend of the fused add+max
    Rq[r] = pk1(last ? Rqr : Rqi);
    Hl[r] = BIAS2 - pk1(gotl + (i + 1) * getl);                    // H(i,-1)   (align_simd.cpp:852-853)
    E[r] = Hl[r] - pk1(last ? QRqr : QRqi);                        // E(i,0)    (align_simd.cpp:855-857)
    asm volatile("" : "+r"(nQRq[r]), "+r"(Rq[r]));
  }
  if (PROF) {
    // rows beyond the query's end score like 'A' (their cells are never read)
    int code[RQ * 4];
#pragma unroll
    for (int r = 0; r < RQ * 4; r++) {
      int const i = row0 + r;
      code[r] = (r < R && i < Q) ? (1 << code_to_2bit(qsym[i] & 15)) : 1;
    }
    for (int tp = 0; tp < 16; tp++) {
      int const dlo = 1 << (tp & 3), dhi = 1 << (tp >> 2);
#pragma unroll
      for (int r4 = 0; r4 < RQ; r4++) {
        uint4 v;
        v.x = pk2(-sp.S[dlo][code[4 * r4 + 0]], -sp.S[dhi][code[4 * r4 + 0]]);
        v.y = pk2(-sp.S[dlo][code[4 * r4 + 1]], -sp.S[dhi][code[4 * r4 + 1]]);
        v.z = pk2(-sp.S[dlo][code[4 * r4 + 2]], -sp.S[dhi][code[4 * r4 + 2]]);
        v.w = pk2(-sp.S[dlo][code[4 * r4 + 3]], -sp.S[dhi][code[4 * r4 + 3]]);
        myprof[(tp * RQ + r4) * 32] = v;   // read back by this lane only: no barrier needed
      }
    }
  } else {
#pragma unroll
    for (int r = 0; r < R; r++) {
      int const i = row0 + r;
      int const code = (i < Q) ? (qsym[i] & 15) : (GENERAL ? 0 : 1);
      rowoff[r] = lut_s + (GENERAL ? static_cast<uint32_t>(code) * 1024u
                                   : (static_cast<uint32_t>(code_to_2bit(code)) * 16u * 32u + lane) * 4u);
      asm volatile("" : "+r"(rowoff[r]));
    }
  }
  // H(row0-1,-1): the diagonal input of this lane's first row at column 0
  uint32_t diag_in = (row0 == 0) ? BIAS2 : BIAS2 - pk1(gotl + row0 * getl);
  uint32_t Hout = BIAS2, Fout = BIAS2;
  uint2 * const myrow = rowck + tk.dir_off;
  uint2 * const mycol = colck + tk.bnd_off;
  bool const capture = (lane == llast);

  // the recurrence of this lane's R rows for one column.  yneg = -(QR_t) per half (fused add+max),
  // z = R_t (plain subtract); hin/fin = H and F handed down by the lane above (lane 0: the top boundary)
  auto column = [&](uint32_t x, uint32_t yneg, uint32_t z, uint32_t hin, uint32_t fin) {
    uint32_t t[R];
    if (PROF) {
      uint32_t const pa = prof_s + x;
#pragma unroll
      for (int r4 = 0; r4 < RQ; r4++) {
        uint4 const S4 = lds128(pa + r4 * 512u);
        uint32_t const Sv[4] = {S4.x, S4.y, S4.z, S4.w};
#pragma unroll
        for (int u = 0; u < 4; u++) {
          int const r = 4 * r4 + u;
          if (r < R) { t[r] = (r == 0 ? diag_in : Hl[r - 1]) - Sv[u]; }
        }
      }
    } else {
#pragma unroll
      for (int r = 0; r < R; r++) { t[r] = (r == 0 ? diag_in : Hl[r - 1]) - lds32(rowoff[r] + x); }
    }
    uint32_t F = fin;
#pragma unroll
    for (int r = 0; r < R; r++) {
      uint32_t const h = __vimax3_u16x2(t[r], F, E[r]);
      Hl[r] = h;
      F = __viaddmax_u16x2(h, yneg, F - z);
      E[r] = __viaddmax_u16x2(h, nQRq[r], E[r] - Rq[r]);
    }
    Hout = Hl[R - 1];
    Fout = F;
    diag_in = hin;
  };

  // the column record of column cc, written by lane (cc & 31) during a refill
  auto make_record = [&](int cc, int a, int b, uint32_t & x, uint2 & yz) {
    x = GENERAL ? static_cast<uint32_t>(a + 16 * b) * 4u
                : static_cast<uint32_t>(code_to_2bit(a) + 4 * code_to_2bit(b)) * (PROF ? RQ * 512u : 128u);
    yz.x = pk2(-(cc >= Dlo - 1 ? QRtr : QRti), -(cc >= Dhi - 1 ? QRtr : QRti));
    yz.y = pk2(cc >= Dlo - 1 ? Rtr : Rti, cc >= Dhi - 1 ? Rtr : Rti);
  };
  // symbols of the column this lane will publish at the next refill (one chunk ahead of their use)
  int nxt_a = 0, nxt_b = 0;
  auto fetch = [&](int cc) {
    nxt_a = (cc < Dlo) ? (dlo_p[cc] & 15) : 0;
    nxt_b = (cc < Dhi) ? (dhi_p[cc] & 15) : 0;
  };
  if (lane < ckpt::CHUNK && lane < dmax) { fetch(lane); }

  int const cap_lo = Dlo - 1 + llast, cap_hi = Dhi - 1 + llast;
  uint32_t const geql2 = pk1(geql);
  for (int s0 = 0; s0 < nsteps; s0 += ckpt::CHUNK) {
    {
      // publish columns [s0, s0+CHUNK): one column per lane; then start loading the next chunk's symbols
      __syncwarp();
      int const cc = s0 + lane;
      if (lane < ckpt::CHUNK && cc < dmax) {
        uint32_t x; uint2 yz;
        make_record(cc, nxt_a, nxt_b, x, yz);
        int const slot = cc & (RING - 1);
        rX[slot] = x; rX[slot + RING] = x;
        rA[slot] = yz; rA[slot + RING] = yz;
      }
      __syncwarp();
      if (lane < ckpt::CHUNK && cc + ckpt::CHUNK < dmax) { fetch(cc + ckpt::CHUNK); }
    }
    uint32_t const slot0 = static_cast<uint32_t>(s0 - lane) & (RING - 1);
    // STEADY chunk: all 32 lanes inside the matrix, no score to pick up, and the target-gap penalties
    // uniform over the chunk's columns (neither target's last column is inside [s0-31, s0+31])
    constexpr unsigned CH = ckpt::CHUNK;
    bool const steady = (s0 >= 32) && (s0 + ckpt::CHUNK - 1 < dmax) &&
                        (static_cast<unsigned>(cap_lo - s0) >= CH) && (static_cast<unsigned>(cap_hi - s0) >= CH) &&
                        (static_cast<unsigned>(Dlo - 1 - (s0 - 31)) >= 31u + CH) && (static_cast<unsigned>(Dhi - 1 - (s0 - 31)) >= 31u + CH);
    if (steady) {
      bool const lo_done = (s0 - 31 > Dlo - 1), hi_done = (s0 - 31 > Dhi - 1);
      uint32_t const yneg = pk2(-(lo_done ? QRtr : QRti), -(hi_done ? QRtr : QRti));
      uint32_t const z = pk2(lo_done ? Rtr : Rti, hi_done ? Rtr : Rti);
      uint32_t const ypos = pk2(lo_done ? QRtr : QRti, hi_done ? QRtr : QRti);
      // lane 0's top boundary, kept arithmetically: H(-1,c) = -(go + (c+1)*ge)   (align_simd.cpp:1895-1901)
      uint32_t htop = BIAS2 - pk1(goql + (s0 - lane + 1) * geql);
      uint32_t aX = rX_s + slot0 * 4u;
      auto step = [&](uint32_t ax) {
        uint32_t hin = __shfl_up_sync(0xffffffffu, Hout, 1);
        uint32_t fin = __shfl_up_sync(0xffffffffu, Fout, 1);
        uint32_t const x = lds32(ax);
        if (lane == 0) { hin = htop; fin = htop - ypos; }          // F(0,c) = H(-1,c) - QR_t  (align_simd.cpp:830-833)
        htop -= geql2;
        column(x, yneg, z, hin, fin);
      };
      if (STORE) {
#pragma unroll 1
        for (int k0 = 0; k0 < ckpt::CHUNK; k0 += 4) {
          uint32_t ho[4], fo[4];
#pragma unroll
          for (int u = 0; u < 4; u++) {
            step(aX + (k0 + u) * 4u);
            ho[u] = Hout; fo[u] = Fout;
          }
          uint4 * const tp = reinterpret_cast<uint4 *>(myrow + ckpt::row_index(s0 + k0, lane));
          tp[0] = make_uint4(ho[0], fo[0], ho[1], fo[1]);
          tp[1] = make_uint4(ho[2], fo[2], ho[3], fo[3]);
        }
      } else {
        // nothing to stage: eight steps per trip, the ring address the only per-trip arithmetic
#pragma unroll 1
        for (int k0 = 0; k0 < ckpt::CHUNK; k0 += CK_SO_STEPS, aX += CK_SO_STEPS * 4u) {
#pragma unroll
          for (int u = 0; u < CK_SO_STEPS; u++) { step(aX + u * 4u); }
        }
      }
    } else {
      int const kend = min(ckpt::CHUNK, nsteps - s0);
      int c = s0 - lane;
      uint32_t aX = rX_s + slot0 * 4u, aA = rA_s + slot0 * 8u;
      for (int k = 0; k < kend; k++, c++, aX += 4u, aA += 8u) {
        uint32_t hin = __shfl_up_sync(0xffffffffu, Hout, 1);
        uint32_t fin = __shfl_up_sync(0xffffffffu, Fout, 1);
        if (c >= 0 && c < dmax) {
          uint32_t const x = lds32(aX);
          uint2 yz;
          asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(yz.x), "=r"(yz.y) : "r"(aA));
          if (lane == 0) {
            hin = BIAS2 - pk1(goql + (c + 1) * geql);
            fin = __vadd2(hin, yz.x);
          }
          column(x, yz.x, yz.y, hin, fin);
          if (STORE) { myrow[ckpt::row_index(s0 + k, lane)] = make_uint2(Hout, Fout); }
          if (capture && (c == Dlo - 1 || c == Dhi - 1)) {
            uint32_t v = 0;
#pragma unroll
            for (int r = 0; r < R; r++) { if (r == rlast) { v = Hl[r]; } }
            if (c == Dlo - 1) { score_lo = static_cast<int>(v & 0xffffu) - static_cast<int>(BIAS); }
            if (c == Dhi - 1) { score_hi = static_cast<int>(v >> 16) - static_cast<int>(BIAS); }
          }
        }
      }
    }
    // column checkpoint at the chunk's end (state after step s0 + 31); the last chunk needs none
    if (STORE && s0 + ckpt::CHUNK < nsteps) {
      uint2 * const cp = mycol + ckpt::col_index(s0 / ckpt::CHUNK + 1, lane, 0, R);
#pragma unroll
      for (int r = 0; r < R; r++) { cp[static_cast<size_t>(r) * 32] = make_uint2(Hl[r], E[r]); }
    }
  }
  if (WRITE != CK_RERUN && lane == llast) {
    // undo the anti-diagonal shift of the scoring (header comment): H = H2 + shift * (Q + D)
    if (tk.out_lo >= 0) { stats[static_cast<size_t>(tk.out_lo) * VSG_STAT_WORDS + VSG_STAT_SCORE] = score_lo + sp.shift * (Q + Dlo); }
    if (tk.out_hi >= 0) { stats[static_cast<size_t>(tk.out_hi) * VSG_STAT_WORDS + VSG_STAT_SCORE] = score_hi + sp.shift * (Q + Dhi); }
  }
}

// ---------------------------------------------------------------------------------------------
// traceback over regenerated tiles (tb_ckpt.h): one thread per pair, the tile's direction bits in
// shared memory (word-interleaved by thread: every thread owns one bank)
// ---------------------------------------------------------------------------------------------

constexpr int TB_CK_THREADS = 128;

template <int NW>
struct SmemBits {
  uint32_t * base;   // this thread's first word
  __device__ __forceinline__ void set(int bj, int k, uint32_t v) { base[(bj * NW + k) * TB_CK_THREADS] = v; }
  __device__ __forceinline__ uint32_t get(int bj, int k) const { return base[(bj * NW + k) * TB_CK_THREADS]; }
  __device__ __forceinline__ void stage_word(int bj, const uint8_t * t, int, int mis, int wi)
  {
    uint32_t const dst = static_cast<uint32_t>(__cvta_generic_to_shared(base + (bj * NW) * TB_CK_THREADS));
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" :: "r"(dst), "l"(reinterpret_cast<const uint32_t *>(t - mis) + wi) : "memory");
  }
  __device__ __forceinline__ void wait() { asm volatile("cp.async.wait_all;" ::: "memory"); }
};

// Row checkpoints of one tile staged in shared memory: the (at most ten) 32-byte sectors that hold the tile's
// steps are copied with cp.async — all in flight at once, no registers — into a thread-interleaved array
// (vector v of thread t at [v][t]: every thread owns its own 16-byte bank group, so the divergent reads of a
// warp's 32 unrelated walks never conflict).
constexpr int TB_CK_ROWVECS = 2 * ((ckpt::CHUNK + 8) / 4);   // sectors of CHUNK + 2 steps at any alignment, x 2 x 16 bytes
struct SmemRows {
  const uint2 * rowck;   // the task's row checkpoints
  uint4 * base;          // this thread's vector 0
  int sa = 0;            // first staged step (a multiple of 4)
  __device__ __forceinline__ void stage(int l, int s0, int s1)
  {
    int const g0 = s0 >> 2;
    int const g1 = s1 >> 2;
    sa = s0 & ~3;
    const char * src = reinterpret_cast<const char *>(rowck + ckpt::row_index(s0 & ~3, l));
    uint32_t dst = static_cast<uint32_t>(__cvta_generic_to_shared(base));
    for (int g = g0; g <= g1; g++) {
      asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" :: "r"(dst), "l"(src) : "memory");
      asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" :: "r"(dst + TB_CK_THREADS * 16u), "l"(src + 16) : "memory");
      src += 32 * 4 * sizeof(uint2);
      dst += 2u * TB_CK_THREADS * 16u;
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  __device__ __forceinline__ void wait() { asm volatile("cp.async.wait_all;" ::: "memory"); }
  __device__ __forceinline__ ckpt::U2 get(int s) const
  {
    int const srel = s - sa;   // vector srel / 2 holds steps srel & ~1 and (srel & ~1) + 1
    uint2 const v = *reinterpret_cast<const uint2 *>(reinterpret_cast<const char *>(base + (srel >> 1) * TB_CK_THREADS) + (srel & 1) * 8);
    return ckpt::U2{v.x, v.y};
  }
};

constexpr size_t tb_ck_smem(int RT)
{
  return static_cast<size_t>(ckpt::CHUNK) * (RT / 8) * TB_CK_THREADS * 4 + static_cast<size_t>(TB_CK_ROWVECS) * TB_CK_THREADS * 16;
}

template <int RT, bool TEXT>
__device__ __forceinline__ void traceback_ckpt_one(const ScoreParams & sp, const DevSeqs & qs, const DevSeqs & ts,
                                                   uint32_t q, uint32_t t, int out, int R, int half, int general,
                                                   const uint2 * __restrict__ rowck, const uint2 * __restrict__ colck,
                                                   char * __restrict__ cigar_region, int32_t * __restrict__ stats,
                                                   unsigned char * smem)
{
  int32_t * const st = stats + static_cast<size_t>(out) * VSG_STAT_WORDS;
  ckpt::PairView pv;
  pv.rowck = reinterpret_cast<const ckpt::U2 *>(rowck);
  pv.colck = reinterpret_cast<const ckpt::U2 *>(colck);
  pv.R = R; pv.half = half; pv.Q = qs.len[q]; pv.D = ts.len[t]; pv.general = general;
  pv.q = qs.sym + qs.off[q];
  pv.t = ts.sym + ts.off[t];
  SmemRows rows{rowck, reinterpret_cast<uint4 *>(smem) + threadIdx.x};
  SmemBits<RT / 8> bits{reinterpret_cast<uint32_t *>(smem + static_cast<size_t>(TB_CK_ROWVECS) * TB_CK_THREADS * 16) + threadIdx.x};
  CigarWriter cw;
  cw.text = TEXT;
  cw.end = TEXT ? (cigar_region + pv.Q + pv.D + 1) : nullptr;
  if (TEXT) { *--cw.end = 0; }
  cw.op = 0; cw.run = 0; cw.len = 0;
  ckpt::TbOut o;
  auto emit = [&](char nop, int n) { if (TEXT) { cw.push_n(nop, n); } };
  if (general) { ckpt::traceback<RT, true>(sp, pv, bits, rows, o, emit); }
  else { ckpt::traceback<RT, false>(sp, pv, bits, rows, o, emit); }
  if (TEXT) { cw.flush(); }
  st[VSG_STAT_ALIGNED] = o.aligned; st[VSG_STAT_MATCHES] = o.matches; st[VSG_STAT_MISMATCHES] = o.mismatches;
  st[VSG_STAT_GAPS] = o.gaps; st[VSG_STAT_TRIM_LEFT] = o.trim_left; st[VSG_STAT_TRIM_RIGHT] = o.trim_right;
  st[VSG_STAT_CIGARLEN] = TEXT ? cw.len : 0;
}

// statistics-only, straight from the forward tasks: pair 2k / 2k+1 = first / second target of task k.  One thread
// per pair: thread i walks pair i (gate.ids[i] when the launch is gated), and the lanes of a warp run their walks'
// rounds together until the last of them is done.
// TRACEBACK ON DEMAND (the batched search driver).  align_delayed hands search16 a group of up to eight candidates of
// a query and then examines them in order until the accept / reject limits are reached (searchcore.cpp:780-880): when
// the first one is accepted and that accept is the last one wanted, the other seven alignments are never looked at.
// Their DP is computed here like every other pair's (it is the work the metric counts), but their walk back through
// the matrix is not: the group's LEADER is walked first (phase 1; its thread also stores the verdict of
// search_acceptable_aligned's identity test next to its statistics), the FOLLOWERS afterwards (phase 2), and a follower
// whose leader was accepted leaves its statistics "not computed" (all bits set).  The verdict is taken with a small
// margin, so a borderline leader just means walked followers; the host replay re-aligns a pair it needs and finds
// not computed (search.cu), which keeps the results independent of this shortcut.
// Score-only tasks (CK_SCOREONLY above) hold followers only: they have no checkpoints until the CK_RERUN launch between
// the two phases has written those of the tasks phase 2 will walk.
struct TbGate {
  const int * ids;            // pair ids (2 * task + half) this launch handles, nids of them; nullptr = all pairs of the tasks
  int nids;
  const int32_t * leader_of;  // per pair slot: slot of its leader, -1 = none (a leader, or not gated); nullptr = no gating
  int phase;                  // 1: leaders (store the verdict), 2: followers (skip when the leader was accepted)
  int iddef;                  // --iddef
  double threshold;           // 100 * --id + margin
};

// the identity of align_trim + search_acceptable_aligned's test for a hit with the default optional filters
// (hit_logic.h finish_hit / acceptable_aligned, searchcore.cpp:409-463, 664-737)
__device__ __forceinline__ bool tb_leader_accepted(const ckpt::TbOut & o, int Q, int D, int iddef, double threshold)
{
  int const nal = o.aligned, ma = o.matches, mi = o.mismatches, ga = o.gaps;
  int const tql = o.trim_left > 0 ? o.trim_left : 0, ttl = o.trim_left < 0 ? -o.trim_left : 0;
  int tqr = o.trim_right > 0 ? o.trim_right : 0, ttr = o.trim_right < 0 ? -o.trim_right : 0;
  if (tql >= nal) { tqr = 0; }
  if (ttl >= nal) { ttr = 0; }
  int const internal = nal - (tql + ttl + tqr + ttr);
  int const shortest = Q < D ? Q : D, longest = Q < D ? D : Q;
  double id;
  switch (iddef) {
    case 0: id = shortest > 0 ? 100.0 * ma / shortest : 0.0; break;
    case 2: id = internal > 0 ? 100.0 * ma / internal : 0.0; break;
    case 3: { double const v = 100.0 * (1.0 - (1.0 * (mi + ga) / longest)); id = v > 0.0 ? v : 0.0; break; }
    default: id = nal > 0 ? 100.0 * ma / nal : 0.0; break;   // 1 and 4
  }
  return ma > 0 && id >= threshold;
}

template <int RT, bool GENERAL>
__device__ __forceinline__ void traceback_ckpt_tasks_body(const ScoreParams & sp, const DevSeqs & qs, const DevSeqs & ts,
                                                          const FastTask * __restrict__ tasks, int ntasks, int R,
                                                          const uint2 * __restrict__ rowck, const uint2 * __restrict__ colck,
                                                          int32_t * __restrict__ stats, const TbGate & gate, unsigned char * smem)
{
  int const total = gate.ids != nullptr ? gate.nids : 2 * ntasks;
  int const p = blockIdx.x * blockDim.x + threadIdx.x;
  SmemRows rows{nullptr, reinterpret_cast<uint4 *>(smem) + threadIdx.x};
  SmemBits<RT / 8> bits{reinterpret_cast<uint32_t *>(smem + static_cast<size_t>(TB_CK_ROWVECS) * TB_CK_THREADS * 16) + threadIdx.x};
  auto emit = [](char, int) {};
  ckpt::Walk<RT, GENERAL> w;
  int out = -1;
  int myQ = 0, myD = 0;
  bool active = false;
  if (p < total) {
    int const id = gate.ids != nullptr ? gate.ids[p] : p;
    FastTask const tk = tasks[id >> 1];
    int const half = id & 1;
    out = half ? tk.out_hi : tk.out_lo;
    active = out >= 0;
    if (active && gate.leader_of != nullptr && gate.phase == 2) {
      int const lead = gate.leader_of[out];
      active = !(lead >= 0 && stats[static_cast<size_t>(lead) * VSG_STAT_WORDS + VSG_STAT_CIGARLEN] == TB_VERDICT_ACCEPTED);
    }
    if (active) {
      uint32_t const q = tk.q, t = half ? tk.thi : tk.tlo;
      ckpt::PairView pv;
      pv.rowck = reinterpret_cast<const ckpt::U2 *>(rowck + tk.dir_off);
      pv.colck = reinterpret_cast<const ckpt::U2 *>(colck + tk.bnd_off);
      pv.R = R; pv.half = half; pv.Q = qs.len[q]; pv.D = ts.len[t]; pv.general = GENERAL ? 1 : 0;
      pv.q = qs.sym + qs.off[q];
      pv.t = ts.sym + ts.off[t];
      myQ = pv.Q; myD = pv.D;
      rows.rowck = rowck + tk.dir_off;
      w.start(pv);
    }
  }
  while (__any_sync(0xffffffffu, active)) {
    if (active) {
      if (w.running()) { w.round(sp, bits, rows, emit); }
      if (!w.running()) {
        ckpt::TbOut o;
        w.finish(o, emit);
        int32_t * const st = stats + static_cast<size_t>(out) * VSG_STAT_WORDS;
        st[VSG_STAT_ALIGNED] = o.aligned; st[VSG_STAT_MATCHES] = o.matches; st[VSG_STAT_MISMATCHES] = o.mismatches;
        st[VSG_STAT_GAPS] = o.gaps; st[VSG_STAT_TRIM_LEFT] = o.trim_left; st[VSG_STAT_TRIM_RIGHT] = o.trim_right;
        st[VSG_STAT_CIGARLEN] = (gate.leader_of != nullptr && gate.phase == 1 && tb_leader_accepted(o, myQ, myD, gate.iddef, gate.threshold))
                                    ? TB_VERDICT_ACCEPTED : 0;
        active = false;
      }
    }
  }
}

template <int RT>
__global__ void __launch_bounds__(TB_CK_THREADS)
traceback_ckpt_tasks_kernel(const __grid_constant__ ScoreParams sp, DevSeqs qs, DevSeqs ts,
                            const FastTask * __restrict__ tasks, int ntasks, int R, int general,
                            const uint2 * __restrict__ rowck, const uint2 * __restrict__ colck,
                            int32_t * __restrict__ stats, TbGate gate)
{
  extern __shared__ __align__(16) unsigned char tb_smem[];
  if (general) { traceback_ckpt_tasks_body<RT, true>(sp, qs, ts, tasks, ntasks, R, rowck, colck, stats, gate, tb_smem); }
  else { traceback_ckpt_tasks_body<RT, false>(sp, qs, ts, tasks, ntasks, R, rowck, colck, stats, gate, tb_smem); }
}

// with CIGAR text, from pair descriptors (PD_CKPT = checkpoint layout; the others belong to traceback_kernel)
template <int RT>
__global__ void __launch_bounds__(TB_CK_THREADS)
traceback_ckpt_pairs_kernel(const __grid_constant__ ScoreParams sp, DevSeqs qs, DevSeqs ts,
                            const PairDesc * __restrict__ pairs, int npairs,
                            const uint2 * __restrict__ rowck, const uint2 * __restrict__ colck,
                            char * __restrict__ cigar_scratch, int32_t * __restrict__ stats)
{
  extern __shared__ __align__(16) unsigned char tb_smem[];
  int const p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npairs) { return; }
  PairDesc const pd = pairs[p];
  if (pd.kind != PD_CKPT || (RT == 8) != (pd.R <= 8)) { return; }
  traceback_ckpt_one<RT, true>(sp, qs, ts, pd.q, pd.t, pd.out, pd.R, pd.half & 1, pd.half >> 1,
                               rowck + pd.dir_off, colck + pd.aux_off, cigar_scratch + pd.cigar_off, stats, tb_smem);
}

}  // namespace vsg
