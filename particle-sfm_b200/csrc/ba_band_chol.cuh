// ba_band_chol.cuh — the reduced camera system of a VIDEO (banded + arrow) solved by one CTA (or two).
//
// Exact-Schur mode (reference rule for <= 1000 images, bundle_adjustment.cc:276-286; Ceres
// SchurComplementSolver semantics, SURVEY.md A.6): S y = rhs with S = 6F x 6F banded (half
// bandwidth bw = 6 * track span + 5) plus an "arrow" of the shared camera's 3 intrinsics slots.
// The factorisation is a chain of 6F dependent pivots: what bounds it is the latency of one
// pivot step, not flops (~4 MFLOP) — grid barriers through L2 (the round-1 kernel,
// k_chol_blocked: 38 panels x ~1.5 us) or cluster barriers (~380 cycles) are the wrong tool.
// Here the whole active window lives in the REGISTERS of one CTA:
//
//   k_band_assemble  band blocks + per-image sums -> compact scaled band matrix Ab (each entry
//                    written exactly once; the dense (6F+3)^2 S is never formed or zeroed)
//   k_band_chol6     right-looking Cholesky on a sliding window of Wb 6 x 6 image blocks (W = 6 Wb > bw,
//                    3 <= Wb <= 25), one BLOCK pivot per step: block index I lives at ring position I mod Wb,
//                    the symmetric window is held as unordered pairs of positions {P, Q}, a tile of one 6 x 6
//                    block per worker thread.  Workers, panel group and loader each run their OWN small loop
//                    (named barriers from different program counters; see the comment above the kernel).
//                    The 4 arrow rows (3 intrinsics + the rhs, so that L^-1 b falls out of the same sweep)
//                    are one more block row of the window.  Then L' x = y by warp 0 in axpy form (per pivot:
//                    one multiply, one shuffle, one fma on the chain), the rows of L staged chunk-wise into
//                    shared memory by the other warps (bc_tail).
//                    TWO-SIDED form (gridDim.x = 2, matrices of >= 4 windows): the chain of nb dependent
//                    pivots is cut in two.  CTA 0 factors the leading k0 pivots of A top-down, CTA 1
//                    the trailing n1 pivots bottom-up (the same code on the index-reversed matrix);
//                    the W rows in between (W > bw, so no top pivot touches a bottom pivot: the two
//                    eliminations commute) collect both Schur updates — CTA 1 hands its update of
//                    that W x W block, of the arrow and of the corner over through global memory,
//                    CTA 0 adds it to its register window and finishes the last W pivots and the
//                    corner.  The back substitution mirrors it: CTA 0 solves the middle rows first
//                    and releases them, then both CTAs walk outwards.  Same arithmetic per pivot as
//                    the one-sided form, different (but fixed) elimination order.
// Block windows wider than 25 images, and systems of fewer than 3 images, go to the dense S + k_chol_blocked route.
#pragma once
#include "ba_schur_explicit.cuh"

namespace psfm {
namespace ba {

constexpr int BC_MAXSLOT = 7;     // 1 + ceil(bw / 32) register slots of the back substitution

// Split of the pivot chain (band_chol_plan): one-sided (two = 0) or two-sided.
struct BandPlan {
  int nb, bw, W, RS;        // nb multiple of 6, W = 6 Wb with 3 <= Wb <= 25 (W = 0: no band plan)
  int two;                  // 1: two CTAs
  int k0, n1;               // pivots factored top-down before the hand-over | bottom-up; k0 + W + n1 = nb
  int nbs[2];               // rows of the matrix each side sees: k0 + W | n1 + W   (one-sided: nb | 0)
  int npiv[2];              // pivots each side factors:           k0 + W | n1       (one-sided: nb | 0)
  int rows[2];              // rows of Ab each side may touch (band_chol_rows)
};

struct BandAsmArgs2 {
  const double* Sband;      // [F][span + 1][36] all-reduced pair-block sums
  const double* lin_cam;    // [F][NVL]  F'F rot (6) | t (6) | ...
  const double* lin_intr;   // [C][NVI]
  const double* prep_intr;  // [C][NVI]
  const double* xcam;       // [F][xstride] rot-t cross (9) | F'G (6) | -(W H~) Wk' (6) | ...
  int xstride;
  const double* scale_c;    // [NS]
  const double* Dc2;        // [NS]
  const double* rhs;        // [NS]
  const unsigned char* active;
  int F, span;
  BandPlan pl;
  double* Ab;               // side 0 [rows[0]][RS]: Ab[r][k] = A[r][r - k] (k <= bw), Ab[r][W + a] = A[nb + a][r], a < 3; Ab[r][W + 3] = rhs[r]
  double* Ab1;              // side 1 [rows[1]][RS]: the same of the index-reversed matrix, middle block and middle arrow zero
  double* C4;               // [2][4][4] arrow corner: intrinsics block (3 x 3) | rhs entries in row / column 3; side 1: zero
  int* fail;                // cleared here, set by k_band_chol6
};

// packed index of element (r, c) of a symmetric 3 x 3 stored as 00 01 02 11 12 22
__device__ __forceinline__ int sym3(int r, int c) {
  const int lo = min(r, c), hi = max(r, c);
  return lo * (5 - lo) / 2 + hi;
}

// scaled reduced-system element A[r][r - e] of the band part (0 <= e <= bw, r - e >= 0), identity below nb
__device__ __forceinline__ double band_entry(const BandAsmArgs2& a, int r, int e) {
  if (r >= a.pl.nb) return e == 0 ? 1.0 : 0.0;
  const int c = r - e;
  double v = 0.0;
  const int ia = r / 6, rr = r % 6, ib = c / 6, cc = c % 6, d = ia - ib;
  const double ss = a.scale_c[r] * a.scale_c[c];
  if (d <= a.span)     // lower element (r, c): mirror of the stored upper block (ib, ib + d)
    v = -ss * a.Sband[((size_t)ib * (a.span + 1) + d) * 36 + (d ? 6 * cc + rr : 6 * rr + cc)];
  if (d == 0) {
    const double* A = a.lin_cam + (size_t)ia * NVL;
    if (rr < 3) v += ss * A[sym3(rr, cc)];                                   // cc <= rr < 3
    else if (cc >= 3) v += ss * A[6 + sym3(rr - 3, cc - 3)];
    else v += ss * a.xcam[(size_t)ia * a.xstride + 3 * cc + (rr - 3)];     // (Jr' Jt)[cc][rr - 3]
    if (e == 0) { if (a.active[r]) v += a.Dc2[r]; else v = 1.0; }
  }
  return v;
}
// arrow entry aa of column r: A[nb + aa][r] (aa < 3) | rhs[r] (aa = 3); zero below nb
__device__ __forceinline__ double arrow_entry(const BandAsmArgs2& a, int r, int aa) {
  if (r >= a.pl.nb) return 0.0;
  if (aa == 3) return a.rhs[r];
  if (aa == 0) {
    const double* X = a.xcam + (size_t)(r / 6) * a.xstride;
    return a.scale_c[r] * a.scale_c[6 * (size_t)a.F] * (X[9 + r % 6] + X[15 + r % 6]);
  }
  return 0.0;
}

__global__ void k_band_assemble(const BandAsmArgs2 a) {
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const BandPlan& pl = a.pl;
  if (t == 0) *a.fail = 0;
  if (t < 32) {   // corner (camera 0: intrinsics are only ever free for a single shared camera); side 1 starts from zero
    const int r = ((int)t & 15) / 4, c = (int)t % 4;
    const size_t sk = 6 * (size_t)a.F;
    double v = 0.0;
    if (t < 16) {
      if (r < 3 && c < 3) {
        v = a.scale_c[sk + r] * a.scale_c[sk + c] * (a.lin_intr[sym3(r, c)] + a.prep_intr[sym3(r, c)]);
        if (r == c) { if (a.active[sk + r]) v += a.Dc2[sk + r]; else v = 1.0; }
      } else if (r == 3 && c < 3) v = a.rhs[sk + c];
      else if (c == 3 && r < 3) v = a.rhs[sk + r];
    }
    a.C4[t] = v;
  }
  const int RS = pl.RS, W = pl.W;
  const size_t n0 = (size_t)pl.rows[0] * RS, n1 = (size_t)pl.rows[1] * RS;
  if (t < n0) {
    const int r = (int)(t / RS), e = (int)(t % RS);
    double v = 0.0;
    if (r >= min(pl.nb, pl.nbs[0])) {
      v = (e == 0) ? 1.0 : 0.0;                       // identity padding below the part this side factors
    } else if (e < W) {
      if (e <= pl.bw && r - e >= 0) v = band_entry(a, r, e);
    } else {
      v = arrow_entry(a, r, e - W);
    }
    a.Ab[t] = v;
  } else if (t < n0 + n1) {
    // index-reversed matrix B[r'][c'] = A[nb-1-r'][nb-1-c']: its lower element (r', r' - e) is the
    // lower element (R, R - e) of A with R = nb - 1 - (r' - e).  Rows / columns >= n1 are the middle
    // block, which side 0 owns: zero here, so that what is left in the window is the pure update.
    const size_t u = t - n0;
    const int r = (int)(u / RS), e = (int)(u % RS);
    double v = 0.0;
    if (r >= pl.nbs[1]) {
      v = (e == 0) ? 1.0 : 0.0;
    } else if (e < W) {
      const int c = r - e;
      if (e <= pl.bw && c >= 0 && !(r >= pl.n1 && c >= pl.n1)) v = band_entry(a, pl.nb - 1 - c, e);
    } else if (r < pl.n1) {
      v = arrow_entry(a, pl.nb - 1 - r, e - W);
    }
    a.Ab1[u] = v;
  }
}

struct BandSide {
  const double* Ab;
  const double* C4;
  int nb, npiv;             // rows of this side's matrix | pivots it factors (multiple of 6)
  double* Lr;               // [nb][bw + 1]  UNNORMALISED columns: Lr[r][k] = A~[r][r - k] (= L[r][r - k] sqrt(d[r - k]))
  double* La;               // [4][nb]       unnormalised arrow rows (row 3 = rhs)
  double* dinv;             // [nb]          pivots d[j], replaced by 1 / sqrt(d[j]) after the factorisation
};

struct BandCholArgs {
  BandSide s[2];            // blockIdx.x = side
  // two-sided | value of the sync flags for this launch | rows of the whole matrix | pivots of side 0 before the
  // hand-over.  The field order matters to k_band_chol6's register allocation under its 128-register cap: with
  // bw .. ns at other offsets, ptxas spilled inside the factorisation loop of the 512-thread 3 x 3 instantiation.
  int two, epoch, nb, k0;
  int bw, W, RS, ns;        // ns: length of x (slots past nb + 3 — other cameras — are zeroed)
  double* x;                // [ns]
  int* fail;                // OR of both sides (cleared by k_band_assemble)
  double* D;                // hand-over of side 1: [W][W] update of the middle block (A orientation) | [4][W] arrow | [16] corner
  int* sync;                // [2] = epoch once: 0 the hand-over is written, 1 the middle x and the intrinsics are written
};

__device__ __forceinline__ void bc_post(int* flag, int v) {
  __threadfence();
  asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(flag), "r"(v) : "memory");
}
__device__ __forceinline__ void bc_wait(const int* flag, int v) {
  int x;
  do {
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(x) : "l"(flag) : "memory");
  } while (x != v);
}

// 1 / d to full double precision (not correctly rounded): MUFU seed + two Newton steps — about
// half the dependent latency of the IEEE division, which sits on the pivot-to-pivot chain
__device__ __forceinline__ double bc_rcp(double d) {
  double r;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(d));
  double e = fma(-d, r, 1.0);
  r = fma(r, e, r);
  e = fma(-d, r, 1.0);
  return fma(r, e, r);
}

// Everything after the factorisation: normalisation, the 3 x 3 arrow corner (s_c4: the 4 x 4 corner block of the
// window, written to shared memory by its owner before the caller's barrier), hand-shake of the two-sided form, back
// substitution.  Called by every thread of the CTA.
__device__ __forceinline__ void bc_tail(const BandCholArgs& a, const BandSide& sd, const int side, double* stage, int& s_fail,
                                        double* s_xI, const double* s_c4) {
  const int tid = threadIdx.x, lane = tid & 31;
  const int nb = sd.nb, npiv = sd.npiv, bw = a.bw, LS = bw + 1;
  // 1 / sqrt(d): normalisation of the stored columns, applied while staging the back substitution
  for (int j = tid; j < npiv; j += blockDim.x) sd.dinv[j] = rsqrt(__ldcg(sd.dinv + j));
  // ---- arrow corner: 3 x 3 intrinsics block and its right-hand side (thread of block {Wb, Wb})
  if (side == 0 && tid == 0) {
    bool cbad = false;
    const double m00 = s_c4[0], m10 = s_c4[4], m20 = s_c4[8], m11 = s_c4[5], m21 = s_c4[9], m22 = s_c4[10];
    cbad |= !(m00 > 0.0);
    const double l00 = sqrt(m00), l10 = m10 / l00, l20 = m20 / l00;
    double t = m11 - l10 * l10;
    cbad |= !(t > 0.0);
    const double l11 = sqrt(t), l21 = (m21 - l20 * l10) / l11;
    t = m22 - l20 * l20 - l21 * l21;
    cbad |= !(t > 0.0);
    const double l22 = sqrt(t);
    const double z0 = s_c4[12] / l00, z1 = (s_c4[13] - l10 * z0) / l11, z2 = (s_c4[14] - l20 * z0 - l21 * z1) / l22;
    const double x2 = z2 / l22, x1 = (z1 - l21 * x2) / l11, x0 = (z0 - l10 * x1 - l20 * x2) / l00;
    s_xI[0] = x0; s_xI[1] = x1; s_xI[2] = x2;
    if (cbad || !isfinite(x0 + x1 + x2)) s_fail = 1;
  }
  __syncthreads();
  if (tid == 0 && s_fail) atomicOr(a.fail, 1);
  if (side == 0) {
    if (s_fail) {
      if (a.two && tid == 0) bc_post(a.sync + 1, a.epoch);     // side 1 must not wait for ever
      return;
    }
    for (int s = a.nb + tid; s < a.ns; s += blockDim.x) a.x[s] = (s < a.nb + 3) ? s_xI[s - a.nb] : 0.0;
  } else {
    // the middle x and the intrinsics come from side 0
    if (tid == 0) {
      bc_wait(a.sync + 1, a.epoch);
      for (int k = 0; k < 3; ++k) s_xI[k] = __ldcg(a.x + a.nb + k);
    }
    __syncthreads();
  }

  // ---- back substitution L' x = y - La' x_I in axpy form (warp 0; the other warps stage).
  //      Lane l holds the running right-hand side of positions 32 (c - m) + l, m = 0 .. msv-1, of the
  //      current 32-column chunk c.  stage[jj][32 + k] = -L[r][r - k] for 1 <= k <= bw (r = 32 c + jj),
  //      zero elsewhere, so the inner step is one shared load and one fma per slot — no predicates;
  //      per pivot one fma, one shuffle and one fma are on the dependent chain.  Rows >= npiv (side 1:
  //      the middle rows) are not solved for: their x is known and only propagated.
  const int ms = 1 + (bw + 31) / 32;
  const int msv = ms <= 4 ? 4 : BC_MAXSLOT;
  const int LSP = 32 * (msv + 1);
  const int ctop = (nb + 31) / 32 - 1;
  const int cpost = (a.two && side == 0) ? a.k0 / 32 : -1;     // after this chunk every middle x is written
  const int CH = 32 * LSP;
  // one row per warp and pass; all loads of a row (<= 7 x 2 per lane) are issued before the first use — with a
  // dependent load pair per element the staging, not the substitution chain, set the pace (measured: 7.5 k cycles
  // per 32-row chunk against 1.3 k for the chain)
  auto stage_chunk = [&](int c, double* buf, int w0, int nw) {
    // RP rows per pass: with 8 warps a warp stages ~5 rows of a chunk, one global-memory latency each would outlast
    // the substitution chain of the chunk
    constexpr int RP = 2;
    for (int j0 = w0; j0 < 32; j0 += RP * nw) {
      double lv[RP][BC_MAXSLOT], dv[RP][BC_MAXSLOT];
#pragma unroll
      for (int h = 0; h < RP; ++h) {
        const int jj = j0 + h * nw, r = 32 * c + jj;
#pragma unroll
        for (int t = 0; t < BC_MAXSLOT; ++t) {
          const int k = lane + 32 * t;                       // element q = 32 (t + 1) + lane of the padded row
          const bool ok = jj < 32 && t < msv && k >= 1 && k <= bw && r < nb && r - k >= 0 && r - k < npiv;
          lv[h][t] = ok ? __ldcg(sd.Lr + (size_t)r * LS + k) : 0.0;
          dv[h][t] = ok ? __ldcg(sd.dinv + r - k) : 0.0;
        }
      }
#pragma unroll
      for (int h = 0; h < RP; ++h) {
        const int jj = j0 + h * nw;
        if (jj < 32) {
          buf[jj * LSP + lane] = 0.0;
#pragma unroll
          for (int t = 0; t < BC_MAXSLOT; ++t)
            if (t < msv) buf[jj * LSP + 32 * (t + 1) + lane] = -lv[h][t] * dv[h][t];
        }
      }
    }
  };
  const double xi0 = s_xI[0], xi1 = s_xI[1], xi2 = s_xI[2];
  auto y0 = [&](int i) -> double {
    if (i < 0 || i >= npiv) return 0.0;
    return __ldcg(sd.dinv + i) * (__ldcg(sd.La + 3 * (size_t)nb + i) -
           (xi0 * __ldcg(sd.La + i) + xi1 * __ldcg(sd.La + (size_t)nb + i) + xi2 * __ldcg(sd.La + 2 * (size_t)nb + i)));
  };
  const int wid = tid >> 5, nwarp = blockDim.x >> 5;
  stage_chunk(ctop, stage, wid, nwarp);
  double yy[BC_MAXSLOT];
#pragma unroll
  for (int m = 0; m < BC_MAXSLOT; ++m) yy[m] = (tid < 32 && m < ms) ? y0(32 * (ctop - m) + lane) : 0.0;
  __syncthreads();
  for (int c = ctop, n = 0; c >= 0; --c, ++n) {
    const double* buf = stage + (n & 1) * CH;
    if (tid >= 32) {
      if (c > 0) stage_chunk(c - 1, stage + ((n + 1) & 1) * CH, wid - 1, nwarp - 1);
    } else {
      const double fresh = (c > 0) ? y0(32 * (c - ms) + lane) : 0.0;     // slot ms - 1 of the next chunk
      const int jl = 32 * c + lane;
      const double dl = (jl < npiv) ? __ldcg(sd.dinv + jl) : 0.0;
      // global index of local row jl: side 0 jl, side 1 a.nb - 1 - jl; rows >= this side's nb (last chunk) write nothing
      const int gl = side ? a.nb - 1 - jl : jl;
      const bool inx = jl < nb && gl >= 0 && gl < a.nb;
      const double xk = (jl >= npiv && inx) ? __ldcg(a.x + gl) : 0.0;   // known x (side 1: middle rows)
      const bool wr = jl < npiv && inx;
      double* xw = a.x + (inx ? gl : 0);
      const double* rp = buf + 31 * LSP + 32 + (31 - lane);             // &stage[jj][32 + jj - lane], jj = 31
      const int step = LSP + 1;
      if (msv == 4) {
#pragma unroll 8
        for (int jj = 31; jj >= 0; --jj) {
          const double xj = __shfl_sync(0xffffffffu, fma(yy[0], dl, xk), jj);
#pragma unroll
          for (int m = 0; m < 4; ++m) yy[m] = fma(rp[32 * m], xj, yy[m]);
          if (lane == jj && wr) *xw = xj;
          rp -= step;
        }
      } else {
#pragma unroll 4
        for (int jj = 31; jj >= 0; --jj) {
          const double xj = __shfl_sync(0xffffffffu, fma(yy[0], dl, xk), jj);
#pragma unroll
          for (int m = 0; m < BC_MAXSLOT; ++m) yy[m] = fma(rp[32 * m], xj, yy[m]);
          if (lane == jj && wr) *xw = xj;
          rp -= step;
        }
      }
#pragma unroll
      for (int m = 0; m < BC_MAXSLOT; ++m) yy[m] = (m == ms - 1) ? fresh : ((m + 1 < BC_MAXSLOT) ? yy[m + 1] : 0.0);
      if (c == cpost) __threadfence();
    }
    __syncthreads();
    if (c == cpost && tid == 0) bc_post(a.sync + 1, a.epoch);
  }
}

// ------------------------------------------------------------------ block-6 Cholesky with look-ahead (k_band_chol6)
//
// A scalar pivot per CTA barrier costs ~450 cycles (measured: ~65 instructions per lone worker warp and one barrier
// for 16 FMAs per thread).  The reduced camera system is made of 6 x 6 image blocks, so the natural unit is a
// BLOCK pivot: per step k one 6 x 6 diagonal block is factored, the 6-column panel below it solved and the
// trailing window updated with a rank-6 product — one barrier per six pivots, and the two dependent chains
// (factor + solve of the next panel | rank-6 update of the window) run side by side in different warps:
//   workers   one thread per unordered pair {P, Q} of ring POSITIONS (block index I lives at position I mod Wb,
//             position Wb = the arrow rows), the 6 x 6 block T{P,Q}[a][b] = S[6 I_P + a][6 I_Q + b] in registers.
//             Step k (pivot position c): every block that touches neither c nor cn = c + 1 takes the rank-6 update
//             with panel k (shared memory); blocks touching c are dead (their content was panel k) and reload the
//             incoming block row k + Wb straight from global memory — a full step ahead of their next use;
//             blocks touching cn are dormant: the panel group carries that column.  At the end of the step the
//             blocks touching cn2 = c + 2 (updated through pivot k) are published for the panel group.
//   panel     one thread per row (position, a) of the next pivot column: takes the published row (or, for a freshly
//             recycled position, the raw row it prefetched from global memory), applies update k itself (its own
//             row of L_k is still in its registers), the 6 rows of the diagonal block are shared, EVERY panel
//             thread factors the 6 x 6 block redundantly (LDL' recurrence: reciprocal, not square root, on the
//             chain) and solves its own row on the fly; the normalised row goes to shared memory for the next
//             step, the unnormalised one to global memory in the layout bc_tail expects.
// One barrier of the 6 - 8 participating warps per step (bar.sync 1), one among the 3 - 5 panel warps (bar.sync 2);
// the remaining warps of the CTA only exist for the back substitution's staging and sleep at the final barrier.
// Phases end with a FLUSH step (no next panel: the workers update the dormant blocks too), after which the whole
// window is current: that is where the two-sided form hands over and where a phase restarts.
// Dataflow emulated block-wise against numpy before it was written (see DESIGN.md); tests/test_gpu_band_chol.py.
constexpr int B6_PBS = 38;        // doubles per 6 x 6 panel block in shared memory (304 bytes: the blocks of eight
                                  // consecutive positions start in eight different groups of four banks)

// Named barriers from role-specific loops: every participating thread executes the same NUMBER of barriers, from
// different program counters.  One warp runs dependent scalar code at several cycles per instruction, so what a role
// does per step is counted in instructions — all roles interleaved in one unrolled body, index arithmetic per pivot,
// was measured several times slower per pivot.  Hence: per-role loops, no early exit.
__device__ __forceinline__ void bc_gbar(int n) { asm volatile("bar.sync 1, %0;\n" ::"r"(n) : "memory"); }
__device__ __forceinline__ void bc_pbar(int n) { asm volatile("bar.sync 2, %0;\n" ::"r"(n) : "memory"); }

template <int MAXT, int TR, int TC>
__global__ void __launch_bounds__(MAXT, 1) k_band_chol6(const BandCholArgs a) {
  // TR x TC: tile of a worker thread inside a 6 x 6 block (6 x 6: one thread per block; 3 x 6: two; 3 x 3: four).  A warp issues
  // about one instruction per several cycles whatever the dependences (measured with clock64 per role), so a step costs
  // what its LONGEST warp executes — many thin threads beat few fat ones as long as the CTA has room for them.
  extern __shared__ __align__(16) double bc_smem[];
  __shared__ int s_fail;
  __shared__ double s_xI[4];
  __shared__ double s_c4[16];
  constexpr int TPB = (6 / TR) * (6 / TC);
  const int side = blockIdx.x;
  BandSide sd;
  sd.Ab = side ? a.s[1].Ab : a.s[0].Ab; sd.C4 = side ? a.s[1].C4 : a.s[0].C4;
  sd.nb = side ? a.s[1].nb : a.s[0].nb; sd.npiv = side ? a.s[1].npiv : a.s[0].npiv;
  sd.Lr = side ? a.s[1].Lr : a.s[0].Lr; sd.La = side ? a.s[1].La : a.s[0].La; sd.dinv = side ? a.s[1].dinv : a.s[0].dinv;
  const int W = a.W, Wb = W / 6, RS = a.RS, nb = sd.nb, LS = a.bw + 1;
  const int nsteps = sd.npiv / 6;
  const int jsw = (a.two && side == 0) ? a.k0 / 6 : -1;
  const int tid = threadIdx.x;
  const int nblk = (Wb + 1) * (Wb + 2) / 2;
  const int NWT = nblk * TPB;                   // worker threads
  const int NW = (NWT + 31) & ~31;
  const int NPR = 6 * (Wb + 1), NP = (NPR + 31) & ~31;
  const int NG = NW + NP;
  const int NG2 = (int)blockDim.x;       // the step barrier includes the loader warps (all remaining warps of the CTA)
  const int PB = (Wb + 1) * B6_PBS;
  // panel of step k in buffer k & 1, UNNORMALISED: Y = rows of the reduced pivot column (y), Z = y / d — the update is
  // T -= Z_P Y_Q', no square root anywhere in the loop (bc_tail normalises what goes to the back substitution)
  double* Ypan = bc_smem;               // [2][PB]
  double* Zpan = Ypan + 2 * PB;         // [2][PB]
  double* Raw = Zpan + 2 * PB;          // [2][PB] rows of the next pivot column, published at the end of step k in buffer k & 1
  double* Raw0 = Raw + 2 * PB;          // [PB]    rows of the pivot column a phase starts with
  double* Dsh = Raw0 + PB;              // [36]    diagonal block being factored
  double* ring = Dsh + 36;              // [4][6 RS] incoming block rows: slot k & 3 holds block row k + Wb (raw rows of Ab) during step k
  const int RB = 6 * RS;
  const double* __restrict__ Ab = sd.Ab;
  if (tid == 0) s_fail = 0;
  bool bad = false;
  const int kb0 = 0, ke0 = jsw >= 0 ? jsw : nsteps;     // phase 0; phase 1 (two-sided, side 0): jsw .. nsteps

  if (tid < NW) {
    // ------------------------------------------------------------ workers
    const bool act = tid < NWT;
    const int blk = tid / TPB, sub = tid % TPB;
    const int sr = TR * (sub / (6 / TC)), sc = TC * (sub % (6 / TC));   // tile origin inside the 6 x 6 block
    int P = 0, Q = 0;
    if (act) {
      P = (int)((sqrtf(8.f * (float)blk + 1.f) - 1.f) * 0.5f);
      while ((P + 1) * (P + 2) / 2 <= blk) ++P;
      while (P * (P + 1) / 2 > blk) --P;
      Q = blk - P * (P + 1) / 2;
    }
    double T[TR][TC];
#pragma unroll
    for (int i = 0; i < TR; ++i)
#pragma unroll
      for (int k = 0; k < TC; ++k) {
        double x = 0.0;
        const int bi = sr + i, bk = sc + k;
        if (act) {
          if (P < Wb) {
            const int r = 6 * P + bi, c = 6 * Q + bk, hi = max(r, c), lo = min(r, c);
            x = __ldg(Ab + (size_t)hi * RS + (hi - lo));
          } else if (Q < Wb) { if (bi < 4) x = __ldg(Ab + (size_t)(6 * Q + bk) * RS + W + bi); }
          else if (bi < 4 && bk < 4) x = __ldg(sd.C4 + 4 * bi + bk);
        }
        T[i][k] = x;
      }
    // rows of pivot column `pos` held by this tile -> dst[row position][a][0..5]
    auto publish = [&](double* dst, int pos) {
      if (Q == pos) {
        double* o = dst + P * B6_PBS + 6 * sr + sc;
#pragma unroll
        for (int i = 0; i < TR; ++i)
#pragma unroll
          for (int k = 0; k < TC; ++k) o[6 * i + k] = T[i][k];
      } else if (P == pos) {
        double* o = dst + Q * B6_PBS + 6 * sc + sr;
#pragma unroll
        for (int k = 0; k < TC; ++k)
#pragma unroll
          for (int i = 0; i < TR; ++i) o[6 * k + i] = T[i][k];
      }
    };
    // T -= Z_P Y_Q' with the panel in shared memory (rows of 6 doubles, 16-byte aligned)
    auto update = [&](const double* Yb, const double* Zb) {
      const double2* lq = reinterpret_cast<const double2*>(Yb + Q * B6_PBS + 6 * sc);
      const double2* lp = reinterpret_cast<const double2*>(Zb + P * B6_PBS + 6 * sr);
      double q[TC][6];
#pragma unroll
      for (int k = 0; k < TC; ++k)
#pragma unroll
        for (int m = 0; m < 3; ++m) { const double2 z = lq[3 * k + m]; q[k][2 * m] = z.x; q[k][2 * m + 1] = z.y; }
#pragma unroll
      for (int i = 0; i < TR; ++i) {
        double pr[6];
#pragma unroll
        for (int m = 0; m < 3; ++m) { const double2 z = lp[3 * i + m]; pr[2 * m] = z.x; pr[2 * m + 1] = z.y; }
#pragma unroll
        for (int k = 0; k < TC; ++k)
#pragma unroll
          for (int m = 0; m < 6; ++m) T[i][k] = fma(-pr[m], q[k][m], T[i][k]);
      }
    };
    // position c takes block row k + Wb (raw entries: no pivot <= k reaches it), staged in ring slot k & 3 by the
    // loader warp; cn = (k + 1) mod Wb holds block k + 1
    auto recycle = [&](int k, int c, int cn) {
      const int rn = 6 * (k + Wb);
      const double* rg = ring + (k & 3) * RB;            // rg[i * RS + e] = A[rn + i][rn + i - e]
      if (P == c && Q == c) {
#pragma unroll
        for (int i = 0; i < TR; ++i)
#pragma unroll
          for (int kk = 0; kk < TC; ++kk) {
            const int bi = sr + i, bk = sc + kk;
            T[i][kk] = rg[max(bi, bk) * RS + (bi > bk ? bi - bk : bk - bi)];
          }
      } else if (P == Wb) {
#pragma unroll
        for (int i = 0; i < TR; ++i)
#pragma unroll
          for (int kk = 0; kk < TC; ++kk) T[i][kk] = (sr + i < 4) ? rg[(sc + kk) * RS + W + sr + i] : 0.0;
      } else {
        const int o = (P == c) ? Q : P;
        int dI = o - cn; if (dI < 0) dI += Wb;
        const int ro = 6 * (k + 1 + dI);
        if (P == c) {
#pragma unroll
          for (int i = 0; i < TR; ++i)
#pragma unroll
            for (int kk = 0; kk < TC; ++kk) T[i][kk] = rg[(sr + i) * RS + (rn + sr + i - ro - sc - kk)];
        } else {
#pragma unroll
          for (int i = 0; i < TR; ++i)
#pragma unroll
            for (int kk = 0; kk < TC; ++kk) T[i][kk] = rg[(sc + kk) * RS + (rn + sc + kk - ro - sr - i)];
        }
      }
    };
    // column block k of the factor (panel k, unnormalised) -> global memory in the layout bc_tail reads; one
    // element per worker thread and pass (the workers have slack: the panel group is the longer chain)
    auto output = [&](int k, int c) {
      const double* Yb = Ypan + (k & 1) * PB;
      const int jb = 6 * k;
      for (int v = tid; v < 36 * (Wb + 1); v += NW) {
        const int p = v / 36, e = v - 36 * p, ar = e / 6, m = e - 6 * ar;
        const double y = Yb[p * B6_PBS + e];
        if (p == c) {
          if (m <= ar) sd.Lr[(size_t)(jb + ar) * LS + (ar - m)] = y;
          if (m == ar) sd.dinv[jb + ar] = y;
        } else if (p < Wb) {
          int dI = p - c; if (dI < 0) dI += Wb;
          const int rr = 6 * (k + dI) + ar, kk = rr - jb - m;
          if (rr < nb && kk < LS) sd.Lr[(size_t)rr * LS + kk] = y;          // beyond bw: structurally zero
        } else if (ar < 4) {
          sd.La[(size_t)ar * nb + jb + m] = y;
        }
      }
    };
#pragma unroll 1
    for (int phase = 0; phase < 2; ++phase) {
      const int kb = phase == 0 ? kb0 : jsw, ke = phase == 0 ? ke0 : nsteps;
      if (phase == 1) {
        if (jsw < 0) break;
        // two-sided form: the window is current through pivot k0 - 1; add side 1's update of the same rows
        if (tid == 0) bc_wait(a.sync, a.epoch);
        bc_gbar(NG2);
        if (act) {
          const int cb = jsw % Wb;
          const double* DA = a.D + (size_t)W * W;
          int dP = P - cb; if (dP < 0) dP += Wb;
          int dQ = Q - cb; if (dQ < 0) dQ += Wb;
#pragma unroll
          for (int i = 0; i < TR; ++i)
#pragma unroll
            for (int k = 0; k < TC; ++k) {
              const int bi = sr + i, bk = sc + k;
              if (P < Wb) T[i][k] += __ldcg(a.D + (size_t)(6 * dP + bi) * W + 6 * dQ + bk);
              else if (Q < Wb) { if (bi < 4) T[i][k] += __ldcg(DA + (size_t)bi * W + 6 * dQ + bk); }
              else if (bi < 4 && bk < 4) T[i][k] += __ldcg(DA + 4 * (size_t)W + 4 * bi + bk);
            }
        }
      }
      // (re)start: the whole window is current; hand the pivot column and the next one to the panel group
      int c = kb % Wb;
      {
        const int cn = c + 1 == Wb ? 0 : c + 1;
        if (act) {
          publish(Raw0, c);
          if (P != c && Q != c) publish(Raw + ((kb - 1) & 1) * PB, cn);
        }
        bc_gbar(NG2);
        bc_gbar(NG2);
      }
#pragma unroll 1
      for (int k = kb; k < ke; ++k) {
        const bool last = k == ke - 1;
        const int cn = c + 1 == Wb ? 0 : c + 1, cn2 = cn + 1 == Wb ? 0 : cn + 1;
        if (act) {
          const bool ic = (P == c || Q == c), icn = (P == cn || Q == cn);
          if (ic) { if (!icn || last) recycle(k, c, cn); }
          else if (!icn || last) update(Ypan + (k & 1) * PB, Zpan + (k & 1) * PB);
          if (!last && !ic && !icn && (P == cn2 || Q == cn2)) publish(Raw + (k & 1) * PB, cn2);
        }
        output(k, c);
        bc_gbar(NG2);
        c = cn;
      }
    }
    if (act && a.two && side == 1) {
      // hand-over: what is left in the window (rows n1 .. n1 + W - 1 of the reversed matrix, zero on input) is the
      // update of the middle block by this side's pivots; reversed row n1 + m is middle row W - 1 - m
      const int cb = nsteps % Wb;
      double* DA = a.D + (size_t)W * W;
      int dP = P - cb; if (dP < 0) dP += Wb;
      int dQ = Q - cb; if (dQ < 0) dQ += Wb;
#pragma unroll
      for (int i = 0; i < TR; ++i)
#pragma unroll
        for (int k = 0; k < TC; ++k) {
          const int bi = sr + i, bk = sc + k;
          const int mk = W - 1 - (6 * dQ + bk);
          if (P < Wb) {
            const int mi = W - 1 - (6 * dP + bi);
            a.D[(size_t)mi * W + mk] = T[i][k];
            if (P != Q) a.D[(size_t)mk * W + mi] = T[i][k];
          } else if (Q < Wb) { if (bi < 4) DA[(size_t)bi * W + mk] = T[i][k]; }
          else if (bi < 4 && bk < 4) DA[4 * (size_t)W + 4 * bi + bk] = T[i][k];
        }
    }
    if (act && blk == nblk - 1) {
#pragma unroll
      for (int i = 0; i < TR; ++i)
#pragma unroll
        for (int k = 0; k < TC; ++k)
          if (sr + i < 4 && sc + k < 4) s_c4[4 * (sr + i) + sc + k] = T[i][k];
    }
  } else if (tid < NG) {
    // ------------------------------------------------------------ panel group: thread = row (position p, a)
    const int r = tid - NW;
    const bool pact = r < NPR;
    const int p = pact ? r / 6 : 0, ar = pact ? r % 6 : 0;
    double yo[6] = {0, 0, 0, 0, 0, 0};     // own row of the current panel (unnormalised)
    int kre = -1;                         // step at which this thread's position was recycled last (in this phase)
    // raw row ar of block row kr + Wb (ring slot kr & 3) against column block j: A[r][6 j + m], r = 6 (kr + Wb) + ar
    auto ring_row = [&](int kr, int j, double (&dst)[6]) {
      const double* rg = ring + (kr & 3) * RB + ar * RS + (6 * (kr + Wb) + ar - 6 * j);
#pragma unroll
      for (int m = 0; m < 6; ++m) dst[m] = rg[-m];
    };
    // col = row (p, ar) of the fully updated pivot column block at position cp: factor the diagonal block (LDL'
    // recurrence, every thread redundantly: one reciprocal per pivot on the chain), solve the row on the fly,
    // publish y and z = y / d
    auto finish = [&](int cp, double (&col)[6], double* Ydst, double* Zdst) {
      if (pact && p == cp) {
        double2* o = reinterpret_cast<double2*>(Dsh + 6 * ar);
#pragma unroll
        for (int m = 0; m < 6; m += 2) o[m >> 1] = make_double2(col[m], col[m + 1]);
      }
      bc_pbar(NP);
      double Dl[6][6], w[6][6], invd[6];
      {
        double dfull[36];
        const double2* dd = reinterpret_cast<const double2*>(Dsh);
#pragma unroll
        for (int t = 0; t < 18; ++t) { const double2 z = dd[t]; dfull[2 * t] = z.x; dfull[2 * t + 1] = z.y; }
#pragma unroll
        for (int i = 0; i < 6; ++i)
#pragma unroll
          for (int j = 0; j <= i; ++j) Dl[i][j] = dfull[6 * i + j];
      }
      const bool diag = p == cp;
      double z[6];
#pragma unroll
      for (int j = 0; j < 6; ++j) {
        const double dj = Dl[j][j];
        bad |= !(dj > 0.0 && dj <= 1.7976931348623157e308);
        invd[j] = bc_rcp(dj);
#pragma unroll
        for (int i = j + 1; i < 6; ++i) w[i][j] = Dl[i][j] * invd[j];
#pragma unroll
        for (int i = j + 1; i < 6; ++i)
#pragma unroll
          for (int i2 = j + 1; i2 <= i; ++i2) Dl[i][i2] = fma(-Dl[i][j], w[i2][j], Dl[i][i2]);
        // row solve, column j: y_j = col_j - sum_{n < j} y_n w[j][n]
        double t = col[j];
#pragma unroll
        for (int n = 0; n < j; ++n) t = fma(-yo[n], w[j][n], t);
        if (diag && j > ar) t = 0.0;       // upper part of the diagonal block
        yo[j] = t;
        z[j] = t * invd[j];
      }
      if (pact) {
        double2* oy = reinterpret_cast<double2*>(Ydst + p * B6_PBS + 6 * ar);
        double2* oz = reinterpret_cast<double2*>(Zdst + p * B6_PBS + 6 * ar);
#pragma unroll
        for (int m = 0; m < 6; m += 2) { oy[m >> 1] = make_double2(yo[m], yo[m + 1]); oz[m >> 1] = make_double2(z[m], z[m + 1]); }
      }
    };
#pragma unroll 1
    for (int phase = 0; phase < 2; ++phase) {
      const int kb = phase == 0 ? kb0 : jsw, ke = phase == 0 ? ke0 : nsteps;
      if (phase == 1) {
        if (jsw < 0) break;
        bc_gbar(NG2);
      }
      int c = kb % Wb;
      kre = -1;
      bc_gbar(NG2);
      {
        double col[6];
#pragma unroll
        for (int m = 0; m < 6; ++m) col[m] = pact ? Raw0[p * B6_PBS + 6 * ar + m] : 0.0;
        finish(c, col, Ypan + (kb & 1) * PB, Zpan + (kb & 1) * PB);
      }
      bc_gbar(NG2);
#pragma unroll 1
      for (int k = kb; k < ke; ++k) {
        const bool last = k == ke - 1;
        const int cn = c + 1 == Wb ? 0 : c + 1;
        if (!last) {
          double col[6];
          const bool useA = pact && p == c && p < Wb;          // recycled in this step: row of block k + Wb, no update
          if (useA) { ring_row(k, k + 1, col); kre = k; }
          else if (pact && kre == k - 1 && kre >= 0) ring_row(k - 1, k + 1, col);   // recycled in the previous step
          else {
            const double2* rawp = reinterpret_cast<const double2*>(Raw + ((k - 1) & 1) * PB + p * B6_PBS + 6 * ar);
#pragma unroll
            for (int m = 0; m < 3; ++m) { const double2 v = rawp[m]; col[2 * m] = pact ? v.x : 0.0; col[2 * m + 1] = pact ? v.y : 0.0; }
          }
          if (!useA) {
            const double2* Zcn = reinterpret_cast<const double2*>(Zpan + (k & 1) * PB + cn * B6_PBS);
#pragma unroll
            for (int m = 0; m < 6; ++m) {
              double t = col[m];
#pragma unroll
              for (int n = 0; n < 3; ++n) { const double2 v = Zcn[3 * m + n]; t = fma(-yo[2 * n], v.x, t); t = fma(-yo[2 * n + 1], v.y, t); }
              col[m] = t;
            }
          }
          finish(cn, col, Ypan + ((k + 1) & 1) * PB, Zpan + ((k + 1) & 1) * PB);
        }
        bc_gbar(NG2);
        c = cn;
      }
    }
  } else {
    // ------------------------------------------------------------ loader warps: block row k + Wb of Ab -> ring slot k & 3,
    //      one step before it is used, loaded from global memory one step before that (registers in between)
    const int lt = tid - NG, nl = (int)blockDim.x - NG;
    const int maxblk = nsteps - 1 + Wb;                  // last block row anybody reads
    constexpr int LPT = 12;                              // double2 per loader thread: 32 loaders x 12 x 2 = 768 >= 6 RS up to Wb = 20, 64 loaders for all
    double2 rg[LPT];
    auto ld = [&](int blk) {
      const double2* src = reinterpret_cast<const double2*>(Ab + (size_t)6 * blk * RS);
#pragma unroll
      for (int u = 0; u < LPT; ++u) {
        const int e = lt + u * nl;
        rg[u] = (blk <= maxblk && 2 * e < RB) ? __ldg(src + e) : make_double2(0.0, 0.0);
      }
    };
    auto st_ = [&](int slot) {
      double2* dst = reinterpret_cast<double2*>(ring + slot * RB);
#pragma unroll
      for (int u = 0; u < LPT; ++u) {
        const int e = lt + u * nl;
        if (2 * e < RB) dst[e] = rg[u];
      }
    };
#pragma unroll 1
    for (int phase = 0; phase < 2; ++phase) {
      const int kb = phase == 0 ? kb0 : jsw, ke = phase == 0 ? ke0 : nsteps;
      if (phase == 1) {
        if (jsw < 0) break;
        bc_gbar(NG2);
      }
      ld(kb + Wb); st_(kb & 3);
      ld(kb + 1 + Wb);
      bc_gbar(NG2);
      bc_gbar(NG2);
#pragma unroll 1
      for (int k = kb; k < ke; ++k) {
        st_((k + 1) & 3);
        ld(k + 2 + Wb);
        bc_gbar(NG2);
      }
    }
  }
  if (a.two && side == 1) __threadfence();
  __syncthreads();
  if (bad) s_fail = 1;
  if (a.two && side == 1 && tid == 0) bc_post(a.sync, a.epoch);
  __syncthreads();
  bc_tail(a, sd, side, bc_smem, s_fail, s_xI, s_c4);
}

// shared memory of the back substitution's staging (bc_tail): two chunks of 32 rows of LSP doubles
inline size_t band_chol_smem(int bw) {
  const int ms = 1 + (bw + 31) / 32, msv = ms <= 4 ? 4 : BC_MAXSLOT;
  return sizeof(double) * (2 * 32 * (size_t)(32 * (msv + 1)));
}

// rows of Ab the kernel may touch (padding rows below the band part are identity rows)
inline int band_chol_rows(int nb, int W) { return ((nb + 7) & ~7) + W + 8; }

// Plan of k_band_chol6, or W = 0 when the matrix has no block-6 plan (the caller takes the dense route): nb must be
// a multiple of 6 of at least 3 blocks and the block window at most 25 blocks, unless it covers the whole matrix.
// How the pivot chain is cut: two-sided from 4 windows on (below that the hand-over costs more than the shorter chain
// saves); PSFM_CHOL_ONE_SIDED forces the one-CTA form.
// blk_span >= 0: blocks further apart than blk_span are zero (the reduced camera system: blk_span = longest image
// span of a track); -1: only the scalar half bandwidth bw is known.
inline BandPlan band_chol_plan(int nb, int bw, int blk_span = -1) {
  BandPlan p{};
  p.nb = nb; p.bw = std::min(bw, nb - 1);
  static const bool one = getenv("PSFM_CHOL_ONE_SIDED") != nullptr;
  // window in blocks: every block at distance >= Wb from the pivot block must be zero
  int Wb = blk_span >= 0 ? blk_span + 1 : (p.bw + 5) / 6 + 1;
  if (nb % 6 != 0 || nb / 6 < 3) return p;
  Wb = std::max(3, std::min(Wb, nb / 6));
  if (Wb > 25 || 6 * Wb <= p.bw) return p;
  const int F = nb / 6;
  p.W = 6 * Wb; p.RS = p.W + 4;
  p.two = (!one && F >= 4 * Wb) ? 1 : 0;
  if (p.two) {
    p.k0 = 6 * ((F - Wb) / 2);
    p.n1 = nb - p.W - p.k0;
    p.nbs[0] = p.k0 + p.W; p.npiv[0] = p.k0 + p.W;
    p.nbs[1] = p.n1 + p.W; p.npiv[1] = p.n1;
    p.rows[0] = band_chol_rows(p.nbs[0], p.W); p.rows[1] = band_chol_rows(p.nbs[1], p.W);
  } else {
    p.nbs[0] = nb; p.npiv[0] = nb; p.rows[0] = band_chol_rows(nb, p.W);
  }
  return p;
}

// device buffers of one plan
struct BandWork {
  BandPlan pl{};
  DBuf<double> Ab, C4, Lr, La, dinv, D;
  DBuf<int> sync;
  int epoch = 0;
  void alloc(const BandPlan& p, cudaStream_t st) {
    pl = p;
    const size_t LS = p.bw + 1;
    Ab.alloc((size_t)(p.rows[0] + p.rows[1]) * p.RS, st);
    C4.alloc(32, st);
    Lr.alloc((size_t)(p.nbs[0] + p.nbs[1]) * LS, st); Lr.zero(st);
    La.alloc(4 * (size_t)(p.nbs[0] + p.nbs[1]), st);
    dinv.alloc((size_t)p.nbs[0] + p.nbs[1], st);
    D.alloc((size_t)p.W * p.W + 4 * (size_t)p.W + 16, st);
    sync.alloc(2, st); sync.zero(st);
    epoch = 0;
  }
  double* ab(int side) { return Ab.p + (side ? (size_t)pl.rows[0] * pl.RS : 0); }
  BandCholArgs args(double* x, int ns, int* fail) {
    BandCholArgs c{};
    const size_t LS = pl.bw + 1;
    for (int s = 0; s < 2; ++s) {
      const size_t o = s ? (size_t)pl.nbs[0] : 0;
      c.s[s].Ab = ab(s); c.s[s].C4 = C4.p + 16 * s; c.s[s].nb = pl.nbs[s]; c.s[s].npiv = pl.npiv[s];
      c.s[s].Lr = Lr.p + o * LS; c.s[s].La = La.p + 4 * o; c.s[s].dinv = dinv.p + o;
    }
    c.two = pl.two; c.nb = pl.nb; c.k0 = pl.k0;
    c.bw = pl.bw; c.W = pl.W; c.RS = pl.RS; c.ns = ns;
    c.x = x; c.fail = fail; c.D = D.p; c.sync = sync.p; c.epoch = ++epoch;
    return c;
  }
};

// one launch: one CTA, or two for the two-sided form
inline void band_chol_launch(const BandCholArgs& c, cudaStream_t st) {
  const int grid = c.two ? 2 : 1;
  const int Wb = c.W / 6, nblk = (Wb + 1) * (Wb + 2) / 2;
  const int np = (6 * (Wb + 1) + 31) & ~31;
  const int ng4 = ((4 * nblk + 31) & ~31) + np, ng1 = ((nblk + 31) & ~31) + np;
  const size_t fact = sizeof(double) * (7 * (size_t)(Wb + 1) * B6_PBS + 36 + 4 * 6 * (size_t)c.RS);
  const size_t smem = std::max(fact, band_chol_smem(c.bw));
#define PSFM_BC6_GO(MT, TRV, TCV)                                                                                      \
  do {                                                                                                             \
    static size_t attr = 0;                                                                                        \
    if (smem > attr) {                                                                                             \
      PSFM_CUDA(cudaFuncSetAttribute(k_band_chol6<MT, TRV, TCV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
      attr = smem;                                                                                                 \
    }                                                                                                              \
    k_band_chol6<MT, TRV, TCV><<<grid, MT, smem, st>>>(c);                                                               \
  } while (0)
  // thin threads while the CTA has room for them (see k_band_chol6), else one fat thread per block; the threads
  // after the workers and the panel group are the loader (>= 32)
  const int ng2 = ((2 * nblk + 31) & ~31) + np;
  if (ng4 + 32 <= 512) PSFM_BC6_GO(512, 3, 3);
  else if (ng2 + 32 <= 384) PSFM_BC6_GO(384, 3, 6);
  else if (ng1 + 64 <= 256) PSFM_BC6_GO(256, 6, 6);
  else if (ng1 + 64 <= 512) PSFM_BC6_GO(512, 6, 6);
  else PSFM_BC6_GO(640, 6, 6);
#undef PSFM_BC6_GO
  PSFM_LAUNCH_CHECK();
}

}  // namespace ba
}  // namespace psfm
