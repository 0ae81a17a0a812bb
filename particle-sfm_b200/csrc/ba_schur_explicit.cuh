// ba_schur_explicit.cuh — EXACT reduced-camera-system solve on the device.
//
// The reference solves the reduced camera system exactly for <= 1000 images (DENSE_SCHUR /
// SPARSE_SCHUR, bundle_adjustment.cc:276-286): Ceres' SchurEliminator forms
//     S = F'F + D_c^2 - sum_p (F'E)_p (E'E + D_p^2)^-1 (E'F)_p
// and factorises it.  This file does the same on the GPU:
//   pair structure   all (i, j) observation pairs of a point keyed by (tile, image a, image b),
//                    one TASK per run of equal keys (built once per problem with a segmented
//                    sort / run-length encode); both paths below run these tasks
//   k_schur_tile[_p] FUSED path: per observation Z_i = W_i G (dense tiles, H~ = G G') or the compact
//                    factors [D | w | Q = Jp H~ | Jp] (pair loop) stay in shared memory; per-image cross blocks / focal column / rhs
//                    correction; the tile's pair tasks sum (W_i H~) W_j' = Jc_i' (Q_i Jp_j') Jc_j
//                    into the band-block accumulator Sband[a][b - a][36]
//   k_schur_w, k_schur_pairs   unfused fallback, used when a tile's staging does not fit the
//                    fused kernel's shared memory: the same per-image sums and the same pair
//                    tasks into the same Sband, with W, W H~ per observation through HBM (AoS)
//   reduced system   [per-image sums | Sband] is all-reduced, then either assembled into a
//                    compact band matrix for k_band_chol6 (ba_band_chol.cuh) or, when the band is
//                    too wide or there are fewer than 3 images, into dense S (k_schur_assemble_*) for k_chol_blocked: cooperative
//                    blocked banded(+arrow) Cholesky, band = 6 * (longest image span of a track)
// Everything accumulates with the UNSCALED factored Jacobian (see ba_kernels.cuh); the
// scaling diag(s) is applied when the reduced system is assembled.
#pragma once
#include <cooperative_groups.h>
#include <cub/cub.cuh>

#include "ba_kernels.cuh"
#include "ba_tile_pipe.cuh"

namespace psfm {
namespace ba {

// per-image sums, stride NVX2 in the accumulator of both paths: rot-t cross block (9) | F'G focal (6) |
// -(W H~) Wk' (6) | -(W w^) rot (3) | t (3).  k_schur_w stages and sends only the first NVX rows (its
// shared memory is what the fallback has to fit); its rhs correction comes from k_schur_prep instead.
constexpr int NVX = 21;
constexpr int NVX2 = 27;

// ------------------------------------------------------------------ per-observation W, W H~

struct SwArgs {
  Lin L;
  const double* pose16;
  const double* X;
  const double* ht;     // [6][P]
  const double* wk;     // [9][P] G'E per point (focal row used)
  const double* K;
  double* W;            // [M][18]  rows: rot 0..2, t 0..2 ; 3 values per row
  double* WH;           // [M][18]
  double* acc_cam;      // [NREP][F][NVX2], rows NVX.. untouched
  size_t rep_stride;
  int intr;
};

template <int TILE, bool ROT>
__global__ void __launch_bounds__(TILE, (TILE == 256 ? 2 : 1)) k_schur_w(const TileCtx tc, const SwArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  TileSmem<TILE> sm;
  sm.carve(smem_raw, NVX, 12, tc.cap_ns, tc.cap_np);
  const TileInfo ti = tile_header(tc);
  const int tid = threadIdx.x;
  const bool act = tid < ti.n;
  const size_t M = tc.M;
  const size_t i = (size_t)ti.base + tid;
  int ls = 0, lp = 0;
  double a00 = 0, a02 = 0, a12 = 0;
  if (act) {
    ls = __ldg(tc.obs_lseg + i);
    lp = __ldg(tc.obs_lpt + i);
    a00 = a.L.a[i]; a02 = a.L.a[M + i]; a12 = a.L.a[2 * M + i];
  }
  const double inv_f = (a.intr >= 1) ? 1.0 / __ldg(a.K) : 0.0;
  // per point: X (0..2), H~ (3..8), focal row of G'E (9..11)
  tile_fill_smem<TILE>(tc, sm, ti, a.pose16, nullptr, a.X, a.ht, a.wk, true);
  double* sv = sm.sv + tid;
#pragma unroll
  for (int k = 0; k < NVX; ++k) sv[k * PSFM_SVS] = 0.0;
  if (act) {
    ObsGeom g;
    load_geom<TILE>(sm, ls, lp, g);
    const int cnp = sm.cap_np;
    double hv[6], wkp[3];
#pragma unroll
    for (int k = 0; k < 6; ++k) hv[k] = sm.prow(3 + k)[lp];
#pragma unroll
    for (int k = 0; k < 3; ++k) wkp[k] = sm.prow(9 + k)[lp];
    double jp[2][3], jc[2][6];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      jp[0][k] = a00 * g.R[k] + a02 * g.R[6 + k];
      jp[1][k] = a00 * g.R[3 + k] + a12 * g.R[6 + k];
    }
    if (ROT) {
      jc[0][0] = 2.0 * a02 * g.w[1]; jc[0][1] = 2.0 * (a00 * g.w[2] - a02 * g.w[0]); jc[0][2] = -2.0 * a00 * g.w[1];
      jc[1][0] = 2.0 * (a12 * g.w[1] - a00 * g.w[2]); jc[1][1] = -2.0 * a12 * g.w[0]; jc[1][2] = 2.0 * a00 * g.w[0];
    } else {
#pragma unroll
      for (int k = 0; k < 3; ++k) { jc[0][k] = 0.0; jc[1][k] = 0.0; }
    }
    jc[0][3] = a00; jc[0][4] = 0.0; jc[0][5] = a02;
    jc[1][3] = 0.0; jc[1][4] = a00; jc[1][5] = a12;
    double W[6][3], WH[6][3];
#pragma unroll
    for (int r = 0; r < 6; ++r) {
#pragma unroll
      for (int k = 0; k < 3; ++k) W[r][k] = jc[0][r] * jp[0][k] + jc[1][r] * jp[1][k];
      WH[r][0] = W[r][0] * hv[0] + W[r][1] * hv[1] + W[r][2] * hv[2];
      WH[r][1] = W[r][0] * hv[1] + W[r][1] * hv[3] + W[r][2] * hv[4];
      WH[r][2] = W[r][0] * hv[2] + W[r][1] * hv[4] + W[r][2] * hv[5];
    }
    double2* Wo = reinterpret_cast<double2*>(a.W + 18 * i);
    double2* WHo = reinterpret_cast<double2*>(a.WH + 18 * i);
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      Wo[k] = make_double2(W[(2 * k) / 3][(2 * k) % 3], W[(2 * k + 1) / 3][(2 * k + 1) % 3]);
      WHo[k] = make_double2(WH[(2 * k) / 3][(2 * k) % 3], WH[(2 * k + 1) / 3][(2 * k + 1) % 3]);
    }
    // rot-t cross block of F'F: (Jr' Jt)[r][c]
    if (ROT) {
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) sv[(3 * r + c) * PSFM_SVS] = jc[0][r] * jc[0][3 + c] + jc[1][r] * jc[1][3 + c];
    }
    if (a.intr >= 1) {
      const double zf = (g.w[2] + g.tz) * inv_f;
      const double jf0 = -a02 * zf, jf1 = -a12 * zf;
#pragma unroll
      for (int r = 0; r < 6; ++r) {
        sv[(9 + r) * PSFM_SVS] = jc[0][r] * jf0 + jc[1][r] * jf1;                               // F'G
        sv[(15 + r) * PSFM_SVS] = -(WH[r][0] * wkp[0] + WH[r][1] * wkp[1] + WH[r][2] * wkp[2]);  // -(W H~) Wk'
      }
    }
  }
  __syncthreads();
  double* dst = a.acc_cam + (size_t)(blockIdx.x & (NREP - 1)) * a.rep_stride;
  tile_reduce_images<TILE>(sm, ti, NVX, [&](int k, int img, double acc) {
    if (acc != 0.0) atomicAdd(dst + (size_t)img * NVX2 + k, acc);
  });
}

// ------------------------------------------------------------------ pair structure

// entries started by observation j (sorted order): (j, j), (j, j+1) ... (j, end of its point)
// plus (j, j') for earlier observations j' of the same point IN THE SAME IMAGE (rare
// duplicates: both orders are needed inside a diagonal block)
__global__ void k_pair_count(const int* pt_ptr, const int* obs_pt, const int* obs_img, int M, int* cnt) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= M) return;
  const int p = obs_pt[j];
  const int b = pt_ptr[p], e = pt_ptr[p + 1];
  int c = e - j;
  for (int k = j - 1; k >= b && obs_img[k] == obs_img[j]; --k) ++c;
  cnt[j] = c;
}

// ------------------------------------------------------------------ block products

struct PairArgs {
  const unsigned int* entries;   // the fused path's pair tasks (see StArgs)
  const int* task_slot;
  const int2* task_rng;
  const int* tile_task;
  const int* tile_start;         // [T + 1] first observation of the tile: entries hold tile-local indices
  const double* W;               // [M][18]
  const double* WH;              // [M][18]
  double* Sband;                 // [nrep][band_stride]  += sum (W_i H~) W_j'
  size_t band_stride;
  int nrep_mask;
};

// One CTA per tile, one thread per pair task: the task's sum over its entries in registers, one RED per
// element into the tile's Sband replica.  A task has few entries (one for each point that sees both
// images), too few to pay for a reduction across lanes.
__global__ void __launch_bounds__(128) k_schur_pairs(const PairArgs a) {
  const int t = blockIdx.x;
  const size_t base = (size_t)__ldg(a.tile_start + t);
  const int q1 = __ldg(a.tile_task + t + 1);
  double* band = a.Sband + (size_t)(t & a.nrep_mask) * a.band_stride;
  for (int q = __ldg(a.tile_task + t) + threadIdx.x; q < q1; q += blockDim.x) {
    const int2 rg = __ldg(a.task_rng + q);
    double acc[36];
#pragma unroll
    for (int k = 0; k < 36; ++k) acc[k] = 0.0;
    for (int e = rg.x; e < rg.y; ++e) {
      const unsigned int u = __ldg(a.entries + e);
      const size_t i = base + (u >> 16), j = base + (u & 0xffffu);
      const double2* wh = reinterpret_cast<const double2*>(a.WH + 18 * i);
      const double2* wj = reinterpret_cast<const double2*>(a.W + 18 * j);
      double A[18], B[18];
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const double2 x = __ldg(wh + k), y = __ldg(wj + k);
        A[2 * k] = x.x; A[2 * k + 1] = x.y;
        B[2 * k] = y.x; B[2 * k + 1] = y.y;
      }
#pragma unroll
      for (int r = 0; r < 6; ++r)
#pragma unroll
        for (int c = 0; c < 6; ++c)
          acc[6 * r + c] += A[3 * r] * B[3 * c] + A[3 * r + 1] * B[3 * c + 1] + A[3 * r + 2] * B[3 * c + 2];
    }
    double* dst = band + (size_t)__ldg(a.task_slot + q) * 36;
#pragma unroll
    for (int k = 0; k < 36; ++k)
      if (acc[k] != 0.0) atomicAdd(dst + k, acc[k]);
  }
}

// ------------------------------------------------------------------ fused tile path: W in shared memory, pairs per tile
//
// A point never straddles a tile, so every (i, j) observation pair of the Schur complement
// lives inside one tile.  k_schur_tile keeps W_i and W_i H~ of its <= TILE observations in
// shared memory (nothing per-observation goes to HBM) and runs the tile's pair TASKS: a task
// is the run of pair entries of one image pair (a, b) inside the tile; two threads share a
// task (block rows 0-2 / 3-5), accumulate sum (W_i H~) W_j' in registers and issue one RED
// per element into the band-block accumulator  Sband[a][b - a][36]  (b - a <= span, the
// longest image span of a track, global over the ranks).  The per-image sums (rot-t cross
// block, focal column, rhs correction -W w^) are reduced per image segment as in the other
// tile kernels.

constexpr int PS = 18;     // shared-memory stride of one observation's record: 9 x 16 bytes, read with LDS.128 — eight
                           // consecutive records tile the 32 banks, so the records of one point (consecutive) do not collide

struct StArgs {
  Lin L;
  const double* pose16;
  const double* X;
  const double* gf;     // [6][P] G, H~ = G G' (k_point_blocks)
  const double* gv;     // [3][P] G' (focal row of G'E)
  const double* gu;     // [3][P] G' g^, so that w^ = H~ g^ = G gu
  const double* K;
  double* acc_cam;      // [NREP][F][NVX2]
  size_t rep_stride;
  int intr;
  const unsigned int* entries;   // (li << 16) | lj, tile-local indices, sorted by (tile, a, b)
  const int* task_slot;          // [ntasks] band-block slot a * (span + 1) + (b - a)
  const int2* task_rng;          // [ntasks] entry range (begin, end) of the task; tasks of a tile ordered by image pair
  const int* tile_task;          // [T + 1] task range of the tile
  double* Sband;                 // [nrep][F * (span + 1) * 36]
  size_t band_stride;
  int nrep_mask;
  int span;
  const unsigned char* tile_dense;   // [T] pair phase of the tile: TILE_PAIRS_LOOP | _DENSE | _DENSE_DUP
};

// ---- dense pair phase (tensor cores)
//
// For a point p with H~_p = G_p G_p' (G_p from k_point_blocks) and its observation i, Z_i = W_i G_p (6 x 3);
// then (W_i H~) W_j' = Z_i Z_j', and a tile's pair blocks are the block-upper part of Z Z' with
// Z = (6 ns) x (3 np): block (image segment s, point p) = sum of Z_i over the observations of p in
// s (two observations of p in one image give Z_i + Z_j, i.e. all their cross terms).  Z is staged
// in the dead reduction rows, zero-padded to 16-row blocks and 8-column pairs of k-steps, in the
// fragment order of mma.m16n8k4.f64: lane l of a warp holds Z[8 q + l / 4][4 k + l % 4] of 8-row
// block q at k-step k, and for Z Z' the A and B operands use that same layout.  Element
// (row, col) lives at ((q * KB2 + k / 2) * 32 + (l ^ (q & 7))) * 2 + k % 2: one LDS.128 per lane
// reads two k-steps of a fragment, a warp reads 512 contiguous bytes (no bank conflicts).  The XOR
// spreads the stores: the observations of one point are rows 6 s + r, all of one parity, and would
// otherwise write one bank.
enum : unsigned char { TILE_PAIRS_LOOP = 0, TILE_PAIRS_DENSE = 1, TILE_PAIRS_DENSE_DUP = 2 };

__host__ __device__ inline int dense_z_kb2(int np) { return (3 * np + 7) >> 3; }
__host__ __device__ inline int dense_z_rb(int ns) { return (6 * ns + 15) >> 4; }
// doubles of the staged Z of a tile with ns image segments and np points
__host__ __device__ inline size_t dense_z_doubles(int ns, int np) { return (size_t)dense_z_rb(ns) * dense_z_kb2(np) * 128; }

__device__ __forceinline__ void dmma_16x8x4(double (&d)[4], double a0, double a1, double b) {
  asm("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
      : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
      : "d"(a0), "d"(a1), "d"(b));
}

// Z Z' of the staged tile -> band blocks.  Warps take 16 x 16 output blocks (I <= J) of the
// block-upper part; per k-step pair 4 LDS.128 and 4 DMMA.16x8x4.  An element (r, c) goes to
// Sband[img(r)][img(c) - img(r)][r % 6][c % 6] when img(r) <= img(c) and its 8-row tile is not
// below the column's; a diagonal image block straddling two 8-row tiles also takes the mirror of
// the upper tile's elements (the lower tile is not computed).  Exact zeros (images that share no
// point of the tile) are not sent.
template <int TILE>
__device__ __forceinline__ void dense_pairs_mma(const double* __restrict__ zf, const int* __restrict__ cimg, int ns, int np,
                                                double* __restrict__ band, int span) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int R = 6 * ns, RB = dense_z_rb(ns), KB2 = dense_z_kb2(np);
  const int nblk = RB * (RB + 1) / 2;
  const double2* z2 = reinterpret_cast<const double2*>(zf);
  for (int blk = warp; blk < nblk; blk += TILE / 32) {
    int I = 0, rem = blk;
    while (rem >= RB - I) { rem -= RB - I; ++I; }
    const int J = I + rem;
    const double2* pa0 = z2 + (size_t)(2 * I) * KB2 * 32 + (lane ^ ((2 * I) & 7));
    const double2* pa1 = z2 + (size_t)(2 * I + 1) * KB2 * 32 + (lane ^ ((2 * I + 1) & 7));
    const double2* pb0 = z2 + (size_t)(2 * J) * KB2 * 32 + (lane ^ ((2 * J) & 7));
    const double2* pb1 = z2 + (size_t)(2 * J + 1) * KB2 * 32 + (lane ^ ((2 * J + 1) & 7));
    double acc[2][4];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[h][e] = 0.0;
#pragma unroll 2
    for (int k = 0; k < KB2; ++k) {
      const double2 a0 = pa0[32 * k], a1 = pa1[32 * k], b0 = pb0[32 * k], b1 = pb1[32 * k];
      dmma_16x8x4(acc[0], a0.x, a1.x, b0.x);
      dmma_16x8x4(acc[1], a0.x, a1.x, b1.x);
      dmma_16x8x4(acc[0], a0.y, a1.y, b0.y);
      dmma_16x8x4(acc[1], a0.y, a1.y, b1.y);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const double v = acc[h][e];
        const int r = 16 * I + (lane >> 2) + 8 * (e >> 1), c = 16 * J + 8 * h + 2 * (lane & 3) + (e & 1);
        if (v == 0.0 || r >= R || c >= R || (r >> 3) > (c >> 3)) continue;
        const int sr = r / 6, sc = c / 6;
        if (sr > sc) continue;
        const int ia = cimg[sr], d = cimg[sc] - ia;
        if (d > span) continue;
        double* blkp = band + ((size_t)ia * (span + 1) + d) * 36;
        atomicAdd(blkp + 6 * (r - 6 * sr) + (c - 6 * sc), v);
        if (sr == sc && (r >> 3) < (c >> 3)) atomicAdd(blkp + 6 * (c - 6 * sc) + (r - 6 * sr), v);
      }
  }
}

// One tile of the fused Schur kernel; shared memory holds the staged inputs (see linearize_tile).
// rep is the tile's index.  DENSE_ONLY: every tile of the launch is dense (the pair loop is not compiled).
template <int TILE, bool ROT, bool DENSE_ONLY = false>
__device__ __forceinline__ void schur_tile_body(const TileCtx& tc, const StArgs& a, TileSmem<TILE>& sm, const TileInfo& ti,
                                                const bool act, const int ls, const int lp, const double a00, const double a02,
                                                const double a12, const int rep, const int t0, const int nt) {
  const int tid = threadIdx.x;
  const double inv_f = (a.intr >= 1) ? 1.0 / __ldg(a.K) : 0.0;
  const unsigned char mode = __ldg(a.tile_dense + rep);
  // Pair tasks of this tile -> lanes: two lanes share a task (q = 2 task + part; entries e0 + part, stride 2).
  // Tried and dropped, both slower: runs cut into units of <= 8 entries so that all 8 warps carry pairs (more
  // REDs), three lanes per task (7 trips instead of 11 on the tile's critical path) — the pair loop is bound by
  // its fp64 instruction count, not by the longest lane.
  constexpr int lpt = 2;
  const int nq = 2 * max(nt, 0);      // nt >= 0; with the clamp ptxas spills 20 B less in k_schur_tile_p<*, true>
  auto lane_task = [&](int q, int& tq, int& par) -> bool {
    par = q & 1; tq = q >> 1;
    return q < nq;
  };
  // the first pass's task range / slot are fetched NOW: two dependent global loads (range, then entries)
  // would otherwise sit on the critical path of every tile right after the last barrier
  int tq_f, par_f;
  const bool valid_f = lane_task(tid, tq_f, par_f);
  int2 rg_f = make_int2(0, 0);
  int slot_f = 0;
  if (!DENSE_ONLY && valid_f) { rg_f = __ldg(a.task_rng + t0 + tq_f); slot_f = __ldg(a.task_slot + t0 + tq_f); }
  double* sv = sm.sv + tid;
#pragma unroll
  for (int k = 0; k < NVX2; ++k) sv[k * PSFM_SVS] = 0.0;
  // per-observation factors kept through the reduction (W = Jc' Jp and W H~ are never formed in memory):
  //   pair loop   rec = [a00 a02 a12 | w (3) | Q = Jp H~ (2x3) | Jp (2x3)]
  //   dense       rec = Z_i = Jc' (Jp G)  (6x3, row-major)
  double rec[18];
#pragma unroll
  for (int k = 0; k < 18; ++k) rec[k] = 0.0;
  if (act) {
    ObsGeom g;
    load_geom<TILE>(sm, ls, lp, g);
    const int cnp = sm.cap_np;
    double gm[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) gm[k] = sm.prow(3 + k)[lp];
    double jp[2][3], jc[2][6], jg[2][3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      jp[0][k] = a00 * g.R[k] + a02 * g.R[6 + k];
      jp[1][k] = a00 * g.R[3 + k] + a12 * g.R[6 + k];
    }
    // JG = Jp G (G upper triangular, packed [g00 g01 g02 g11 g12 g22]); W H~ v = Jc' JG (G' v) for any v
#pragma unroll
    for (int m = 0; m < 2; ++m) {
      jg[m][0] = jp[m][0] * gm[0];
      jg[m][1] = jp[m][0] * gm[1] + jp[m][1] * gm[3];
      jg[m][2] = jp[m][0] * gm[2] + jp[m][1] * gm[4] + jp[m][2] * gm[5];
    }
    if (ROT) {
      jc[0][0] = 2.0 * a02 * g.w[1]; jc[0][1] = 2.0 * (a00 * g.w[2] - a02 * g.w[0]); jc[0][2] = -2.0 * a00 * g.w[1];
      jc[1][0] = 2.0 * (a12 * g.w[1] - a00 * g.w[2]); jc[1][1] = -2.0 * a12 * g.w[0]; jc[1][2] = 2.0 * a00 * g.w[0];
    } else {
#pragma unroll
      for (int k = 0; k < 3; ++k) { jc[0][k] = 0.0; jc[1][k] = 0.0; }
    }
    jc[0][3] = a00; jc[0][4] = 0.0; jc[0][5] = a02;
    jc[1][3] = 0.0; jc[1][4] = a00; jc[1][5] = a12;
    if (ROT) {   // rot-t cross block of F'F: (Jr' Jt)[r][c]
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) sv[(3 * r + c) * PSFM_SVS] = jc[0][r] * jc[0][3 + c] + jc[1][r] * jc[1][3 + c];
    }
    if (a.intr >= 1) {
      const double zf = (g.w[2] + g.tz) * inv_f;
      const double jf0 = -a02 * zf, jf1 = -a12 * zf;
      const double gk[3] = {sm.prow(9)[lp], sm.prow(10)[lp], sm.prow(11)[lp]};
      const double qk0 = jg[0][0] * gk[0] + jg[0][1] * gk[1] + jg[0][2] * gk[2];
      const double qk1 = jg[1][0] * gk[0] + jg[1][1] * gk[1] + jg[1][2] * gk[2];
#pragma unroll
      for (int r = 0; r < 6; ++r) {
        sv[(9 + r) * PSFM_SVS] = jc[0][r] * jf0 + jc[1][r] * jf1;            // F'G
        sv[(15 + r) * PSFM_SVS] = -(jc[0][r] * qk0 + jc[1][r] * qk1);          // -(W H~) Wk'
      }
    }
    const double gg[3] = {sm.prow(12)[lp], sm.prow(13)[lp], sm.prow(14)[lp]};
    const double pw0 = jg[0][0] * gg[0] + jg[0][1] * gg[1] + jg[0][2] * gg[2];
    const double pw1 = jg[1][0] * gg[0] + jg[1][1] * gg[1] + jg[1][2] * gg[2];
#pragma unroll
    for (int r = (ROT ? 0 : 3); r < 6; ++r) sv[(21 + r) * PSFM_SVS] = -(jc[0][r] * pw0 + jc[1][r] * pw1);   // -(W w^)
    if (!DENSE_ONLY && mode == TILE_PAIRS_LOOP) {
      rec[0] = a00; rec[1] = a02; rec[2] = a12;
#pragma unroll
      for (int m = 0; m < 2; ++m) {   // Q = JG G'
        rec[6 + 3 * m] = jg[m][0] * gm[0] + jg[m][1] * gm[1] + jg[m][2] * gm[2];
        rec[7 + 3 * m] = jg[m][1] * gm[3] + jg[m][2] * gm[4];
        rec[8 + 3 * m] = jg[m][2] * gm[5];
      }
#pragma unroll
      for (int k = 0; k < 3; ++k) { rec[3 + k] = g.w[k]; rec[12 + k] = jp[0][k]; rec[15 + k] = jp[1][k]; }
    } else {
#pragma unroll
      for (int r = 0; r < 6; ++r)
#pragma unroll
        for (int k = 0; k < 3; ++k) rec[3 * r + k] = jc[0][r] * jg[0][k] + jc[1][r] * jg[1][k];
    }
  }
  __syncthreads();
  {
    double* dst = a.acc_cam + (size_t)(rep & (NREP - 1)) * a.rep_stride;
    tile_reduce_images<TILE>(sm, ti, NVX2, [&](int k, int img, double acc) {
      if (acc != 0.0) atomicAdd(dst + (size_t)img * NVX2 + k, acc);
    });
  }
  __syncthreads();
  double* band = a.Sband + (size_t)(rep & a.nrep_mask) * a.band_stride;
  if (DENSE_ONLY || mode != TILE_PAIRS_LOOP) {
    // the reduction rows are dead: stage Z there
    double* zf = sm.sv;
    const int KB2 = dense_z_kb2(ti.np), zrows = 16 * dense_z_rb(ti.ns), zcols = 8 * KB2;
    auto zat = [&](int row, int col) -> double* {
      const int q = row >> 3;
      return zf + (((q * KB2 + (col >> 3)) * 32 + (((row & 7) * 4 + (col & 3)) ^ (q & 7))) * 2 + ((col >> 2) & 1));
    };
    // zero blocks where a point has no observation; two observations of a point in one image
    // (TILE_PAIRS_DENSE_DUP) add into one block
    const int nz2 = zrows * zcols / 2;
    for (int k = tid; k < nz2; k += TILE) reinterpret_cast<double2*>(zf)[k] = make_double2(0.0, 0.0);
    __syncthreads();
    if (act) {
#pragma unroll
      for (int r = 0; r < 6; ++r)
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          double* z = zat(6 * ls + r, 3 * lp + k);
          if (mode == TILE_PAIRS_DENSE_DUP) atomicAdd(z, rec[3 * r + k]); else *z = rec[3 * r + k];
        }
    }
    __syncthreads();
    dense_pairs_mma<TILE>(zf, sm.cimg, ti.ns, ti.np, band, a.span);
    return;
  }
  // first entries of the first pass (three in flight per lane: one trip is shorter than an L2 round trip)
  unsigned int uf0 = 0u, uf1 = 0u, uf2 = 0u;
  {
    const int e = rg_f.x + par_f;
    if (e < rg_f.y) uf0 = __ldg(a.entries + e);
    if (e + lpt < rg_f.y) uf1 = __ldg(a.entries + e + lpt);
    if (e + 2 * lpt < rg_f.y) uf2 = __ldg(a.entries + e + 2 * lpt);
  }
  // the reduction rows are dead: the same shared memory now holds the per-observation records
  double* srec = sm.sv;
  if (act) {
    double2* o = reinterpret_cast<double2*>(srec + (size_t)tid * PS);
#pragma unroll
    for (int k = 0; k < 9; ++k) o[k] = make_double2(rec[2 * k], rec[2 * k + 1]);
  }
  __syncthreads();
  // Pair tasks.  Block(i, j) = (W_i H~) W_j' = Jc_i' M Jc_j with the 2x2 M = Q_i Jp_j': per
  // entry 12 16-byte shared-memory loads (ncu, round 2: 64 % of the L1 data-pipe cycles with 24 8-byte loads at a
  // 19-double stride, the busiest unit of the kernel) and ~110 flops.  Two lanes per task (even | odd entries), the full 6x6 block in
  // registers, one shuffle per element to combine, 18 REDs per lane.  Uniform trip count.
  for (int q0 = 0; q0 < nq; q0 += TILE) {
    int tq = tq_f, par = par_f, e0 = rg_f.x, e1 = rg_f.y, slot = slot_f;
    bool valid = valid_f;
    unsigned int u0 = uf0, u1 = uf1, u2 = uf2;
    if (q0 > 0) {
      valid = lane_task(q0 + tid, tq, par);
      e0 = e1 = 0; u0 = u1 = u2 = 0u;
      if (valid) {
        const int2 rg = __ldg(a.task_rng + t0 + tq);
        slot = __ldg(a.task_slot + t0 + tq);
        e0 = rg.x; e1 = rg.y;
        const int e = e0 + par;
        if (e < e1) u0 = __ldg(a.entries + e);
        if (e + lpt < e1) u1 = __ldg(a.entries + e + lpt);
        if (e + 2 * lpt < e1) u2 = __ldg(a.entries + e + 2 * lpt);
      }
    }
    double acc[36];
#pragma unroll
    for (int k = 0; k < 36; ++k) acc[k] = 0.0;
    for (int e = e0 + par; e < e1; e += lpt) {
      const unsigned int u = u0;
      u0 = u1; u1 = u2;
      u2 = (e + 3 * lpt < e1) ? __ldg(a.entries + e + 3 * lpt) : 0u;
      const double2* Pi = reinterpret_cast<const double2*>(srec + (size_t)(u >> 16) * PS);
      const double2* Pj = reinterpret_cast<const double2*>(srec + (size_t)(u & 0xffffu) * PS);
      // 12 LDS.128 per entry: [a00 a02 | a12 w0 | w1 w2 | Q (3 x 16 B)] of i, [a00 a02 | a12 w0 | w1 w2 | Jp (3 x 16 B)] of j
      double Ci[12], Cj[18];
#pragma unroll
      for (int k = 0; k < 6; ++k) { const double2 x = Pi[k]; Ci[2 * k] = x.x; Ci[2 * k + 1] = x.y; }
#pragma unroll
      for (int k = 0; k < 3; ++k) { const double2 x = Pj[k]; Cj[2 * k] = x.x; Cj[2 * k + 1] = x.y; }
#pragma unroll
      for (int k = 6; k < 9; ++k) { const double2 x = Pj[k]; Cj[2 * k] = x.x; Cj[2 * k + 1] = x.y; }
      // M = Q_i Jp_j'
      double m00 = 0.0, m01 = 0.0, m10 = 0.0, m11 = 0.0;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double qa = Ci[6 + k], qb = Ci[9 + k], pa = Cj[12 + k], pb = Cj[15 + k];
        m00 = fma(qa, pa, m00); m01 = fma(qa, pb, m01); m10 = fma(qb, pa, m10); m11 = fma(qb, pb, m11);
      }
      // The camera Jacobian of an observation is Jc = [Jr | Jt] with Jt = [[a, 0, b], [0, a, c]] (a00, a02, a12)
      // and the rows of Jr twice the cross products w x (row of Jt), i.e. Jr' = 2 [w]x Jt'.  With
      // N = Jt_i' M Jt_j (3 x 3), u = w_i, v = w_j the 6 x 6 block is
      //     tt = N      rt = 2 [u]x N      tr = 2 B      rr = 4 [u]x B,     B[r, :] = v x N[r, :]
      // — 104 fp64 instructions per entry instead of 144 for the products with the explicit 2 x 6 Jacobians
      // (the fp64 pipe is what bounds this loop); the factors 2 and 4 are applied once per task.
      double N[3][3];
      {
        const double aj = Cj[0], bj = Cj[1], cj = Cj[2], ai = Ci[0], bi = Ci[1], ci = Ci[2];
        const double t00 = m00 * aj, t01 = m01 * aj, t02 = fma(m01, cj, m00 * bj);
        const double t10 = m10 * aj, t11 = m11 * aj, t12 = fma(m11, cj, m10 * bj);
        N[0][0] = ai * t00; N[0][1] = ai * t01; N[0][2] = ai * t02;
        N[1][0] = ai * t10; N[1][1] = ai * t11; N[1][2] = ai * t12;
        N[2][0] = fma(ci, t10, bi * t00); N[2][1] = fma(ci, t11, bi * t01); N[2][2] = fma(ci, t12, bi * t02);
      }
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[6 * (3 + r) + 3 + c] += N[r][c];
      if (ROT) {
        const double u0 = Ci[3], u1 = Ci[4], u2 = Ci[5], v0 = Cj[3], v1 = Cj[4], v2 = Cj[5];
        double B[3][3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          B[r][0] = fma(v1, N[r][2], -(v2 * N[r][1]));
          B[r][1] = fma(v2, N[r][0], -(v0 * N[r][2]));
          B[r][2] = fma(v0, N[r][1], -(v1 * N[r][0]));
#pragma unroll
          for (int c = 0; c < 3; ++c) acc[6 * (3 + r) + c] += B[r][c];                       // tr / 2
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          // rt / 2: column k of [u]x N;   rr / 4: column k of [u]x B
          acc[6 * 0 + 3 + k] = fma(u1, N[2][k], fma(-u2, N[1][k], acc[6 * 0 + 3 + k]));
          acc[6 * 1 + 3 + k] = fma(u2, N[0][k], fma(-u0, N[2][k], acc[6 * 1 + 3 + k]));
          acc[6 * 2 + 3 + k] = fma(u0, N[1][k], fma(-u1, N[0][k], acc[6 * 2 + 3 + k]));
          acc[6 * 0 + k] = fma(u1, B[2][k], fma(-u2, B[1][k], acc[6 * 0 + k]));
          acc[6 * 1 + k] = fma(u2, B[0][k], fma(-u0, B[2][k], acc[6 * 1 + k]));
          acc[6 * 2 + k] = fma(u0, B[1][k], fma(-u1, B[0][k], acc[6 * 2 + k]));
        }
      }
    }
    if (ROT) {
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) { acc[6 * r + c] *= 4.0; acc[6 * r + 3 + c] *= 2.0; acc[6 * (3 + r) + c] *= 2.0; }
    }
    // combine the lanes of a task: lane `par` ends up with the sums of ITS share of the 36 elements (every
    // lane sends what its reader owns), then one RED per element
    double* dst = band + (size_t)slot * 36;
#pragma unroll
    for (int i = 0; i < 18; ++i) {
      const double mine = par ? acc[18 + i] : acc[i];
      const double x = par ? acc[i] : acc[18 + i];
      const double v = mine + __shfl_xor_sync(0xffffffffu, x, 1);
      if (valid && (ROT || v != 0.0)) atomicAdd(dst + 18 * par + i, v);
    }
  }
}

template <int TILE, bool ROT>
__global__ void __launch_bounds__(TILE, (TILE == 256 ? 2 : 1)) k_schur_tile(const TileCtx tc, const StArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  TileSmem<TILE> sm;
  sm.carve(smem_raw, NVX2, 15, tc.cap_ns, tc.cap_np);
  const TileInfo ti = tile_header(tc);
  const int tid = threadIdx.x;
  const bool act = tid < ti.n;
  const size_t M = tc.M;
  const size_t i = (size_t)ti.base + tid;
  int ls = 0, lp = 0;
  double a00 = 0, a02 = 0, a12 = 0;
  if (act) {
    ls = __ldg(tc.obs_lseg + i);
    lp = __ldg(tc.obs_lpt + i);
    a00 = a.L.a[i]; a02 = a.L.a[M + i]; a12 = a.L.a[2 * M + i];
  }
  const int t0 = __ldg(a.tile_task + blockIdx.x), nt = __ldg(a.tile_task + blockIdx.x + 1) - t0;
  // per point: X (0..2), G (3..8), G' (focal row of G'E) (9..11), G' g^ (12..14)
  tile_fill_smem<TILE>(tc, sm, ti, a.pose16, nullptr, a.X, a.gf, a.gv, true, a.gu);
  schur_tile_body<TILE, ROT>(tc, a, sm, ti, act, ls, lp, a00, a02, a12, blockIdx.x, t0, nt);
}

// persistent, pipelined form (ba_tile_pipe.cuh): the inputs of the next tile are in flight
// (cp.async) while this tile's pair tasks run
template <int TILE, bool ROT, bool DENSE_ONLY>
__device__ __forceinline__ void schur_tile_pipe(const TileCtx& tc, const PipeSrc& ps, const StArgs& a, unsigned char* smem_raw) {
  __shared__ __align__(16) int4 hdr_ring[4][2];
  __shared__ __align__(8) unsigned long long bars[2];
  const int cns = tc.cap_ns, cnp = tc.cap_np;
  const size_t sb = PipeStage<TILE>::bytes(false, true, 15, cns, cnp);
  TileSmem<TILE> sm;
  sm.cap_ns = cns; sm.cap_np = cnp;
  sm.sv = reinterpret_cast<double*>(smem_raw + 2 * sb);
  sm.sw = nullptr; sm.sred = nullptr; sm.sx = nullptr;
  pipe_run<TILE>(tc, ps, smem_raw, hdr_ring, bars, 15, cns, cnp, [&](const TileInfo& ti, const PipeStage<TILE>& s, int tile) {
    view_stage<TILE>(sm, s);
    const int tid = threadIdx.x;
    const bool act = tid < ti.n;
    int ls = 0, lp = 0;
    double a00 = 0, a02 = 0, a12 = 0;
    if (act) { ls = s.lseg[tid]; lp = s.lpt[tid]; a00 = s.a0[tid]; a02 = s.a1[tid]; a12 = s.a2[tid]; }
    int t0 = 0, nt = 0;
    if (!DENSE_ONLY) { t0 = __ldg(a.tile_task + tile); nt = __ldg(a.tile_task + tile + 1) - t0; }
    schur_tile_body<TILE, ROT, DENSE_ONLY>(tc, a, sm, ti, act, ls, lp, a00, a02, a12, tile, t0, nt);
  });
}

template <int TILE, bool ROT>
__global__ void __launch_bounds__(TILE, (TILE == 256 ? 2 : 1)) k_schur_tile_p(const TileCtx tc, const PipeSrc ps, const StArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  schur_tile_pipe<TILE, ROT, false>(tc, ps, a, smem_raw);
}

// the same kernel when every tile of the problem is dense (k_tile_pairs_mode): without the pair loop's code ptxas
// keeps the dense phase in registers (k_schur_tile_p spills in it)
template <int TILE, bool ROT>
__global__ void __launch_bounds__(TILE, (TILE == 256 ? 2 : 1)) k_schur_dense_p(const TileCtx tc, const PipeSrc ps, const StArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  schur_tile_pipe<TILE, ROT, true>(tc, ps, a, smem_raw);
}

template <int TILE>
inline size_t pipe_smem_schur_tile(int cns, int cnp) {
  return 2 * PipeStage<TILE>::bytes(false, true, 15, cns, cnp) + sizeof(double) * NVX2 * (TILE + 1);
}

// ---- tile-local pair structure (built once per problem)

// entries started by observation j (see k_pair_count); key = (tile, image a, image b), value =
// the two tile-local observation indices
__global__ void k_pair_fill_tile(const int* pt_ptr, const int* obs_pt, const int* obs_img, const int* ptr, int M,
                                 const int* tile_start, int T, int fbits, unsigned long long* keys, unsigned int* vals) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= M) return;
  int lo = 0, hi = T;           // tile of j: last tile with tile_start <= j
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (tile_start[mid] <= j) lo = mid; else hi = mid;
  }
  const int base = tile_start[lo];
  const int p = obs_pt[j];
  const int b = pt_ptr[p], e = pt_ptr[p + 1];
  const unsigned long long a = (unsigned long long)obs_img[j];
  const unsigned long long khi = ((unsigned long long)lo << (2 * fbits)) | (a << fbits);
  size_t o = (size_t)ptr[j];
  for (int k = j; k < e; ++k, ++o) {
    keys[o] = khi | (unsigned long long)obs_img[k];
    vals[o] = ((unsigned)(j - base) << 16) | (unsigned)(k - base);
  }
  for (int k = j - 1; k >= b && obs_img[k] == (int)a; --k, ++o) {
    keys[o] = khi | a;
    vals[o] = ((unsigned)(j - base) << 16) | (unsigned)(k - base);
  }
}

// pair phase of every tile: dense (Z Z' on tensor cores) when allowed and its Z fits the reduction rows
// (zcap doubles), else the pair loop; tiles with two observations of a point in one image accumulate
// Z with shared-memory atomics.  ndense counts the dense tiles.
__global__ void k_tile_pairs_mode(const int* tile_start, const int* tile_pt, const int* cseg_ptr, const int* obs_pt,
                                  const int* obs_img, int T, size_t zcap, int allow, unsigned char* mode, int* ndense) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  unsigned char m = TILE_PAIRS_LOOP;
  if (allow && dense_z_doubles(cseg_ptr[t + 1] - cseg_ptr[t], tile_pt[t + 1] - tile_pt[t]) <= zcap) {
    m = TILE_PAIRS_DENSE;
    for (int j = tile_start[t] + 1; j < tile_start[t + 1]; ++j)
      if (obs_pt[j] == obs_pt[j - 1] && obs_img[j] == obs_img[j - 1]) { m = TILE_PAIRS_DENSE_DUP; break; }
    atomicAdd(ndense, 1);
  }
  mode[t] = m;
}

// first entry of every tile (entries are written in observation order, tiles are observation ranges)
__global__ void k_tile_entry_offsets(const int* tile_start, const int* ptr, int T, int* seg) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t <= T) seg[t] = ptr[tile_start[t]];
}

// One task per run of equal (tile, image a, image b) keys, in key order: band-block slot and entry range
// [beg, beg + count) of the run (beg: exclusive scan of the run lengths)
__global__ void k_pair_tasks(const unsigned long long* run_key, const int* run_count, const int* run_beg, int nruns,
                             int fbits, int span, int* slot, int2* rng) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nruns) return;
  const unsigned long long k = run_key[t], mask = (1ull << fbits) - 1;
  const int b = (int)(k & mask), a = (int)((k >> fbits) & mask);
  slot[t] = a * (span + 1) + (b - a);
  rng[t] = make_int2(run_beg[t], run_beg[t] + run_count[t]);
}

// tile -> first task (lower bound over the tiles of the sorted run keys)
__global__ void k_tile_tasks(const unsigned long long* run_key, int nruns, int fbits, int T, int* tile_task) {
  const int tile = blockIdx.x * blockDim.x + threadIdx.x;
  if (tile > T) return;
  int lo = 0, hi = nruns;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if ((long long)(run_key[mid] >> (2 * fbits)) < tile) lo = mid + 1; else hi = mid;
  }
  tile_task[tile] = lo;
}

// band blocks -> dense S:  S[6a+r][6b+c] -= s s' Sband[a][b-a][r][c]  (mirrored for a != b)
struct BandAsmArgs {
  const double* Sband;
  const double* scale_c;
  int F, span, lda;
  double* S;
};

__global__ void k_schur_assemble_band(const BandAsmArgs a) {
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t per_img = (size_t)(a.span + 1) * 36;
  if (t >= (size_t)a.F * per_img) return;
  const double x = a.Sband[t];
  if (x == 0.0) return;
  const int ia = (int)(t / per_img), rem = (int)(t % per_img), d = rem / 36, e = rem % 36, r = e / 6, c = e % 6;
  const int ib = ia + d;
  if (ib >= a.F) return;
  const size_t row = 6 * (size_t)ia + r, col = 6 * (size_t)ib + c;
  const double v = -a.scale_c[row] * a.scale_c[col] * x;
  a.S[row * a.lda + col] += v;
  if (d != 0) a.S[col * a.lda + row] += v;
}

// ------------------------------------------------------------------ assembly of the dense reduced system

struct AsmArgs {
  const double* lin_cam;    // [F][NVL]  rot F'F (6) | t F'F (6) | ...
  const double* lin_intr;   // [C][NVI]
  const double* prep_intr;  // [C][NVI]
  const double* xcam;       // [F][xstride] per-image sums (NVX2)
  int xstride;
  const double* scale_c;    // [NS]
  const double* Dc2;        // [NS]
  const unsigned char* active;
  const double* rhs;        // [NS]
  int F, C, NS;
  int lda;                  // leading dimension of S (NS + 1: the extra row carries the rhs)
  double* S;                // [lda][lda] row-major, zeroed
};

// per-image parts: rot-t cross block of F'F and the focal column
__global__ void k_schur_assemble_local(const AsmArgs a) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int NS = a.lda, F = a.F;
  if (j >= F) return;
  const double* X = a.xcam + (size_t)j * a.xstride;
  const size_t s0 = 6 * (size_t)j;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      const double x = a.scale_c[s0 + r] * a.scale_c[s0 + 3 + c] * X[3 * r + c];
      if (x != 0.0) { atomicAdd(a.S + (s0 + r) * NS + s0 + 3 + c, x); atomicAdd(a.S + (s0 + 3 + c) * NS + s0 + r, x); }
    }
  const size_t sk = 6 * (size_t)F;   // single shared camera when intrinsics are free
  for (int r = 0; r < 6; ++r) {
    const double v = a.scale_c[s0 + r] * a.scale_c[sk] * (X[9 + r] + X[15 + r]);
    if (v != 0.0) { atomicAdd(a.S + (s0 + r) * NS + sk, v); atomicAdd(a.S + sk * NS + s0 + r, v); }
  }
}

// parts built from already all-reduced accumulators: F'F rot/t diagonal blocks, intrinsics block
__global__ void k_schur_assemble_global(const AsmArgs a) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int NS = a.lda, F = a.F;
  const int ut[3][3] = {{0, 1, 2}, {1, 3, 4}, {2, 4, 5}};
  if (j < F) {
    const double* A = a.lin_cam + (size_t)j * NVL;
    const size_t s0 = 6 * (size_t)j;
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) {
        a.S[(s0 + r) * NS + s0 + c] += a.scale_c[s0 + r] * a.scale_c[s0 + c] * A[ut[r][c]];
        a.S[(s0 + 3 + r) * NS + s0 + 3 + c] += a.scale_c[s0 + 3 + r] * a.scale_c[s0 + 3 + c] * A[6 + ut[r][c]];
      }
  } else if (j < F + a.C) {
    const int c = j - F;
    const size_t sk = 6 * (size_t)F + 3 * c;
    const double* G = a.lin_intr + (size_t)c * NVI;
    const double* Gc = a.prep_intr + (size_t)c * NVI;
    for (int r = 0; r < 3; ++r)
      for (int cc = 0; cc < 3; ++cc)
        a.S[(sk + r) * NS + sk + cc] += a.scale_c[sk + r] * a.scale_c[sk + cc] * (G[ut[r][cc]] + Gc[ut[r][cc]]);
  }
}

// LM diagonal on active slots, identity on inactive ones (their rows/cols are zero: scale 0)
__global__ void k_schur_assemble_finish(const AsmArgs a) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= a.NS) return;
  if (a.active[s]) a.S[(size_t)s * a.lda + s] += a.Dc2[s];
  else a.S[(size_t)s * a.lda + s] = 1.0;
  a.S[(size_t)a.NS * a.lda + s] = a.rhs[s];      // rhs as an extra (arrow) row: its factor row is L^-1 b
}

// ------------------------------------------------------------------ blocked, band-aware Cholesky (cooperative, multi-CTA)

// In-place lower Cholesky of the leading ns x ns part of A (row-major, leading dimension
// lda), where A[i][j] == 0 for |i - j| > bw among the first nb rows and rows nb..ns-1 are
// dense ("arrow": shared intrinsics).  Row ns of A holds the right-hand side b: it is
// carried through the factorisation as one more arrow row, so that its solved entries are
// L^-1 b; CTA 0 then solves L' x = L^-1 b.  One cooperative launch: per 32-column panel
// (1) every CTA factors the 32x32 diagonal block redundantly, (2) per trailing tile pair a CTA
// solves the two row tiles it needs against it and updates its tile, (3) ONE grid barrier.
// The factor lives in its own storage (Ld, Lp); A keeps the unsolved panels so that no CTA
// has to wait for another one's row solves.  fail[0] = 1 when a pivot is not positive.
constexpr int CB = 32;

struct CholArgs {
  double* A;
  int ns, lda, nb, bw;
  double* x;      // [ns]
  int* fail;
  unsigned int* bar;          // grid barrier counter, zeroed before the launch
  double* Lp;                 // [npanel][rmax][CB]  solved rows below each panel (the factor's off-diagonal part)
  double* Ld;                 // [npanel][CB][CB]    diagonal blocks of the factor
  int rmax;                   // rows reserved per panel in Lp
};

// Grid-wide barrier for the few (co-resident, cooperative launch) CTAs of k_chol_blocked: one
// atomic per CTA on a monotone counter and an acquire spin — about half the cost of
// cooperative_groups' grid.sync(), which this kernel pays twice per 32-column panel.
__device__ __forceinline__ void chol_grid_barrier(unsigned int* counter, unsigned int& target) {
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    target += gridDim.x;
    atomicAdd(counter, 1u);
    unsigned int v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
    } while (v < target);
  }
  __syncthreads();
}

__device__ __forceinline__ int chol_row_of(int pos, int c1, int nband, int arrow0) {
  return pos < nband ? c1 + pos : arrow0 + (pos - nband);
}

// Warp-level Cholesky of one w x w (w <= 32) diagonal block at A (leading dimension lda):
// lane r owns row r in registers, the block is padded to 32 x 32 with an identity tail.
// Writes L to sD and 1/L[k][k] to sDinv; returns true on a non-positive pivot.
__device__ __noinline__ bool chol_diag_warp(const double* __restrict__ A, int lda, int w,
                                            double (*sD)[CB + 1], double* sDinv) {
  const int lane = threadIdx.x & 31;
  double arow[CB];
#pragma unroll
  for (int c = 0; c < CB; ++c)
    arow[c] = (lane < w && c <= lane) ? __ldcg(A + (size_t)lane * lda + c) : ((c == lane && lane >= w) ? 1.0 : 0.0);
  bool bad = false;
  double myinv = 1.0;
#pragma unroll
  for (int j = 0; j < CB; ++j) {
    const double d = __shfl_sync(0xffffffffu, arow[j], j);
    if (!(d > 0.0) || isinf(d)) bad = true;
    // L_jj = sqrt(d) correctly rounded and its reciprocal, as LAPACK's potf2 scales a column: d * rsqrt(d) is not
    // correctly rounded and disagrees with the reciprocal it scales by, which cost up to 9x LAPACK's forward error
    // on ill-conditioned Laplacians (tests/test_gpu_dense_chol.py)
    const double ljj = sqrt(d), idj = 1.0 / ljj;
    if (lane == j) { arow[j] = ljj; myinv = idj; }
    else if (lane > j) arow[j] = arow[j] * idj;
    const double lr = arow[j];
#pragma unroll
    for (int c = j + 1; c < CB; ++c) {
      const double lc = __shfl_sync(0xffffffffu, lr, c);
      if (lane >= c) arow[c] -= lr * lc;
    }
  }
#pragma unroll
  for (int c = 0; c < CB; ++c) sD[lane][c] = arow[c];
  sDinv[lane] = myinv;
  return __any_sync(0xffffffffu, bad);
}

// One row of the panel below the diagonal block: x L11' = a (registers, right-looking so that the
// updates of one step are independent), from the (unsolved) global row into a shared-memory tile
// row and, when lprow != nullptr, into the factor storage.
__device__ __noinline__ void chol_row_solve_to(const double* __restrict__ grow, int w, const double (*sD)[CB + 1],
                                               const double* sDinv, double* __restrict__ srow, double* __restrict__ lprow) {
  double xr[CB];
#pragma unroll
  for (int k = 0; k < CB; ++k) xr[k] = (k < w) ? __ldcg(grow + k) : 0.0;
#pragma unroll
  for (int k = 0; k < CB; ++k) {
    xr[k] *= sDinv[k];
#pragma unroll
    for (int m = k + 1; m < CB; ++m) xr[m] -= xr[k] * sD[m][k];
  }
#pragma unroll
  for (int k = 0; k < CB; ++k) srow[k] = xr[k];
  if (lprow) {
#pragma unroll
    for (int k = 0; k < CB; ++k) lprow[k] = xr[k];
  }
}

__global__ void __launch_bounds__(256) k_chol_blocked(const CholArgs a) {
  unsigned int bar_target = 0;
  __shared__ double sD[CB][CB + 1];
  __shared__ double sLi[CB][CB + 1];
  __shared__ double sLj[CB][CB + 1];
  __shared__ double sDinv[CB];
  __shared__ int s_bad;
  const int tid = threadIdx.x;
  const int ns = a.ns, lda = a.lda, nrows = a.ns + 1;     // rows incl. the rhs row
  double* A = a.A;
  if (tid == 0) s_bad = 0;
  __syncthreads();
  for (int c0 = 0; c0 < ns; c0 += CB) {
    const int w = min(CB, ns - c0), c1 = c0 + w;
    // ---- (1) diagonal block, redundantly per CTA: warp 0 factors it in registers
    if (tid < CB && chol_diag_warp(A + (size_t)c0 * lda + c0, lda, w, sD, sDinv)) s_bad = 1;
    __syncthreads();
    if (s_bad) break;     // uniform across the grid: every CTA factors the same block
    // ---- rows below the panel that can be non-zero
    const int rb = (c1 < a.nb) ? min(a.nb, c1 + a.bw) : c1;
    const int nband = max(0, rb - c1);
    const int arrow0 = max(a.nb, c1);
    const int npos = nband + (nrows - arrow0);
    const int p = c0 / CB;
    // the factor's diagonal block goes to its own storage (the unfactored block in A is still
    // being read by slower CTAs)
    if (blockIdx.x == 0)
      for (int t = tid; t < CB * CB; t += 256) a.Ld[(size_t)p * CB * CB + t] = sD[t / CB][t % CB];
    // ---- (2+3) per tile pair of the rows below the panel: this CTA solves the two row tiles
    //      it needs itself (X L11' = A21, from the UNSOLVED panel in A: nobody waits for a
    //      row-solve phase of another CTA), then updates its trailing tile.  Solved rows are
    //      stored to Lp by the CTA of pair (ti, 0).  ONE grid barrier per panel.
    const int ntile = (npos + CB - 1) / CB;
    const int npair = ntile * (ntile + 1) / 2;
    for (int pr = blockIdx.x; pr < npair; pr += gridDim.x) {
      int ti = 0;
      while ((ti + 1) * (ti + 2) / 2 <= pr) ++ti;          // pr -> (ti, tj), tj <= ti; a handful of tiles
      const int tj = pr - ti * (ti + 1) / 2;
      __syncthreads();
      if (tid < 2 * CB) {
        const int which = tid >> 5, lr = tid & 31;
        const int pos = (which ? tj : ti) * CB + lr;
        double* srow = which ? sLj[lr] : sLi[lr];
        if (!(which && ti == tj)) {
          if (pos < npos) {
            const int g = chol_row_of(pos, c1, nband, arrow0);
            double* lprow = (!which && tj == 0) ? a.Lp + ((size_t)p * a.rmax + pos) * CB : nullptr;
            chol_row_solve_to(A + (size_t)g * lda + c0, w, sD, sDinv, srow, lprow);
          } else {
#pragma unroll
            for (int k = 0; k < CB; ++k) srow[k] = 0.0;
          }
        }
      }
      double* dst[4];
      double old[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {          // this thread's four outputs: issue the loads early
        const int r = (tid + 256 * u) / CB, c = (tid + 256 * u) % CB;
        const int pi = ti * CB + r, pj = tj * CB + c;
        dst[u] = nullptr;
        old[u] = 0.0;
        if (pi < npos && pj < npos && pj <= pi) {
          const int gi = chol_row_of(pi, c1, nband, arrow0), gj = chol_row_of(pj, c1, nband, arrow0);
          if (gj < ns) {       // the rhs row has no column
            dst[u] = A + (size_t)gi * lda + gj;
            old[u] = __ldcg(dst[u]);
          }
        }
      }
      __syncthreads();
      if (ti == tj) {
        for (int t = tid; t < CB * CB; t += 256) sLj[t / CB][t % CB] = sLi[t / CB][t % CB];
        __syncthreads();
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (dst[u]) {
          const int r = (tid + 256 * u) / CB, c = (tid + 256 * u) % CB;
          double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;      // four chains: a dependent fp64 op costs ~25-30 cycles
#pragma unroll
          for (int k = 0; k < CB; k += 4) {
            s0 = fma(sLi[r][k], sLj[c][k], s0);
            s1 = fma(sLi[r][k + 1], sLj[c][k + 1], s1);
            s2 = fma(sLi[r][k + 2], sLj[c][k + 2], s2);
            s3 = fma(sLi[r][k + 3], sLj[c][k + 3], s3);
          }
          *dst[u] = old[u] - ((s0 + s1) + (s2 + s3));
        }
      }
    }
    chol_grid_barrier(a.bar, bar_target);
  }
  if (blockIdx.x != 0) return;
  if (tid == 0) *a.fail = s_bad;
  if (s_bad) return;
  // ---- back substitution L' x = y (CTA 0, panel by panel from the end); y = L^-1 b is the
  //      solved rhs row, the last row below every panel in Lp
  __shared__ double sacc[8][CB];
  const int npanel = (ns + CB - 1) / CB;
  for (int t = tid; t < npanel * CB; t += 256) {
    const int p = t / CB, c = t % CB, c0 = p * CB, w = min(CB, ns - c0), c1 = c0 + w;
    if (c < w) {
      const int rb = (c1 < a.nb) ? min(a.nb, c1 + a.bw) : c1;
      const int npos_all = max(0, rb - c1) + (nrows - max(a.nb, c1));
      a.x[c0 + c] = __ldcg(a.Lp + ((size_t)p * a.rmax + (npos_all - 1)) * CB + c);
    }
  }
  __syncthreads();
  for (int p = npanel - 1; p >= 0; --p) {
    const int c0 = p * CB, w = min(CB, ns - c0), c1 = c0 + w;
    const int rb = (c1 < a.nb) ? min(a.nb, c1 + a.bw) : c1;
    const int nband = max(0, rb - c1);
    const int arrow0 = max(a.nb, c1);
    const int npos = nband + (ns - arrow0);          // rhs row excluded
    const double* Lp = a.Lp + (size_t)p * a.rmax * CB;
    // partial sums: column c of the panel, rows strided over the 8 row-groups
    const int c = tid % CB, g = tid / CB;
    for (int t = tid; t < CB * CB; t += 256) sD[t / CB][t % CB] = __ldcg(a.Ld + (size_t)p * CB * CB + t);
    double s = 0.0;
    if (c < w) {
      int pos = g;
      for (; pos + 24 < npos; pos += 32) {       // four independent loads in flight
        double av[4], xv[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          av[u] = __ldcg(Lp + (size_t)(pos + 8 * u) * CB + c);
          xv[u] = a.x[chol_row_of(pos + 8 * u, c1, nband, arrow0)];
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) s += av[u] * xv[u];
      }
      for (; pos < npos; pos += 8) s += __ldcg(Lp + (size_t)pos * CB + c) * a.x[chol_row_of(pos, c1, nband, arrow0)];
    }
    sacc[g][c] = s;
    __syncthreads();
    if (tid < w) {
      double t = 0.0;
      for (int gg = 0; gg < 8; ++gg) t += sacc[gg][tid];
      sacc[0][tid] = a.x[c0 + tid] - t;
    }
    __syncthreads();
    // in-panel backward substitution (warp 0; L11 staged in shared memory above)
    if (tid < CB) {
      double mine = (tid < w) ? sacc[0][tid] : 0.0;
      const double dinv = (tid < w) ? 1.0 / sD[tid][tid] : 0.0;
      for (int j = w - 1; j >= 0; --j) {
        const double v = __shfl_sync(0xffffffffu, mine * dinv, j);
        if (tid == j) a.x[c0 + j] = v;
        if (tid < j) mine -= sD[j][tid] * v;
      }
    }
    __syncthreads();
  }
}

}  // namespace ba
}  // namespace psfm
