// ba_kernels.cuh — sm_90a tile kernels of HP2 (global bundle adjustment), FACTORED-JACOBIAN
// formulation.
//
// Replaces what ceres::Solve does inside BundleAdjuster::Solve
// (reference sfm/gmapper/src/optim/bundle_adjustment.cc:306): per-observation
// reprojection residual/Jacobian evaluation (COLMAP BundleAdjustmentCostFunction<
// SimplePinholeCameraModel>, call sites bundle_adjustment.cc:380-411), loss correction
// (CreateLossFunction :54-69), per-point 3x3 Schur elimination and the implicit
// reduced-camera-system product used by PCG.
//
// Factored Jacobian (DESIGN.md §3.2).  For observation i of point p in image m the
// loss-corrected Jacobian blocks of the reprojection residual are
//     J_point = D_i R_m      J_trans = D_i      J_rot = D_i N(w_i)      J_focal = sq_i (u_i, v_i)'
// with D_i = sqrt(rho') d r/d p = [[a00, 0, a02], [0, a00, a12]]   (3 distinct numbers),
//      w_i = R_m X_p,  N(w) = -2 [w]x  (Ceres QuaternionParameterization: q+ = exp(d) (x) q),
//      sq_i (u_i, v_i) = -(a02, a12) z_i / f,   z_i = w_i[2] + t_m[2].
// Only (a00, a02, a12) and the corrected residual are STORED per observation (40 B instead
// of the 176 B of an explicit 2x(6+3+1) Jacobian row pair); R_m, t_m and X_p are staged in
// shared memory once per tile and every product with J or J' goes through the 3-vectors
// D'v / D y.  Ceres' Jacobi column scaling never touches these kernels: all per-image and
// per-point sums are accumulated UNSCALED and the diagonal scaling s is applied by the
// O(#images)/O(#points) kernels of ba_small_kernels.cuh (J diag(s) is the scaled Jacobian,
// so S_scaled = diag(s) S_unscaled diag(s) etc. — algebraically identical).
//
// Tiling: observations sorted by (point, image), packed into tiles of <= TILE observations
// that never split a point; one CTA per tile, one thread per observation.  Per-point sums are
// reduced inside the tile through shared memory in a fixed order (no atomics); per-image
// sums are reduced per (image segment, component) inside the tile, then one fp64 RED per
// segment goes to a replicated global accumulator (replica = tile mod NREP).
#pragma once
#include "psfm_common.cuh"

namespace psfm {
namespace ba {

constexpr int NVL = 18;   // camera-side accumulator stride per image
constexpr int NVI = 9;    // intrinsics accumulator stride per camera
// Concurrently resident tiles are consecutive tiles and therefore touch the SAME few
// images: their fp64 REDs would serialise on a handful of L2 addresses.  Every per-image
// accumulator is therefore replicated NREP times (replica = tile index mod NREP) and the
// replicas are folded by k_fold_replicas before use.
constexpr int NREP = 32;

struct TileCtx {
  const int* tile_start;   // [T+1] first observation of each tile
  const int* tile_pt;      // [T+1] first (internal) point of each tile
  const int* pt_ptr;       // [P+1] observation range of each point
  const int* obs_img;      // [M]  (k_cost only)
  const int* obs_pt;       // [M]  (k_cost only)
  const unsigned short* obs_lseg;  // [M] index of the observation's image in the tile's segment list
  const unsigned short* obs_lpt;   // [M] index of the observation's point inside the tile
  const double2* obs_xy;   // [M]
  const unsigned short* tile_perm;  // [M] e-th observation of the tile in image order
  const int* cseg_ptr;     // [T+1] image segments of each tile
  const int* cseg_img;     // [nseg]
  const unsigned short* cseg_off;  // [nseg] start of the segment in the tile's image order
  const int* img_cam;      // [F]
  int F, P, M, C, T;
  int cap_ns, cap_np;      // max segments / points of any tile (shared-memory sizing)
};

struct Lin {        // stored linearisation, SoA by component, index k*M + i
  double* r;        // [M][2] loss-corrected residuals (interleaved: one 16-byte access per observation)
  double* a;        // [3][M] a00, a02, a12
};

struct LossP {
  int type;
  double a;
};

// ceres::{Trivial,SoftLOne,Cauchy}Loss::Evaluate -> rho0, rho1 (rho2 <= 0 always, so the
// Corrector takes the first-order branch: residual and Jacobian scaled by sqrt(rho1)).
__device__ __forceinline__ void loss_eval(const LossP l, const double s, double& rho0, double& rho1) {
  if (l.type == PSFM_LOSS_SOFT_L1) {
    const double b = l.a * l.a, c = 1.0 / b;
    const double sum = 1.0 + s * c;
    const double tmp = sqrt(sum);
    rho0 = 2.0 * b * (tmp - 1.0);
    rho1 = fmax(2.2250738585072014e-308, 1.0 / tmp);
  } else if (l.type == PSFM_LOSS_CAUCHY) {
    const double b = l.a * l.a, c = 1.0 / b;
    const double sum = 1.0 + s * c;
    rho0 = b * log(sum);
    rho1 = fmax(2.2250738585072014e-308, 1.0 / sum);
  } else {
    rho0 = s;
    rho1 = 1.0;
  }
}

// ------------------------------------------------------------------ tile plumbing

// Shared memory of a tile kernel:
//   sv   [NV][TILE + 1]  per-observation values being reduced (row stride PSFM_SVS)
//   sw   [4][cap_np]     per-point scratch
//   sred [9*32]          block-reduction scratch
//   simg [cap_ns][14]    per image segment, AoS: R (row-major 9), t (3), pad (2) — 112 bytes: 16-byte aligned rows
//                        (one bulk copy per tile from seg_pose) and eight consecutive segments start in eight
//                        different groups of four banks
//   sx   [6][cap_ns]     per image segment: scaled input vector (rot 3 | t 3)
//   sxyz [cap_np][3]     per point, AoS: X
//   spt  rows 3..NPT-1   per point, SoA rows of stride pstr: H~ (rows 3-8), w^ or G'E focal row (9-11), w^ (12-14);
//                        row r starts at spt + r * pstr + lead, where lead (0 | 1 doubles) is what the 16-byte
//                        alignment of the bulk copy of that row left in front (0 in the non-pipelined kernels)
// Row stride of sv: TILE + 1 so that lanes working on different components k of the same
// observation column hit different banks (the reductions below run component-fastest).
#define PSFM_SVS (TILE + 1)
constexpr int PSFM_SPS = 14;      // doubles per segment pose record

template <int TILE>
struct TileSmem {
  double *sv, *sw, *sred, *simg, *sx, *spt, *sxyz;
  int *pstart, *coff, *cimg;
  unsigned short* perm;
  int cap_ns, cap_np;
  int pstr, plead0, plead1;    // spt row stride; lead of the rows that are EVEN / ODD rows of their global SoA array
  static size_t bytes(int nv, int npt, int cap_ns, int cap_np) {
    return sizeof(double) * ((size_t)nv * PSFM_SVS + 4 * (size_t)cap_np + 9 * 32 + (PSFM_SPS + 6) * (size_t)cap_ns + (size_t)npt * cap_np +
                             3 * (size_t)cap_np + 2) +
           sizeof(int) * ((size_t)cap_np + 2 * (size_t)cap_ns + 4) + sizeof(unsigned short) * (size_t)TILE + 32;
  }
  __device__ __forceinline__ void carve(unsigned char* base, int nv, int npt, int cns, int cnp) {
    cap_ns = cns; cap_np = cnp;
    pstr = cnp; plead0 = 0; plead1 = 0;
    sv = reinterpret_cast<double*>(base);
    sw = sv + (size_t)nv * PSFM_SVS;
    sred = sw + 4 * (size_t)cnp;
    simg = sred + 9 * 32;
    sx = simg + PSFM_SPS * (size_t)cns;
    spt = sx + 6 * (size_t)cns;
    sxyz = spt + (size_t)npt * cnp;
    pstart = reinterpret_cast<int*>(sxyz + 3 * (size_t)cnp + 2);
    coff = pstart + cnp + 1;
    cimg = coff + cns + 1;
    perm = reinterpret_cast<unsigned short*>(cimg + cns + 1);
  }
  // row r (3 .. 14) of the per-point SoA block: rows 3-8 are rows 0-5 of their global array, 9-11 and 12-14 rows 0-2
  __device__ __forceinline__ const double* prow(int r) const {
    const int kpar = (r < 12) ? ((r + 1) & 1) : (r & 1);
    return spt + (size_t)r * pstr + (kpar ? plead1 : plead0);
  }
  __device__ __forceinline__ double* prow_w(int r) const { return const_cast<double*>(prow(r)); }
};

struct TileInfo {
  int base, n, pt0, np, ns, cs0;
};

// Tile header: scalar loads.  The caller then issues ALL of its global loads before the
// barrier of tile_fill_smem(), so that a CTA pays one global-memory latency for the batch.
__device__ __forceinline__ TileInfo tile_header(const TileCtx& tc) {
  TileInfo ti;
  const int tile = blockIdx.x;
  ti.base = __ldg(tc.tile_start + tile);
  ti.n = __ldg(tc.tile_start + tile + 1) - ti.base;
  ti.pt0 = __ldg(tc.tile_pt + tile);
  ti.np = __ldg(tc.tile_pt + tile + 1) - ti.pt0;
  ti.cs0 = __ldg(tc.cseg_ptr + tile);
  ti.ns = __ldg(tc.cseg_ptr + tile + 1) - ti.cs0;
  return ti;
}

// pose16 row of an image: R (row-major 9), t (3), pad(4).  xs: scaled camera-side vector in
// slot layout [6F + 3C] (may be null).  X: [3P] points.  p6/p3: optional per-point SoA arrays
// ([6][P], [3][P]) staged after X.  Ends with a barrier.
template <int TILE>
__device__ __forceinline__ void tile_fill_smem(const TileCtx& tc, TileSmem<TILE>& sm, const TileInfo& ti,
                                               const double* __restrict__ pose16, const double* __restrict__ xs,
                                               const double* __restrict__ X, const double* __restrict__ p6,
                                               const double* __restrict__ p3, bool need_cam,
                                               const double* __restrict__ p3b = nullptr) {
  const int tid = threadIdx.x;
  const int cns = sm.cap_ns, cnp = sm.cap_np;
  for (int j = tid; j <= ti.np; j += TILE) sm.pstart[j] = __ldg(tc.pt_ptr + ti.pt0 + j) - ti.base;
  for (int j = tid; j < ti.ns; j += TILE) {
    sm.cimg[j] = __ldg(tc.cseg_img + ti.cs0 + j);
    if (need_cam) sm.coff[j] = __ldg(tc.cseg_off + ti.cs0 + j);
  }
  if (need_cam) {
    if (tid == 0) sm.coff[ti.ns] = ti.n;
    if (tid < ti.n) sm.perm[tid] = __ldg(tc.tile_perm + ti.base + tid);
  }
  for (int j = tid; j < ti.ns * 12; j += TILE) {
    const int s = j / 12, k = j - 12 * s;
    const int img = __ldg(tc.cseg_img + ti.cs0 + s);
    sm.simg[s * PSFM_SPS + k] = __ldg(pose16 + 16 * (size_t)img + k);
  }
  if (xs) {
    for (int j = tid; j < ti.ns * 6; j += TILE) {
      const int s = j / 6, k = j - 6 * s;
      const int img = __ldg(tc.cseg_img + ti.cs0 + s);
      sm.sx[k * cns + s] = __ldg(xs + 6 * (size_t)img + k);
    }
  }
  for (int j = tid; j < ti.np * 3; j += TILE) sm.sxyz[j] = __ldg(X + 3 * (size_t)ti.pt0 + j);
  if (p6) {
    for (int j = tid; j < ti.np * 6; j += TILE) {
      const int k = j / ti.np, l = j - k * ti.np;
      sm.prow_w(3 + k)[l] = __ldg(p6 + (size_t)k * tc.P + ti.pt0 + l);
    }
  }
  if (p3) {
    for (int j = tid; j < ti.np * 3; j += TILE) {
      const int k = j / ti.np, l = j - k * ti.np;
      sm.prow_w(9 + k)[l] = __ldg(p3 + (size_t)k * tc.P + ti.pt0 + l);
    }
  }
  if (p3b) {
    for (int j = tid; j < ti.np * 3; j += TILE) {
      const int k = j / ti.np, l = j - k * ti.np;
      sm.prow_w(12 + k)[l] = __ldg(p3b + (size_t)k * tc.P + ti.pt0 + l);
    }
  }
  __syncthreads();
}

// N block sums with one barrier pair; results valid in threads 0..N-1 (thread j holds
// value j) — all threads must call.
template <int N>
__device__ __forceinline__ double block_sum_multi(const double (&v)[N], double* sbuf) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  __syncthreads();
#pragma unroll
  for (int j = 0; j < N; ++j) {
    const double s = warp_sum(v[j]);
    if (lane == 0) sbuf[j * 32 + wid] = s;
  }
  __syncthreads();
  double out = 0.0;
  if (threadIdx.x < N) {
    for (int w = 0; w < nw; ++w) out += sbuf[threadIdx.x * 32 + w];
  }
  return out;
}

// per (point, component) sums of sv rows [0, nv) -> fn(k, local point, sum)
template <int TILE, typename Fn>
__device__ __forceinline__ void tile_reduce_points(const TileSmem<TILE>& sm, const TileInfo& ti, int nv, Fn fn) {
  for (int pair = threadIdx.x; pair < nv * ti.np; pair += TILE) {
    const int l = pair / nv, k = pair - l * nv;       // component fastest: conflict-free rows, see PSFM_SVS
    const double* row = sm.sv + k * PSFM_SVS;
    double acc = 0.0;
    int e = sm.pstart[l];
    const int e1 = sm.pstart[l + 1];
    for (; e + 4 <= e1; e += 4) {
      const double v0 = row[e], v1 = row[e + 1], v2 = row[e + 2], v3 = row[e + 3];
      acc += v0; acc += v1; acc += v2; acc += v3;
    }
    for (; e < e1; ++e) acc += row[e];
    fn(k, l, acc);
  }
}

// per (image segment, component) sums of sv rows -> fn(k, image, sum)
template <int TILE, typename Fn>
__device__ __forceinline__ void tile_reduce_images(const TileSmem<TILE>& sm, const TileInfo& ti, int nv, Fn fn) {
  for (int pair = threadIdx.x; pair < nv * ti.ns; pair += TILE) {
    const int s = pair / nv, k = pair - s * nv;       // component fastest; perm[e] is a broadcast
    const double* row = sm.sv + k * PSFM_SVS;
    double acc = 0.0;
    // same order of additions as the plain loop; four loads in flight instead of one dependent pair per element
    int e = sm.coff[s];
    const int e1 = sm.coff[s + 1];
    for (; e + 4 <= e1; e += 4) {
      const int i0 = sm.perm[e], i1 = sm.perm[e + 1], i2 = sm.perm[e + 2], i3 = sm.perm[e + 3];
      const double v0 = row[i0], v1 = row[i1], v2 = row[i2], v3 = row[i3];
      acc += v0; acc += v1; acc += v2; acc += v3;
    }
    for (; e < e1; ++e) acc += row[sm.perm[e]];
    fn(k, sm.cimg[s], acc);
  }
}

// ------------------------------------------------------------------ per-observation geometry

struct ObsGeom {
  double R[9];
  double w[3];      // R X
  double tz;
};

template <int TILE>
__device__ __forceinline__ void load_geom(const TileSmem<TILE>& sm, int ls, int lp, ObsGeom& g) {
  const int cns = sm.cap_ns, cnp = sm.cap_np;
#pragma unroll
  for (int k = 0; k < 9; ++k) g.R[k] = sm.simg[ls * PSFM_SPS + k];
  g.tz = sm.simg[ls * PSFM_SPS + 11];
  const double X0 = sm.sxyz[3 * lp], X1 = sm.sxyz[3 * lp + 1], X2 = sm.sxyz[3 * lp + 2];
#pragma unroll
  for (int a = 0; a < 3; ++a) g.w[a] = g.R[3 * a] * X0 + g.R[3 * a + 1] * X1 + g.R[3 * a + 2] * X2;
}

// u = J_cam x~  (unscaled J, scaled input): y3 = x~_t + 2 x~_r x w ; u = D y3 (+ focal / pp)
template <int TILE, bool ROT>
__device__ __forceinline__ void apply_Jc(const TileSmem<TILE>& sm, int ls, const ObsGeom& g, double a00, double a02,
                                         double a12, int intr, const double* xk, double inv_f, double& u0, double& u1,
                                         double& jf0, double& jf1, double& sq) {
  const int cns = sm.cap_ns;
  double y0 = sm.sx[3 * cns + ls], y1 = sm.sx[4 * cns + ls], y2 = sm.sx[5 * cns + ls];
  if (ROT) {
    const double r0 = sm.sx[ls], r1 = sm.sx[cns + ls], r2 = sm.sx[2 * cns + ls];
    y0 += 2.0 * (r1 * g.w[2] - r2 * g.w[1]);
    y1 += 2.0 * (r2 * g.w[0] - r0 * g.w[2]);
    y2 += 2.0 * (r0 * g.w[1] - r1 * g.w[0]);
  }
  u0 = a00 * y0 + a02 * y2;
  u1 = a00 * y1 + a12 * y2;
  jf0 = jf1 = sq = 0.0;
  if (intr >= 1) {
    const double zf = (g.w[2] + g.tz) * inv_f;
    jf0 = -a02 * zf;          // sq * u
    jf1 = -a12 * zf;          // sq * v
    u0 += jf0 * xk[0];
    u1 += jf1 * xk[0];
    if (intr == 3) {
      sq = a00 * zf;
      u0 += sq * xk[1];
      u1 += sq * xk[2];
    }
  }
}

// ------------------------------------------------------------------ K1: Jacobian sweep

struct LinArgs {
  const double* pose16;   // [F*16] R(9) t(3)
  const double* X;        // [P*3]
  const double* K;        // [C*3]
  LossP loss;
  int intr;               // 0: intrinsics constant, 1: focal only, 3: focal + principal point
  Lin L;
  double* hpp;            // [6][P]  E'E unscaled (upper: 00 01 02 11 12 22)
  double* gp;             // [3][P]  E'r
  double* wk;             // [9][P]  (G'E) rows: focal (3) | cx (3) | cy (3)
  double* acc_cam;        // [NREP][F][NVL] rot F'F (6) | t F'F (6) | g rot (3) | g t (3)   (unscaled)
  size_t rep_stride;
  double* acc_intr;       // [C][NVI] G'G (6: ff fx fy xx xy yy) | g_k (3)
  double* acc_cost;       // [1]
};

// One tile of the Jacobian sweep.  Shared memory (sm.simg, sm.spt, sm.pstart, sm.coff, sm.cimg,
// sm.perm) holds the tile's staged inputs and is synchronised; ls / lp / xy are this thread's
// observation.  Ends without a barrier.
// racc (optional, shared memory [3][TILE]): the persistent kernel accumulates the block-wide sums (cost, focal terms)
// per THREAD across its tiles and reduces them once at the end (linearize_flush) instead of a barrier pair per tile;
// the principal-point sums (intr == 3: not what the pipeline runs) keep their per-tile block sum.
template <int TILE, bool ROT>
__device__ __forceinline__ void linearize_tile(const TileCtx& tc, const LinArgs& a, TileSmem<TILE>& sm, const TileInfo& ti,
                                               const bool act, const int ls, const int lp, const double2 xy, const int rep,
                                               double* racc = nullptr) {
  const int tid = threadIdx.x;
  const size_t M = tc.M;
  const size_t i = (size_t)ti.base + tid;
  double r0 = 0, r1 = 0, cost = 0, a00 = 0, a02 = 0, a12 = 0, jf0 = 0, jf1 = 0, sq = 0;
  double jp0[3] = {0, 0, 0}, jp1[3] = {0, 0, 0};
  ObsGeom g;
#pragma unroll
  for (int k = 0; k < 3; ++k) g.w[k] = 0.0;
  if (act) {
    load_geom<TILE>(sm, ls, lp, g);
    const int cns = sm.cap_ns;
    const double p0 = g.w[0] + sm.simg[ls * PSFM_SPS + 9], p1 = g.w[1] + sm.simg[ls * PSFM_SPS + 10], p2 = g.w[2] + g.tz;
    const double iz = 1.0 / p2;
    const double u = p0 * iz, v = p1 * iz;
    const int cam = __ldg(tc.img_cam + sm.cimg[ls]);
    const double f = __ldg(a.K + 3 * cam), cx = __ldg(a.K + 3 * cam + 1), cy = __ldg(a.K + 3 * cam + 2);
    const double e0 = f * u + cx - xy.x, e1 = f * v + cy - xy.y;
    double rho0, rho1;
    loss_eval(a.loss, e0 * e0 + e1 * e1, rho0, rho1);
    sq = sqrt(rho1);
    cost = 0.5 * rho0;
    r0 = sq * e0;
    r1 = sq * e1;
    a00 = sq * f * iz;
    a02 = -a00 * u;
    a12 = -a00 * v;
    reinterpret_cast<double2*>(a.L.r)[i] = make_double2(r0, r1);
    a.L.a[i] = a00;
    a.L.a[M + i] = a02;
    a.L.a[2 * M + i] = a12;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      jp0[k] = a00 * g.R[k] + a02 * g.R[6 + k];
      jp1[k] = a00 * g.R[3 + k] + a12 * g.R[6 + k];
    }
    jf0 = sq * u;
    jf1 = sq * v;
  }

  // ---- point side: E'E (6), E'r (3), G'E (3 per free intrinsic) ----
  const int nvp = 9 + 3 * a.intr;
  {
    double* sv = sm.sv + tid;
    sv[0 * PSFM_SVS] = jp0[0] * jp0[0] + jp1[0] * jp1[0];
    sv[1 * PSFM_SVS] = jp0[0] * jp0[1] + jp1[0] * jp1[1];
    sv[2 * PSFM_SVS] = jp0[0] * jp0[2] + jp1[0] * jp1[2];
    sv[3 * PSFM_SVS] = jp0[1] * jp0[1] + jp1[1] * jp1[1];
    sv[4 * PSFM_SVS] = jp0[1] * jp0[2] + jp1[1] * jp1[2];
    sv[5 * PSFM_SVS] = jp0[2] * jp0[2] + jp1[2] * jp1[2];
#pragma unroll
    for (int k = 0; k < 3; ++k) sv[(6 + k) * PSFM_SVS] = jp0[k] * r0 + jp1[k] * r1;
    if (a.intr >= 1) {
#pragma unroll
      for (int k = 0; k < 3; ++k) sv[(9 + k) * PSFM_SVS] = jf0 * jp0[k] + jf1 * jp1[k];
      if (a.intr == 3) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          sv[(12 + k) * PSFM_SVS] = sq * jp0[k];
          sv[(15 + k) * PSFM_SVS] = sq * jp1[k];
        }
      }
    }
  }
  __syncthreads();
  tile_reduce_points<TILE>(sm, ti, nvp, [&](int k, int l, double acc) {
    const size_t gpt = (size_t)ti.pt0 + l;
    if (k < 6) a.hpp[(size_t)k * tc.P + gpt] = acc;
    else if (k < 9) a.gp[(size_t)(k - 6) * tc.P + gpt] = acc;
    else a.wk[(size_t)(k - 9) * tc.P + gpt] = acc;
  });
  __syncthreads();

  // ---- image side: diagonal 3x3 blocks of F'F (rot | t) and F'r, unscaled ----
  {
    double* sv = sm.sv + tid;
    if (ROT) {
      const double jr00 = 2.0 * a02 * g.w[1], jr01 = 2.0 * (a00 * g.w[2] - a02 * g.w[0]), jr02 = -2.0 * a00 * g.w[1];
      const double jr10 = 2.0 * (a12 * g.w[1] - a00 * g.w[2]), jr11 = -2.0 * a12 * g.w[0], jr12 = 2.0 * a00 * g.w[0];
      sv[0 * PSFM_SVS] = jr00 * jr00 + jr10 * jr10;
      sv[1 * PSFM_SVS] = jr00 * jr01 + jr10 * jr11;
      sv[2 * PSFM_SVS] = jr00 * jr02 + jr10 * jr12;
      sv[3 * PSFM_SVS] = jr01 * jr01 + jr11 * jr11;
      sv[4 * PSFM_SVS] = jr01 * jr02 + jr11 * jr12;
      sv[5 * PSFM_SVS] = jr02 * jr02 + jr12 * jr12;
      sv[12 * PSFM_SVS] = jr00 * r0 + jr10 * r1;
      sv[13 * PSFM_SVS] = jr01 * r0 + jr11 * r1;
      sv[14 * PSFM_SVS] = jr02 * r0 + jr12 * r1;
    }
    sv[6 * PSFM_SVS] = a00 * a00;
    sv[7 * PSFM_SVS] = 0.0;
    sv[8 * PSFM_SVS] = a00 * a02;
    sv[9 * PSFM_SVS] = a00 * a00;
    sv[10 * PSFM_SVS] = a00 * a12;
    sv[11 * PSFM_SVS] = a02 * a02 + a12 * a12;
    sv[15 * PSFM_SVS] = a00 * r0;
    sv[16 * PSFM_SVS] = a00 * r1;
    sv[17 * PSFM_SVS] = a02 * r0 + a12 * r1;
  }
  __syncthreads();
  {
    // components handled: ROT -> 0..17, else 6..11 and 15..17 (9 values); 7 is structurally 0
    double* dst = a.acc_cam + (size_t)(rep & (NREP - 1)) * a.rep_stride;
    const int nvc = ROT ? 18 : 9;
    for (int pair = tid; pair < nvc * ti.ns; pair += TILE) {
      const int s = pair / nvc;
      int k = pair - s * nvc;
      if (!ROT) k = (k < 6) ? k + 6 : k + 9;
      if (k == 7) continue;
      const double* row = sm.sv + k * PSFM_SVS;
      double acc = 0.0;
      for (int e = sm.coff[s]; e < sm.coff[s + 1]; ++e) acc += row[sm.perm[e]];
      atomicAdd(dst + (size_t)sm.cimg[s] * NVL + k, acc);
    }
  }
  // ---- cost and intrinsics (block sums; a single shared camera when intrinsics are free) ----
  {
    double v[3];
    v[0] = cost;
    v[1] = jf0 * jf0 + jf1 * jf1;
    v[2] = jf0 * r0 + jf1 * r1;
    double u[7];
    u[0] = jf0 * sq;                 // f-cx
    u[1] = jf1 * sq;                 // f-cy
    u[2] = act ? sq * sq : 0.0;      // cx-cx
    u[3] = 0.0;                      // cx-cy
    u[4] = act ? sq * sq : 0.0;      // cy-cy
    u[5] = sq * r0;                  // g cx
    u[6] = sq * r1;                  // g cy
    if (racc != nullptr) {
      // per-thread running sums in shared memory (stride TILE; registers are what this kernel has least of)
#pragma unroll
      for (int k = 0; k < 3; ++k) racc[k * TILE + tid] += v[k];
    } else {
      const double s = block_sum_multi<3>(v, sm.sred);
      if (tid == 0) atomicAdd(a.acc_cost, s);
      if (a.intr >= 1) {
        if (tid == 1) atomicAdd(a.acc_intr + 0, s);
        if (tid == 2) atomicAdd(a.acc_intr + 6, s);
      }
    }
    if (a.intr == 3) {
      const double s2 = block_sum_multi<7>(u, sm.sred);
      if (tid < 5) atomicAdd(a.acc_intr + 1 + tid, s2);
      else if (tid < 7) atomicAdd(a.acc_intr + 7 + (tid - 5), s2);
    }
  }
}

// the deferred sums of a persistent CTA (racc of linearize_tile) -> global accumulators
template <int TILE>
__device__ __forceinline__ void linearize_flush(const LinArgs& a, const double* racc, double* sred) {
  const int tid = threadIdx.x;
  double v[3] = {racc[tid], racc[TILE + tid], racc[2 * TILE + tid]};
  const double s = block_sum_multi<3>(v, sred);
  if (tid == 0) atomicAdd(a.acc_cost, s);
  if (a.intr >= 1) {
    if (tid == 1) atomicAdd(a.acc_intr + 0, s);
    if (tid == 2) atomicAdd(a.acc_intr + 6, s);
  }
}

template <int TILE, bool ROT>
__global__ void __launch_bounds__(TILE, (TILE == 256 ? 3 : 1)) k_linearize(const TileCtx tc, const LinArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  TileSmem<TILE> sm;
  sm.carve(smem_raw, 18, 3, tc.cap_ns, tc.cap_np);
  const TileInfo ti = tile_header(tc);
  const int tid = threadIdx.x;
  const bool act = tid < ti.n;
  const size_t i = (size_t)ti.base + tid;
  int ls = 0, lp = 0;
  double2 xy = make_double2(0.0, 0.0);
  if (act) {
    ls = __ldg(tc.obs_lseg + i);
    lp = __ldg(tc.obs_lpt + i);
    xy = tc.obs_xy[i];
  }
  tile_fill_smem<TILE>(tc, sm, ti, a.pose16, nullptr, a.X, nullptr, nullptr, true);
  linearize_tile<TILE, ROT>(tc, a, sm, ti, act, ls, lp, xy, blockIdx.x);
}

// ------------------------------------------------------------------ K2: point blocks

struct PtsArgs {
  const double* hpp;   // [6][P] unscaled E'E
  const double* gp;    // [3][P] unscaled E'r
  const double* wk;    // [9][P] unscaled G'E
  const double* scale_p;  // [3P]
  double radius, min_diag, max_diag;
  int intr;
  int P;
  double* ht;          // [6][P] H~ = diag(s_p) (s_p E'E s_p + D^2)^-1 diag(s_p)
  double* wt;          // [3][P] w^ = H~ E'r
  // factor of H~ for the fused exact Schur kernel (null: not written).  With s_p E'E s_p + D^2 = L L',
  // G = diag(s_p) L^-T is upper triangular and G G' = H~
  double* gf;          // [6][P] G packed [g00 g01 g02 g11 g12 g22]
  double* gv;          // [3][P] G' (focal row of G'E)
  double* gu;          // [3][P] G' E'r
  double* acc_intr;   // [NVI] -(G'E) H~ (E'G) (6) | -(G'E) w^ (3)   (unscaled in the intrinsics)
  double* acc_fail;    // [1] > 0 when a block is not positive definite
  double* gmax;        // [1] max |gradient| over point parameters (atomic max)
};

__global__ void __launch_bounds__(256) k_point_blocks(const PtsArgs a) {
  __shared__ double sred[9 * 32];
  const int p = blockIdx.x * 256 + threadIdx.x;
  double gm = 0.0, fail = 0.0;
  double ci[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) ci[k] = 0.0;
  if (p < a.P) {
    const size_t P = a.P;
    const double s0 = a.scale_p[3 * (size_t)p], s1 = a.scale_p[3 * (size_t)p + 1], s2 = a.scale_p[3 * (size_t)p + 2];
    double h00 = a.hpp[p] * s0 * s0, h01 = a.hpp[P + p] * s0 * s1, h02 = a.hpp[2 * P + p] * s0 * s2,
           h11 = a.hpp[3 * P + p] * s1 * s1, h12 = a.hpp[4 * P + p] * s1 * s2, h22 = a.hpp[5 * P + p] * s2 * s2;
    const double g0 = a.gp[p], g1 = a.gp[P + p], g2 = a.gp[2 * P + p];
    // LevenbergMarquardtStrategy: D^2 = clamp(diag(J'J)) / radius  (scaled Jacobian)
    h00 += fmin(fmax(h00, a.min_diag), a.max_diag) / a.radius;
    h11 += fmin(fmax(h11, a.min_diag), a.max_diag) / a.radius;
    h22 += fmin(fmax(h22, a.min_diag), a.max_diag) / a.radius;
    // Cholesky-based inverse
    bool bad = !(h00 > 0.0);
    const double l00 = sqrt(h00);
    const double l10 = h01 / l00, l20 = h02 / l00;
    double d = h11 - l10 * l10;
    bad |= !(d > 0.0);
    const double l11 = sqrt(d);
    const double l21 = (h12 - l20 * l10) / l11;
    d = h22 - l20 * l20 - l21 * l21;
    bad |= !(d > 0.0);
    const double l22 = sqrt(d);
    const double i00 = 1.0 / l00, i11 = 1.0 / l11, i22 = 1.0 / l22;
    const double i10 = -l10 * i00 * i11;
    const double i21 = -l21 * i11 * i22;
    const double i20 = -(l20 * i00 + l21 * i10) * i22;
    double v00 = i00 * i00 + i10 * i10 + i20 * i20, v01 = i10 * i11 + i20 * i21, v02 = i20 * i22,
           v11 = i11 * i11 + i21 * i21, v12 = i21 * i22, v22 = i22 * i22;
    if (bad) { fail = 1.0; v00 = v11 = v22 = 1.0; v01 = v02 = v12 = 0.0; }
    if (a.gf) {
      // G = diag(s) L^-T (diag(s) where the inverse above was replaced by the identity)
      double f00 = s0, f01 = 0.0, f02 = 0.0, f11 = s1, f12 = 0.0, f22 = s2;
      if (!bad) { f00 = s0 * i00; f01 = s0 * i10; f02 = s0 * i20; f11 = s1 * i11; f12 = s1 * i21; f22 = s2 * i22; }
      a.gf[p] = f00; a.gf[P + p] = f01; a.gf[2 * P + p] = f02;
      a.gf[3 * P + p] = f11; a.gf[4 * P + p] = f12; a.gf[5 * P + p] = f22;
      a.gu[p] = f00 * g0; a.gu[P + p] = f01 * g0 + f11 * g1; a.gu[2 * P + p] = f02 * g0 + f12 * g1 + f22 * g2;
      double k0 = 0.0, k1 = 0.0, k2 = 0.0;
      if (a.intr >= 1) { k0 = a.wk[p]; k1 = a.wk[P + p]; k2 = a.wk[2 * P + p]; }
      a.gv[p] = f00 * k0; a.gv[P + p] = f01 * k0 + f11 * k1; a.gv[2 * P + p] = f02 * k0 + f12 * k1 + f22 * k2;
    }
    // H~ = diag(s) Hinv diag(s)
    v00 *= s0 * s0; v01 *= s0 * s1; v02 *= s0 * s2; v11 *= s1 * s1; v12 *= s1 * s2; v22 *= s2 * s2;
    a.ht[p] = v00; a.ht[P + p] = v01; a.ht[2 * P + p] = v02;
    a.ht[3 * P + p] = v11; a.ht[4 * P + p] = v12; a.ht[5 * P + p] = v22;
    const double w0 = v00 * g0 + v01 * g1 + v02 * g2;
    const double w1 = v01 * g0 + v11 * g1 + v12 * g2;
    const double w2 = v02 * g0 + v12 * g1 + v22 * g2;
    a.wt[p] = w0; a.wt[P + p] = w1; a.wt[2 * P + p] = w2;
    gm = fmax(fmax(fabs(g0), fabs(g1)), fabs(g2));
    if (a.intr >= 1) {
      double W[3][3], WH[3][3];
      for (int j = 0; j < 3; ++j)
        for (int k = 0; k < 3; ++k) W[j][k] = (j < a.intr) ? a.wk[(size_t)(3 * j + k) * P + p] : 0.0;
      for (int j = 0; j < 3; ++j) {
        WH[j][0] = W[j][0] * v00 + W[j][1] * v01 + W[j][2] * v02;
        WH[j][1] = W[j][0] * v01 + W[j][1] * v11 + W[j][2] * v12;
        WH[j][2] = W[j][0] * v02 + W[j][1] * v12 + W[j][2] * v22;
      }
      int c = 0;
      for (int j = 0; j < 3; ++j)
        for (int k = j; k < 3; ++k) ci[c++] = -(WH[j][0] * W[k][0] + WH[j][1] * W[k][1] + WH[j][2] * W[k][2]);
      for (int j = 0; j < 3; ++j) ci[6 + j] = -(W[j][0] * w0 + W[j][1] * w1 + W[j][2] * w2);
    }
  }
  const double m = block_max(gm, sred);
  if (threadIdx.x == 0 && m > 0.0) atomic_max_nonneg(a.gmax, m);
  const double f = block_sum(fail, sred);
  if (threadIdx.x == 0 && f > 0.0) atomicAdd(a.acc_fail, f);
  if (a.intr >= 1) {
    const double s = block_sum_multi<9>(ci, sred);
    if (threadIdx.x < 9) atomicAdd(a.acc_intr + threadIdx.x, s);
  }
}

// ------------------------------------------------------------------ K3: Schur-Jacobi / rhs corrections

struct PrepArgs {
  Lin L;
  const double* pose16;
  const double* X;
  const double* ht;     // [6][P]
  const double* wt;     // [3][P]
  double* acc_cam;      // [NREP][F][NVL]: -(W H~ W') rot (6) | t (6) | -(W w^) rot (3) | t (3)   (unscaled)
  size_t rep_stride;
};

template <int TILE, bool ROT>
__global__ void __launch_bounds__(TILE, (TILE == 256 ? 2 : 1)) k_schur_prep(const TileCtx tc, const PrepArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  TileSmem<TILE> sm;
  sm.carve(smem_raw, 18, 12, tc.cap_ns, tc.cap_np);
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
  tile_fill_smem<TILE>(tc, sm, ti, a.pose16, nullptr, a.X, a.ht, a.wt, true);
  double* sv = sm.sv + tid;
  if (act) {
    ObsGeom g;
    load_geom<TILE>(sm, ls, lp, g);
    const int cnp = sm.cap_np;
    double hv[6], w[3];
#pragma unroll
    for (int k = 0; k < 6; ++k) hv[k] = sm.prow(3 + k)[lp];
#pragma unroll
    for (int k = 0; k < 3; ++k) w[k] = sm.prow(9 + k)[lp];
    double jp[2][3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      jp[0][k] = a00 * g.R[k] + a02 * g.R[6 + k];
      jp[1][k] = a00 * g.R[3 + k] + a12 * g.R[6 + k];
    }
    // block b: 0 = rot (ROT only), 1 = translation
#pragma unroll
    for (int b = (ROT ? 0 : 1); b < 2; ++b) {
      double jc0[3], jc1[3];
      if (b == 0) {
        jc0[0] = 2.0 * a02 * g.w[1]; jc0[1] = 2.0 * (a00 * g.w[2] - a02 * g.w[0]); jc0[2] = -2.0 * a00 * g.w[1];
        jc1[0] = 2.0 * (a12 * g.w[1] - a00 * g.w[2]); jc1[1] = -2.0 * a12 * g.w[0]; jc1[2] = 2.0 * a00 * g.w[0];
      } else {
        jc0[0] = a00; jc0[1] = 0.0; jc0[2] = a02;
        jc1[0] = 0.0; jc1[1] = a00; jc1[2] = a12;
      }
      double W[3][3], WH[3][3];
#pragma unroll
      for (int j = 0; j < 3; ++j)
#pragma unroll
        for (int k = 0; k < 3; ++k) W[j][k] = jc0[j] * jp[0][k] + jc1[j] * jp[1][k];
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        WH[j][0] = W[j][0] * hv[0] + W[j][1] * hv[1] + W[j][2] * hv[2];
        WH[j][1] = W[j][0] * hv[1] + W[j][1] * hv[3] + W[j][2] * hv[4];
        WH[j][2] = W[j][0] * hv[2] + W[j][1] * hv[4] + W[j][2] * hv[5];
      }
      int c = 6 * b;
#pragma unroll
      for (int j = 0; j < 3; ++j)
#pragma unroll
        for (int k = j; k < 3; ++k) { sv[c * PSFM_SVS] = -(WH[j][0] * W[k][0] + WH[j][1] * W[k][1] + WH[j][2] * W[k][2]); ++c; }
#pragma unroll
      for (int j = 0; j < 3; ++j) sv[(12 + 3 * b + j) * PSFM_SVS] = -(W[j][0] * w[0] + W[j][1] * w[1] + W[j][2] * w[2]);
    }
  }
  __syncthreads();
  double* dst = a.acc_cam + (size_t)(blockIdx.x & (NREP - 1)) * a.rep_stride;
  const int nvc = ROT ? 18 : 9;
  for (int pair = tid; pair < nvc * ti.ns; pair += TILE) {
    const int s = pair / nvc;
    int k = pair - s * nvc;
    if (!ROT) k = (k < 6) ? k + 6 : k + 9;
    const double* row = sm.sv + k * PSFM_SVS;
    double acc = 0.0;
    for (int e = sm.coff[s]; e < sm.coff[s + 1]; ++e) acc += row[sm.perm[e]];
    atomicAdd(dst + (size_t)sm.cimg[s] * NVL + k, acc);
  }
}

// ------------------------------------------------------------------ K4: implicit S * p

struct SpArgs {
  Lin L;
  const double* pose16;
  const double* X;
  const double* ht;     // [6][P]
  const double* xs;     // [6F + 3C] scaled input vector s o x (slot layout)
  double* y;            // [NREP][6F + 3C] += F'(I - E H~ E') F xs   (unscaled; folded and scaled later)
  size_t rep_stride;
  const int* flag;      // PCG state: != 0 -> nothing to do
  const double* K;      // [3C]
  int intr;
};

#ifndef PSFM_SP_MINB
#define PSFM_SP_MINB 4
#endif
template <int TILE, bool ROT>
__global__ void __launch_bounds__(TILE, (TILE == 256 ? PSFM_SP_MINB : 1)) k_schur_product(const TileCtx tc, const SpArgs a) {
  if (*a.flag != 0) return;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  TileSmem<TILE> sm;
  sm.carve(smem_raw, 6, 9, tc.cap_ns, tc.cap_np);
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
  double xk[3] = {0, 0, 0};
  double inv_f = 0.0;
  if (a.intr >= 1) {
    xk[0] = __ldg(a.xs + 6 * (size_t)tc.F); xk[1] = __ldg(a.xs + 6 * (size_t)tc.F + 1); xk[2] = __ldg(a.xs + 6 * (size_t)tc.F + 2);
    inv_f = 1.0 / __ldg(a.K);
  }
  tile_fill_smem<TILE>(tc, sm, ti, a.pose16, a.xs, a.X, a.ht, nullptr, true);
  ObsGeom g;
  double u0 = 0, u1 = 0, jf0 = 0, jf1 = 0, sq = 0;
#pragma unroll
  for (int k = 0; k < 9; ++k) g.R[k] = 0.0;
#pragma unroll
  for (int k = 0; k < 3; ++k) g.w[k] = 0.0;
  if (act) {
    load_geom<TILE>(sm, ls, lp, g);
    apply_Jc<TILE, ROT>(sm, ls, g, a00, a02, a12, a.intr, xk, inv_f, u0, u1, jf0, jf1, sq);
  }
  double* sv = sm.sv + tid;
  {
    // E'u = R'(D'u)
    const double d0 = a00 * u0, d1 = a00 * u1, d2 = a02 * u0 + a12 * u1;
#pragma unroll
    for (int k = 0; k < 3; ++k) sv[k * PSFM_SVS] = g.R[k] * d0 + g.R[3 + k] * d1 + g.R[6 + k] * d2;
  }
  __syncthreads();
  const int cnp = sm.cap_np;
  tile_reduce_points<TILE>(sm, ti, 3, [&](int k, int l, double acc) { sm.sw[k * cnp + l] = acc; });
  __syncthreads();
  if (tid < ti.np) {
    const double t0 = sm.sw[tid], t1 = sm.sw[cnp + tid], t2 = sm.sw[2 * cnp + tid];
    const double h0 = sm.prow(3)[tid], h1 = sm.prow(4)[tid], h2 = sm.prow(5)[tid],
                 h3 = sm.prow(6)[tid], h4 = sm.prow(7)[tid], h5 = sm.prow(8)[tid];
    sm.sw[tid] = h0 * t0 + h1 * t1 + h2 * t2;
    sm.sw[cnp + tid] = h1 * t0 + h3 * t1 + h4 * t2;
    sm.sw[2 * cnp + tid] = h2 * t0 + h4 * t1 + h5 * t2;
  }
  __syncthreads();
  double v0 = 0, v1 = 0;
  {
    const double z0 = sm.sw[lp], z1 = sm.sw[cnp + lp], z2 = sm.sw[2 * cnp + lp];
    // E z = D (R z)
    const double y0 = g.R[0] * z0 + g.R[1] * z1 + g.R[2] * z2;
    const double y1 = g.R[3] * z0 + g.R[4] * z1 + g.R[5] * z2;
    const double y2 = g.R[6] * z0 + g.R[7] * z1 + g.R[8] * z2;
    v0 = u0 - (a00 * y0 + a02 * y2);
    v1 = u1 - (a00 * y1 + a12 * y2);
  }
  __syncthreads();   // sv is rewritten below
  {
    // F'v: e = D'v ; rot = 2 w x e ; t = e
    const double e0 = a00 * v0, e1 = a00 * v1, e2 = a02 * v0 + a12 * v1;
    if (ROT) {
      sv[0 * PSFM_SVS] = 2.0 * (g.w[1] * e2 - g.w[2] * e1);
      sv[1 * PSFM_SVS] = 2.0 * (g.w[2] * e0 - g.w[0] * e2);
      sv[2 * PSFM_SVS] = 2.0 * (g.w[0] * e1 - g.w[1] * e0);
      sv[3 * PSFM_SVS] = e0; sv[4 * PSFM_SVS] = e1; sv[5 * PSFM_SVS] = e2;
    } else {
      sv[0 * PSFM_SVS] = e0; sv[1 * PSFM_SVS] = e1; sv[2 * PSFM_SVS] = e2;
    }
  }
  __syncthreads();
  {
    constexpr int NC = ROT ? 6 : 3;
    double* dst = a.y + (size_t)(blockIdx.x & (NREP - 1)) * a.rep_stride + (ROT ? 0 : 3);
    tile_reduce_images<TILE>(sm, ti, NC, [&](int k, int img, double acc) { atomicAdd(dst + 6 * (size_t)img + k, acc); });
  }
  if (a.intr >= 1) {
    double v[3];
    v[0] = jf0 * v0 + jf1 * v1;
    v[1] = sq * v0;
    v[2] = sq * v1;
    const double s = block_sum_multi<3>(v, sm.sred);
    if (tid < a.intr) atomicAdd(a.y + (size_t)(blockIdx.x & (NREP - 1)) * a.rep_stride + 6 * (size_t)tc.F + tid, s);
  }
}

// ------------------------------------------------------------------ K5: back-substitution + model cost + candidate points

struct BackArgs {
  Lin L;
  const double* pose16;
  const double* X;      // [3P] current points
  const double* ht;     // [6][P]
  const double* wt;     // [3][P] H~ E'r
  const double* xs;     // [6F + 3C] s o y_c  (y_c = reduced-system solution; step_c = -y_c)
  const double* K;
  double* Xc;           // [3P] candidate points
  double* acc;          // [0] sum m(r + m/2)   [1] |dX|^2   [2] |Xc|^2
  int intr;
};

// One tile of the back-substitution.  Shared memory (sm.simg, sm.sx, sm.spt rows 0..11, sm.pstart) holds the tile's
// staged inputs and is synchronised; the arguments are this thread's observation.  Ends with the tile's REDs.
template <int TILE, bool ROT>
__device__ __forceinline__ void back_substitute_tile(const TileCtx& tc, const BackArgs& a, TileSmem<TILE>& sm, const TileInfo& ti,
                                                     const bool act, const int ls, const int lp, const double a00, const double a02,
                                                     const double a12, const double r0, const double r1, const double* xk,
                                                     const double inv_f, double* racc = nullptr) {
  const int tid = threadIdx.x;
  ObsGeom g;
  double u0 = 0, u1 = 0, jf0 = 0, jf1 = 0, sq = 0;
#pragma unroll
  for (int k = 0; k < 9; ++k) g.R[k] = 0.0;
#pragma unroll
  for (int k = 0; k < 3; ++k) g.w[k] = 0.0;
  if (act) {
    load_geom<TILE>(sm, ls, lp, g);
    apply_Jc<TILE, ROT>(sm, ls, g, a00, a02, a12, a.intr, xk, inv_f, u0, u1, jf0, jf1, sq);
  }
  double* sv = sm.sv + tid;
  {
    const double d0 = a00 * u0, d1 = a00 * u1, d2 = a02 * u0 + a12 * u1;
#pragma unroll
    for (int k = 0; k < 3; ++k) sv[k * PSFM_SVS] = g.R[k] * d0 + g.R[3 + k] * d1 + g.R[6 + k] * d2;
  }
  __syncthreads();
  const int cnp = sm.cap_np;
  tile_reduce_points<TILE>(sm, ti, 3, [&](int k, int l, double acc) { sm.sw[k * cnp + l] = acc; });
  __syncthreads();
  double dx2 = 0.0, xc2 = 0.0;
  if (tid < ti.np) {
    const size_t gp_ = (size_t)ti.pt0 + tid;
    const double t0 = sm.sw[tid], t1 = sm.sw[cnp + tid], t2 = sm.sw[2 * cnp + tid];
    const double h0 = sm.prow(3)[tid], h1 = sm.prow(4)[tid], h2 = sm.prow(5)[tid],
                 h3 = sm.prow(6)[tid], h4 = sm.prow(7)[tid], h5 = sm.prow(8)[tid];
    // unscaled point update: dX = -(w^ - H~ t)
    const double y0 = sm.prow(9)[tid] - (h0 * t0 + h1 * t1 + h2 * t2);
    const double y1 = sm.prow(10)[tid] - (h1 * t0 + h3 * t1 + h4 * t2);
    const double y2 = sm.prow(11)[tid] - (h2 * t0 + h4 * t1 + h5 * t2);
    sm.sw[tid] = y0; sm.sw[cnp + tid] = y1; sm.sw[2 * cnp + tid] = y2;
    const double X0 = sm.sxyz[3 * tid], X1 = sm.sxyz[3 * tid + 1], X2 = sm.sxyz[3 * tid + 2];
    const double c0 = X0 + (-y0), c1 = X1 + (-y1), c2 = X2 + (-y2);
    a.Xc[3 * gp_] = c0; a.Xc[3 * gp_ + 1] = c1; a.Xc[3 * gp_ + 2] = c2;
    const double e0 = X0 - c0, e1 = X1 - c1, e2 = X2 - c2;
    dx2 = e0 * e0 + e1 * e1 + e2 * e2;
    xc2 = c0 * c0 + c1 * c1 + c2 * c2;
  }
  __syncthreads();
  // model residual of this observation: m = J step = -(u + E y_p)
  double mm = 0.0;
  if (act) {
    const double z0 = sm.sw[lp], z1 = sm.sw[cnp + lp], z2 = sm.sw[2 * cnp + lp];
    const double y0 = g.R[0] * z0 + g.R[1] * z1 + g.R[2] * z2;
    const double y1 = g.R[3] * z0 + g.R[4] * z1 + g.R[5] * z2;
    const double y2 = g.R[6] * z0 + g.R[7] * z1 + g.R[8] * z2;
    const double m0 = -(u0 + a00 * y0 + a02 * y2);
    const double m1 = -(u1 + a00 * y1 + a12 * y2);
    mm = m0 * (r0 + 0.5 * m0) + m1 * (r1 + 0.5 * m1);
  }
  double v[3] = {mm, dx2, xc2};
  if (racc != nullptr) {       // persistent kernel: per-thread sums (shared memory, stride TILE) across its tiles, one reduction at the end
#pragma unroll
    for (int k = 0; k < 3; ++k) racc[k * TILE + tid] += v[k];
    return;
  }
  const double s = block_sum_multi<3>(v, sm.sred);
  if (tid < 3) atomicAdd(a.acc + tid, s);
}

template <int TILE, bool ROT>
__global__ void __launch_bounds__(TILE, (TILE == 256 ? 4 : 1)) k_back_substitute(const TileCtx tc, const BackArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  TileSmem<TILE> sm;
  sm.carve(smem_raw, 3, 12, tc.cap_ns, tc.cap_np);
  const TileInfo ti = tile_header(tc);
  const int tid = threadIdx.x;
  const bool act = tid < ti.n;
  const size_t M = tc.M;
  const size_t i = (size_t)ti.base + tid;
  int ls = 0, lp = 0;
  double a00 = 0, a02 = 0, a12 = 0, r0 = 0, r1 = 0;
  if (act) {
    ls = __ldg(tc.obs_lseg + i);
    lp = __ldg(tc.obs_lpt + i);
    a00 = a.L.a[i]; a02 = a.L.a[M + i]; a12 = a.L.a[2 * M + i];
    const double2 rr = reinterpret_cast<const double2*>(a.L.r)[i];
    r0 = rr.x; r1 = rr.y;
  }
  double xk[3] = {0, 0, 0};
  double inv_f = 0.0;
  if (a.intr >= 1) {
    xk[0] = __ldg(a.xs + 6 * (size_t)tc.F); xk[1] = __ldg(a.xs + 6 * (size_t)tc.F + 1); xk[2] = __ldg(a.xs + 6 * (size_t)tc.F + 2);
    inv_f = 1.0 / __ldg(a.K);
  }
  tile_fill_smem<TILE>(tc, sm, ti, a.pose16, a.xs, a.X, a.ht, a.wt, false);
  back_substitute_tile<TILE, ROT>(tc, a, sm, ti, act, ls, lp, a00, a02, a12, r0, r1, xk, inv_f);
}

// ------------------------------------------------------------------ K6: cost only

struct CostArgs {
  const double* pose;   // [F*8] q(4) t(3) pad
  const double* X;
  const double* K;
  LossP loss;
  double* acc_cost;
};

__global__ void __launch_bounds__(256) k_cost(const TileCtx tc, const CostArgs a) {
  __shared__ double sred[32];
  double cost = 0.0;
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < (size_t)tc.M; i += (size_t)gridDim.x * 256) {
    const int img = tc.obs_img[i], pt = tc.obs_pt[i], cam = tc.img_cam[img];
    const double2 xy = tc.obs_xy[i];
    const double2* pp = reinterpret_cast<const double2*>(a.pose + 8 * (size_t)img);
    const double2 qa = __ldg(pp), qb = __ldg(pp + 1), ta = __ldg(pp + 2), tb = __ldg(pp + 3);
    const double q0 = qa.x, q1 = qa.y, q2 = qb.x, q3 = qb.y;
    const double X0 = a.X[3 * (size_t)pt], X1 = a.X[3 * (size_t)pt + 1], X2 = a.X[3 * (size_t)pt + 2];
    const double p0 = (1.0 - 2.0 * (q2 * q2 + q3 * q3)) * X0 + 2.0 * (q1 * q2 - q0 * q3) * X1 + 2.0 * (q1 * q3 + q0 * q2) * X2 + ta.x;
    const double p1 = 2.0 * (q1 * q2 + q0 * q3) * X0 + (1.0 - 2.0 * (q1 * q1 + q3 * q3)) * X1 + 2.0 * (q2 * q3 - q0 * q1) * X2 + ta.y;
    const double p2 = 2.0 * (q1 * q3 - q0 * q2) * X0 + 2.0 * (q2 * q3 + q0 * q1) * X1 + (1.0 - 2.0 * (q1 * q1 + q2 * q2)) * X2 + tb.x;
    const double iz = 1.0 / p2;
    const double f = a.K[3 * cam], cx = a.K[3 * cam + 1], cy = a.K[3 * cam + 2];
    const double e0 = f * p0 * iz + cx - xy.x, e1 = f * p1 * iz + cy - xy.y;
    double rho0, rho1;
    loss_eval(a.loss, e0 * e0 + e1 * e1, rho0, rho1);
    cost += 0.5 * rho0;
  }
  const double s = block_sum(cost, sred);
  if (threadIdx.x == 0) atomicAdd(a.acc_cost, s);
}

}  // namespace ba
}  // namespace psfm
