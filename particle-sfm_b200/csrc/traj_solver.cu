// traj_solver.cu — HP1: path-consistency trajectory optimiser on sm_90a.
//
// Drop-in target: particlesfm::optimize_location
//   (reference point_trajectory/optimize/src/trajectory_optimize.cpp:30-96): N residual
//   blocks of 6 residuals / 4 parameters (PathConsistencyError, path_consistency_cost.h:
//   42-59) over a bilinear flow lookup (BiLinearInterpolator, linear_interpolation.h:
//   97-123, ceres::Grid2D index clamping), solved as ONE Ceres problem:
//   SPARSE_NORMAL_CHOLESKY + DOGLEG, <= 200 iterations, default tolerances (:74-79).
//
// Design (DESIGN.md §4): the whole trust-region solve is ONE persistent cooperative
// kernel.  One thread owns one trajectory (grid-stride over 256-wide chunks); the 4x4
// normal blocks are factorised in registers; the handful of global scalars Ceres'
// dogleg needs per iteration (|g~|^2, |J g|^2, |gn|^2, g~.gn, model cost change,
// candidate cost, step norms, max|g|) are produced by a deterministic "canonical sum"
// (chunk tree + strided combine) followed by one grid-wide barrier, so there is no host
// round trip inside the <= 200-iteration loop.  The canonical sum has the same
// definition as oracle/traj_oracle.c and this file is compiled with -fmad=false, which
// makes the iterates bit-identical to the oracle (the tracker thresholds these doubles
// into integer track connectivity).
#include <cooperative_groups.h>

#include <chrono>
#include <mutex>

#include "traj_solver.cuh"

namespace cg = cooperative_groups;

namespace psfm {
namespace traj {

constexpr int CH = 256;          // chunk = CTA size
constexpr int MAXV = 5;          // values reduced per phase
constexpr double kMinMu = 1e-8, kMaxMu = 1.0, kMuInc = 10.0;   // DoglegStrategy
constexpr double kMinDiag = 1e-6, kMaxDiag = 1e32;             // min/max_lm_diagonal

struct Args {
  const double* uv12; const double* ref1; const double* ref2; const double* scale;
  const float* flow;
  int n, w, h, nchunks;
  psfm_traj_options o;
  double* x[2];     // [n][4] current / candidate (swapped on acceptance)
  double* r;        // [n][6]
  double* jac;      // [n][4]
  double* sc;       // [n][4]
  double* dg;       // [n][4]
  double* gt;       // [n][4]
  double* gn;       // [n][4]
  double* part;     // [2][MAXV][nchunks]
  double* out;      // [n][4]
  psfm_traj_summary* summary;
};

__device__ __forceinline__ void grid_get(const float* __restrict__ flow, int w, int h, int r, int c, double& f0, double& f1) {
  const int ri = r < 0 ? 0 : (r > h - 1 ? h - 1 : r);
  const int ci = c < 0 ? 0 : (c > w - 1 ? w - 1 : c);
  const float2 px = __ldg(reinterpret_cast<const float2*>(flow) + ((size_t)ri * w + ci));
  f0 = (double)px.x;
  f1 = (double)px.y;
}

// BiLinearInterpolator::Evaluate(r, c): value, d/dr, d/dc (2 channels)
__device__ __forceinline__ void bilinear(const float* flow, int w, int h, double r, double c, double (&f)[2],
                                         double (&dr)[2], double (&dc)[2]) {
  const int row = (int)floor(r);
  const int col = (int)floor(c);
  const double xc = c - col, xr = r - row;
  double p0[2], p1[2], f0[2], f1[2], d0[2], d1[2];
  grid_get(flow, w, h, row, col, p0[0], p0[1]);
  grid_get(flow, w, h, row, col + 1, p1[0], p1[1]);
#pragma unroll
  for (int k = 0; k < 2; ++k) { f0[k] = (1 - xc) * p0[k] + xc * p1[k]; d0[k] = p1[k] - p0[k]; }
  grid_get(flow, w, h, row + 1, col, p0[0], p0[1]);
  grid_get(flow, w, h, row + 1, col + 1, p1[0], p1[1]);
#pragma unroll
  for (int k = 0; k < 2; ++k) { f1[k] = (1 - xc) * p0[k] + xc * p1[k]; d1[k] = p1[k] - p0[k]; }
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    f[k] = (1 - xr) * f0[k] + xr * f1[k];
    dr[k] = f1[k] - f0[k];
    dc[k] = (1 - xr) * d0[k] + xr * d1[k];
  }
}

// PathConsistencyError::operator() and the four non-trivial Jacobian entries
__device__ __forceinline__ void eval_block(const Args& a, int i, const double (&x)[4], double (&r)[6], double (&j)[4]) {
  double ft[2], dr[2], dc[2];
  bilinear(a.flow, a.w, a.h, x[1], x[0], ft, dr, dc);
  const double s = a.scale[i];
  r[0] = x[0] - a.ref1[2 * (size_t)i];
  r[1] = x[1] - a.ref1[2 * (size_t)i + 1];
  r[2] = (x[2] - a.ref2[2 * (size_t)i]) * s;
  r[3] = (x[3] - a.ref2[2 * (size_t)i + 1]) * s;
  r[4] = (x[2] - x[0]) - ft[0];
  r[5] = (x[3] - x[1]) - ft[1];
  j[0] = -1.0 - dc[0];
  j[1] = 0.0 - dr[0];
  j[2] = 0.0 - dc[1];
  j[3] = -1.0 - dr[1];
}

struct SJac { double e0, e1, e2, e3, A, B, C, D, f2, f3; };
__device__ __forceinline__ SJac scaled_jac(const double (&sc)[4], const double (&j)[4], double s) {
  SJac J;
  J.e0 = sc[0]; J.e1 = sc[1]; J.e2 = s * sc[2]; J.e3 = s * sc[3];
  J.A = j[0] * sc[0]; J.B = j[1] * sc[1]; J.C = j[2] * sc[0]; J.D = j[3] * sc[1];
  J.f2 = sc[2]; J.f3 = sc[3];
  return J;
}

__device__ __forceinline__ void ld4(const double* p, size_t i, double (&v)[4]) {
  const double2* q = reinterpret_cast<const double2*>(p + 4 * i);
  const double2 a = q[0], b = q[1];
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
}
__device__ __forceinline__ void st4(double* p, size_t i, const double (&v)[4]) {
  double2* q = reinterpret_cast<double2*>(p + 4 * i);
  q[0] = make_double2(v[0], v[1]);
  q[1] = make_double2(v[2], v[3]);
}

// ---- canonical sum (same definition as oracle/traj_oracle.c: tree256 / canon_sum) ----

// chunk tree of NV per-thread values; thread k < NV returns the chunk total of value k
template <int NV>
__device__ __forceinline__ double chunk_tree(const double (&v)[NV], double* s_part /*[MAXV][8]*/) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  __syncthreads();
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    double w = v[k];
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) w = w + __shfl_xor_sync(0xffffffffu, w, off);
    if (lane == 0) s_part[k * 8 + wid] = w;
  }
  __syncthreads();
  double t = 0.0;
  if (threadIdx.x < NV) {
    t = s_part[threadIdx.x * 8];
#pragma unroll
    for (int g = 1; g < 8; ++g) t = t + s_part[threadIdx.x * 8 + g];
  }
  return t;
}

// Reduce NV sums (+ one max carried as value index NV when HAS_MAX) over the grid.
// Each CTA loops over its chunks calling `body(idx, active, vals, mx)`.
template <int NV, bool HAS_MAX, typename Body>
__device__ __forceinline__ void grid_phase(const Args& a, cg::grid_group& grid, int& phase, double* s_part,
                                           double* s_res, double (&result)[NV], double& result_max, Body body) {
  double* part = a.part + (size_t)(phase & 1) * MAXV * a.nchunks;
  for (int c = blockIdx.x; c < a.nchunks; c += gridDim.x) {
    const int idx = c * CH + threadIdx.x;
    double vals[NV];
#pragma unroll
    for (int k = 0; k < NV; ++k) vals[k] = 0.0;
    double mx = 0.0;
    body(idx, idx < a.n, vals, mx);
    const double t = chunk_tree<NV>(vals, s_part);
    if (threadIdx.x < NV) part[(size_t)threadIdx.x * a.nchunks + c] = t;
    if (HAS_MAX) {
      const double m = block_max(mx, s_res);
      if (threadIdx.x == 0) part[(size_t)NV * a.nchunks + c] = m;
    }
  }
  __threadfence();
  grid.sync();
  // strided combine + tree, identical on every CTA
  double q[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    double acc = 0.0;
    for (int j = threadIdx.x; j < a.nchunks; j += CH) acc = acc + part[(size_t)k * a.nchunks + j];
    q[k] = acc;
  }
  const double t = chunk_tree<NV>(q, s_part);
  __syncthreads();
  if (threadIdx.x < NV) s_res[threadIdx.x] = t;
  __syncthreads();
#pragma unroll
  for (int k = 0; k < NV; ++k) result[k] = s_res[k];
  __syncthreads();
  if (HAS_MAX) {
    double m = 0.0;
    for (int j = threadIdx.x; j < a.nchunks; j += CH) m = fmax(m, part[(size_t)NV * a.nchunks + j]);
    m = block_max(m, s_res);
    __syncthreads();
    if (threadIdx.x == 0) s_res[40] = m;
    __syncthreads();
    result_max = s_res[40];
    __syncthreads();
  }
  ++phase;
}

__global__ void __launch_bounds__(CH) k_traj_solve(const Args a) {
  cg::grid_group grid = cg::this_grid();
  __shared__ double s_part[MAXV * 8];
  __shared__ double s_res[64];
  const psfm_traj_options o = a.o;
  int phase = 0;
  int cur = 0;   // a.x[cur] is x, a.x[1-cur] the candidate

  // initial x
  for (int c = blockIdx.x; c < a.nchunks; c += gridDim.x) {
    const int idx = c * CH + threadIdx.x;
    if (idx < a.n) {
      double v[4];
      ld4(a.uv12, idx, v);
      st4(a.x[0], idx, v);
      const double one[4] = {1.0, 1.0, 1.0, 1.0};
      st4(a.sc, idx, one);
    }
  }

  double radius = o.initial_trust_region_radius;
  double mu = kMinMu;
  bool reuse = false;
  double dogleg_step_norm = 0.0, alpha = 0.0, gt_norm = 0.0, gn_norm = 0.0, gt_dot_gn = 0.0;
  int num_invalid = 0, iteration = 0, nsucc = 0, nunsucc = 0;
  int term = PSFM_TERM_NO_CONVERGENCE;
  double x_cost = 0.0, x_norm = 0.0, gmax = 0.0, initial_cost = 0.0;
  bool need_eval = true, step_ok_prev = true, gn_valid = false;

  for (;;) {
    if (need_eval) {
      // EvaluateGradientAndJacobian at x
      double res[2], gm;
      const bool first = (iteration == 0);
      const double* xcur = a.x[cur];
      grid_phase<2, true>(a, grid, phase, s_part, s_res, res, gm,
        [&](int i, bool act, double (&vals)[2], double& mx) {
          if (!act) return;
          double x[4], r[6], j[4];
          ld4(xcur, i, x);
          eval_block(a, i, x, r, j);
          const double s = a.scale[i];
#pragma unroll
          for (int k = 0; k < 6; ++k) a.r[6 * (size_t)i + k] = r[k];
          st4(a.jac, i, j);
          vals[0] = 0.5 * (((((r[0] * r[0] + r[1] * r[1]) + r[2] * r[2]) + r[3] * r[3]) + r[4] * r[4]) + r[5] * r[5]);
          vals[1] = ((x[0] * x[0] + x[1] * x[1]) + x[2] * x[2]) + x[3] * x[3];
          const double g0 = (r[0] + j[0] * r[4]) + j[2] * r[5];
          const double g1 = (r[1] + j[1] * r[4]) + j[3] * r[5];
          const double g2 = s * r[2] + r[4];
          const double g3 = s * r[3] + r[5];
          mx = fmax(fmax(fabs(g0), fabs(g1)), fmax(fabs(g2), fabs(g3)));
          if (first && o.jacobi_scaling) {
            double sc[4];
            sc[0] = 1.0 / (1.0 + sqrt((1.0 + j[0] * j[0]) + j[2] * j[2]));
            sc[1] = 1.0 / (1.0 + sqrt((1.0 + j[1] * j[1]) + j[3] * j[3]));
            sc[2] = 1.0 / (1.0 + sqrt(s * s + 1.0));
            sc[3] = 1.0 / (1.0 + sqrt(s * s + 1.0));
            st4(a.sc, i, sc);
          }
        });
      x_cost = res[0];
      x_norm = sqrt(res[1]);
      gmax = gm;
      if (first) initial_cost = x_cost;
      need_eval = false;
      reuse = false;
    }
    // FinalizeIterationAndCheckIfMinimizerCanContinue
    if (step_ok_prev && iteration > 0) ++nsucc;
    if (iteration >= o.max_num_iterations) { term = PSFM_TERM_NO_CONVERGENCE; break; }
    if (gmax <= o.gradient_tolerance) { term = PSFM_TERM_CONVERGENCE_GRADIENT; break; }
    if (radius <= o.min_trust_region_radius) { term = PSFM_TERM_MIN_RADIUS; break; }
    ++iteration;
    step_ok_prev = false;

    // ---- DoglegStrategy::ComputeStep ----
    bool ls_failed = false;
    if (!reuse) {
      reuse = true;
      double res[2], dummy;
      grid_phase<2, false>(a, grid, phase, s_part, s_res, res, dummy,
        [&](int i, bool act, double (&vals)[2], double&) {
          if (!act) return;
          double sc[4], j[4], r[6];
          ld4(a.sc, i, sc);
          ld4(a.jac, i, j);
#pragma unroll
          for (int k = 0; k < 6; ++k) r[k] = a.r[6 * (size_t)i + k];
          const SJac J = scaled_jac(sc, j, a.scale[i]);
          const double h00 = (J.e0 * J.e0 + J.A * J.A) + J.C * J.C;
          const double h11 = (J.e1 * J.e1 + J.B * J.B) + J.D * J.D;
          const double h22 = J.e2 * J.e2 + J.f2 * J.f2;
          const double h33 = J.e3 * J.e3 + J.f3 * J.f3;
          double dg[4], gt[4];
          dg[0] = sqrt(fmin(fmax(h00, kMinDiag), kMaxDiag));
          dg[1] = sqrt(fmin(fmax(h11, kMinDiag), kMaxDiag));
          dg[2] = sqrt(fmin(fmax(h22, kMinDiag), kMaxDiag));
          dg[3] = sqrt(fmin(fmax(h33, kMinDiag), kMaxDiag));
          const double gs0 = (J.e0 * r[0] + J.A * r[4]) + J.C * r[5];
          const double gs1 = (J.e1 * r[1] + J.B * r[4]) + J.D * r[5];
          const double gs2 = J.e2 * r[2] + J.f2 * r[4];
          const double gs3 = J.e3 * r[3] + J.f3 * r[5];
          gt[0] = gs0 / dg[0]; gt[1] = gs1 / dg[1]; gt[2] = gs2 / dg[2]; gt[3] = gs3 / dg[3];
          st4(a.dg, i, dg);
          st4(a.gt, i, gt);
          vals[0] = ((gt[0] * gt[0] + gt[1] * gt[1]) + gt[2] * gt[2]) + gt[3] * gt[3];
          const double v0 = gt[0] / dg[0], v1 = gt[1] / dg[1], v2 = gt[2] / dg[2], v3 = gt[3] / dg[3];
          const double m0 = J.e0 * v0, m1 = J.e1 * v1, m2 = J.e2 * v2, m3 = J.e3 * v3;
          const double m4 = (J.A * v0 + J.B * v1) + J.f2 * v2;
          const double m5 = (J.C * v0 + J.D * v1) + J.f3 * v3;
          vals[1] = ((((m0 * m0 + m1 * m1) + m2 * m2) + m3 * m3) + m4 * m4) + m5 * m5;
        });
      gt_norm = sqrt(res[0]);
      alpha = res[0] / res[1];
      // ComputeGaussNewtonStep
      ls_failed = true;
      gn_valid = false;
      while (mu < kMaxMu) {
        const double sqmu = sqrt(mu);
        double res2[2], fail;
        grid_phase<2, true>(a, grid, phase, s_part, s_res, res2, fail,
          [&](int i, bool act, double (&vals)[2], double& mx) {
            if (!act) return;
            double sc[4], j[4], r[6], dg[4], gt[4], gn[4];
            ld4(a.sc, i, sc);
            ld4(a.jac, i, j);
            ld4(a.dg, i, dg);
            ld4(a.gt, i, gt);
#pragma unroll
            for (int k = 0; k < 6; ++k) r[k] = a.r[6 * (size_t)i + k];
            const SJac J = scaled_jac(sc, j, a.scale[i]);
            const double l0 = dg[0] * sqmu, l1 = dg[1] * sqmu, l2 = dg[2] * sqmu, l3 = dg[3] * sqmu;
            const double h00 = ((J.e0 * J.e0 + J.A * J.A) + J.C * J.C) + l0 * l0;
            const double h01 = J.A * J.B + J.C * J.D;
            const double h02 = J.A * J.f2;
            const double h03 = J.C * J.f3;
            const double h11 = ((J.e1 * J.e1 + J.B * J.B) + J.D * J.D) + l1 * l1;
            const double h12 = J.B * J.f2;
            const double h13 = J.D * J.f3;
            const double h22 = (J.e2 * J.e2 + J.f2 * J.f2) + l2 * l2;
            const double h33 = (J.e3 * J.e3 + J.f3 * J.f3) + l3 * l3;
            const double b0 = (J.e0 * r[0] + J.A * r[4]) + J.C * r[5];
            const double b1 = (J.e1 * r[1] + J.B * r[4]) + J.D * r[5];
            const double b2 = J.e2 * r[2] + J.f2 * r[4];
            const double b3 = J.e3 * r[3] + J.f3 * r[5];
            bool bad = false;
            double d;
            if (!(h00 > 0.0)) bad = true;
            const double L00 = sqrt(h00);
            const double L10 = h01 / L00, L20 = h02 / L00, L30 = h03 / L00;
            d = h11 - L10 * L10; if (!(d > 0.0)) bad = true;
            const double L11 = sqrt(d);
            const double L21 = (h12 - L20 * L10) / L11;
            const double L31 = (h13 - L30 * L10) / L11;
            d = (h22 - L20 * L20) - L21 * L21; if (!(d > 0.0)) bad = true;
            const double L22 = sqrt(d);
            const double L32 = ((0.0 - L30 * L20) - L31 * L21) / L22;
            d = ((h33 - L30 * L30) - L31 * L31) - L32 * L32; if (!(d > 0.0)) bad = true;
            const double L33 = sqrt(d);
            const double y0 = b0 / L00;
            const double y1 = (b1 - L10 * y0) / L11;
            const double y2 = ((b2 - L20 * y0) - L21 * y1) / L22;
            const double y3 = (((b3 - L30 * y0) - L31 * y1) - L32 * y2) / L33;
            const double z3 = y3 / L33;
            const double z2 = (y2 - L32 * z3) / L22;
            const double z1 = ((y1 - L21 * z2) - L31 * z3) / L11;
            const double z0 = (((y0 - L10 * z1) - L20 * z2) - L30 * z3) / L00;
            if (!isfinite(z0) || !isfinite(z1) || !isfinite(z2) || !isfinite(z3)) bad = true;
            gn[0] = z0 * (-dg[0]); gn[1] = z1 * (-dg[1]); gn[2] = z2 * (-dg[2]); gn[3] = z3 * (-dg[3]);
            st4(a.gn, i, gn);
            vals[0] = ((gn[0] * gn[0] + gn[1] * gn[1]) + gn[2] * gn[2]) + gn[3] * gn[3];
            vals[1] = ((gt[0] * gn[0] + gt[1] * gn[1]) + gt[2] * gn[2]) + gt[3] * gn[3];
            mx = bad ? 1.0 : 0.0;
          });
        if (fail > 0.0) { mu *= kMuInc; continue; }
        gn_norm = sqrt(res2[0]);
        gt_dot_gn = res2[1];
        ls_failed = false;
        gn_valid = true;
        break;
      }
    }
    double mcc = 0.0, cand_cost = 0.0, step_sq = 0.0;
    bool valid = false;
    if (!ls_failed && gn_valid) {
      // ComputeTraditionalDoglegStep + candidate + model cost change
      int kase;
      double beta = 0.0, cauchy_scale = 0.0;
      if (gn_norm <= radius) kase = 1;
      else if (gt_norm * alpha >= radius) { kase = 2; cauchy_scale = -(radius / gt_norm); }
      else {
        kase = 3;
        const double b_dot_a = -alpha * gt_dot_gn;
        const double an = alpha * gt_norm;
        const double a_sq = an * an;
        const double bma_sq = (a_sq - 2 * b_dot_a) + gn_norm * gn_norm;
        const double cc = b_dot_a - a_sq;
        const double dd = sqrt(cc * cc + bma_sq * (radius * radius - a_sq));
        beta = (cc <= 0) ? (dd - cc) / bma_sq : (radius * radius - a_sq) / (dd + cc);
        cauchy_scale = -alpha * (1.0 - beta);
      }
      double res4[4], dummy;
      const double* xcur = a.x[cur];
      double* xcand = a.x[1 - cur];
      grid_phase<4, false>(a, grid, phase, s_part, s_res, res4, dummy,
        [&](int i, bool act, double (&vals)[4], double&) {
          if (!act) return;
          double sc[4], j[4], r[6], dg[4], gt[4], gn[4], x[4], xc[4];
          ld4(a.sc, i, sc);
          ld4(a.jac, i, j);
          ld4(a.dg, i, dg);
          ld4(a.gt, i, gt);
          ld4(a.gn, i, gn);
          ld4(xcur, i, x);
#pragma unroll
          for (int k = 0; k < 6; ++k) r[k] = a.r[6 * (size_t)i + k];
          const SJac J = scaled_jac(sc, j, a.scale[i]);
          double s0, s1, s2, s3;
          if (kase == 1) { s0 = gn[0]; s1 = gn[1]; s2 = gn[2]; s3 = gn[3]; }
          else if (kase == 2) { s0 = cauchy_scale * gt[0]; s1 = cauchy_scale * gt[1]; s2 = cauchy_scale * gt[2]; s3 = cauchy_scale * gt[3]; }
          else {
            s0 = cauchy_scale * gt[0] + beta * gn[0]; s1 = cauchy_scale * gt[1] + beta * gn[1];
            s2 = cauchy_scale * gt[2] + beta * gn[2]; s3 = cauchy_scale * gt[3] + beta * gn[3];
          }
          vals[3] = ((s0 * s0 + s1 * s1) + s2 * s2) + s3 * s3;
          const double p0 = s0 / dg[0], p1 = s1 / dg[1], p2 = s2 / dg[2], p3 = s3 / dg[3];
          const double m0 = J.e0 * p0, m1 = J.e1 * p1, m2 = J.e2 * p2, m3 = J.e3 * p3;
          const double m4 = (J.A * p0 + J.B * p1) + J.f2 * p2;
          const double m5 = (J.C * p0 + J.D * p1) + J.f3 * p3;
          vals[0] = ((((m0 * (r[0] + m0 / 2.0) + m1 * (r[1] + m1 / 2.0)) + m2 * (r[2] + m2 / 2.0)) +
                      m3 * (r[3] + m3 / 2.0)) + m4 * (r[4] + m4 / 2.0)) + m5 * (r[5] + m5 / 2.0);
          xc[0] = x[0] + p0 * sc[0]; xc[1] = x[1] + p1 * sc[1];
          xc[2] = x[2] + p2 * sc[2]; xc[3] = x[3] + p3 * sc[3];
          st4(xcand, i, xc);
          double rc[6], jc[4];
          eval_block(a, i, xc, rc, jc);
          vals[1] = 0.5 * (((((rc[0] * rc[0] + rc[1] * rc[1]) + rc[2] * rc[2]) + rc[3] * rc[3]) + rc[4] * rc[4]) + rc[5] * rc[5]);
          const double e0 = x[0] - xc[0], e1 = x[1] - xc[1], e2 = x[2] - xc[2], e3 = x[3] - xc[3];
          vals[2] = ((e0 * e0 + e1 * e1) + e2 * e2) + e3 * e3;
        });
      mcc = -res4[0];
      cand_cost = res4[1];
      step_sq = res4[2];
      if (kase == 1) dogleg_step_norm = gn_norm;
      else if (kase == 2) dogleg_step_norm = radius;
      else dogleg_step_norm = sqrt(res4[3]);
      valid = mcc > 0.0;
    }
    if (!valid) {
      // HandleInvalidStep -> DoglegStrategy::StepIsInvalid
      ++nunsucc;
      if (++num_invalid >= o.max_num_consecutive_invalid_steps) { term = PSFM_TERM_FAILURE; break; }
      mu *= kMuInc;
      reuse = false;
      continue;
    }
    num_invalid = 0;
    const double step_norm = sqrt(step_sq);
    if (step_norm <= o.parameter_tolerance * (x_norm + o.parameter_tolerance)) { term = PSFM_TERM_CONVERGENCE_PARAMETER; break; }
    const double cost_change = x_cost - cand_cost;
    if (fabs(cost_change) <= o.function_tolerance * x_cost) { term = PSFM_TERM_CONVERGENCE_FUNCTION; break; }
    const double rho = cost_change / mcc;
    if (rho > o.min_relative_decrease) {
      cur = 1 - cur;
      need_eval = true;
      step_ok_prev = true;
      // DoglegStrategy::StepAccepted
      if (rho < 0.25) radius *= 0.5;
      if (rho > 0.75) radius = fmax(radius, 3.0 * dogleg_step_norm);
      mu = fmax(kMinMu, 2.0 * mu / kMuInc);
      reuse = false;
    } else {
      ++nunsucc;
      radius *= 0.5;
      reuse = true;
    }
  }
  // result
  const double* xfin = a.x[cur];
  for (int c = blockIdx.x; c < a.nchunks; c += gridDim.x) {
    const int idx = c * CH + threadIdx.x;
    if (idx < a.n) {
      double v[4];
      ld4(xfin, idx, v);
      st4(a.out, idx, v);
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    a.summary->num_iterations = iteration;
    a.summary->num_successful_steps = nsucc;
    a.summary->num_unsuccessful_steps = nunsucc;
    a.summary->termination = term;
    a.summary->initial_cost = initial_cost;
    a.summary->final_cost = x_cost;
  }
}

// ---------------------------------------------------------------- host

struct Workspace {
  std::mutex mu;
  DBuf<double> x0, x1, r, jac, sc, dg, gt, gn, part, in_uv, in_ref1, in_ref2, in_scale, out;
  DBuf<float> flow;
  DBuf<psfm_traj_summary> summary;
  size_t cap_n = 0, cap_flow = 0, cap_chunks = 0;
  int grid_limit = 0;
  int grid_limit_dev = -1;      // the device grid_limit was computed for (psfm_set_device may change it)
  cudaStream_t stream = nullptr;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  void ensure(size_t n, size_t nchunks) {
    if (!stream) {
      PSFM_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
      PSFM_CUDA(cudaEventCreate(&e0));
      PSFM_CUDA(cudaEventCreate(&e1));
      summary.alloc(1);
    }
    if (n > cap_n) {
      const size_t m = n + n / 4 + 1024;
      x0.alloc(4 * m); x1.alloc(4 * m); r.alloc(6 * m); jac.alloc(4 * m); sc.alloc(4 * m); dg.alloc(4 * m);
      gt.alloc(4 * m); gn.alloc(4 * m);
      in_uv.alloc(4 * m); in_ref1.alloc(2 * m); in_ref2.alloc(2 * m); in_scale.alloc(m); out.alloc(4 * m);
      cap_n = m;
    }
    if (nchunks > cap_chunks) {
      const size_t m = nchunks + nchunks / 4 + 64;
      part.alloc(2 * (size_t)MAXV * m);
      cap_chunks = m;
    }
  }
};

static Workspace g_ws;

static int launch_solve(Workspace& ws, const double* d_uv12, const double* d_ref1, const double* d_ref2,
                        const double* d_scale, const float* d_flow, int n, int w, int h,
                        const psfm_traj_options* opts, double* d_out, psfm_traj_summary* summary, cudaStream_t stream) {
  Args a;
  a.uv12 = d_uv12; a.ref1 = d_ref1; a.ref2 = d_ref2; a.scale = d_scale; a.flow = d_flow;
  a.n = n; a.w = w; a.h = h; a.nchunks = (n + CH - 1) / CH;
  if (opts) a.o = *opts; else psfm_traj_default_options(&a.o);
  a.x[0] = ws.x0.p; a.x[1] = ws.x1.p; a.r = ws.r.p; a.jac = ws.jac.p; a.sc = ws.sc.p; a.dg = ws.dg.p;
  a.gt = ws.gt.p; a.gn = ws.gn.p; a.part = ws.part.p; a.out = d_out; a.summary = ws.summary.p;
  int cur_dev = 0;
  PSFM_CUDA(cudaGetDevice(&cur_dev));
  if (ws.grid_limit == 0 || ws.grid_limit_dev != cur_dev) {
    int dev = cur_dev, sms = 0, per_sm = 0, coop = 0;
    PSFM_CUDA(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
    if (!coop) { set_error("device does not support cooperative launch"); return PSFM_ERR_UNSUPPORTED; }
    PSFM_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    PSFM_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_traj_solve, CH, 0));
    ws.grid_limit = std::max(1, sms * per_sm);
    ws.grid_limit_dev = dev;
  }
  const int grid = std::min(a.nchunks, ws.grid_limit);
  void* kargs[] = {(void*)&a};
  PSFM_CUDA(cudaEventRecord(ws.e0, stream));
  PSFM_CUDA(cudaLaunchCooperativeKernel((void*)k_traj_solve, dim3(grid), dim3(CH), kargs, 0, stream));
  PSFM_LAUNCH_CHECK();
  PSFM_CUDA(cudaEventRecord(ws.e1, stream));
  psfm_traj_summary s;
  PSFM_CUDA(cudaMemcpyAsync(&s, ws.summary.p, sizeof(s), cudaMemcpyDeviceToHost, stream));
  PSFM_CUDA(cudaStreamSynchronize(stream));
  float ms = 0.f;
  PSFM_CUDA(cudaEventElapsedTime(&ms, ws.e0, ws.e1));
  s.solve_ms = ms;
  s.total_ms = ms;
  if (summary) *summary = s;
  return PSFM_OK;
}

int solve_device(const double* d_uv12, const double* d_ref1, const double* d_ref2, const double* d_scale,
                 const float* d_flow12, int n, int w, int h, const psfm_traj_options* opts, double* d_out,
                 psfm_traj_summary* summary, cudaStream_t stream) {
  std::lock_guard<std::mutex> lock(g_ws.mu);
  g_ws.ensure((size_t)n, (size_t)(n + CH - 1) / CH);
  return launch_solve(g_ws, d_uv12, d_ref1, d_ref2, d_scale, d_flow12, n, w, h, opts, d_out, summary,
                      stream ? stream : g_ws.stream);
}

}  // namespace traj
}  // namespace psfm

using namespace psfm;

extern "C" void psfm_traj_default_options(psfm_traj_options* o) {
  o->max_num_iterations = 200;             // trajectory_optimize.cpp:76
  o->function_tolerance = 1e-6;            // Ceres 2.0.0 defaults
  o->gradient_tolerance = 1e-10;
  o->parameter_tolerance = 1e-8;
  o->initial_trust_region_radius = 1e4;
  o->max_trust_region_radius = 1e16;
  o->min_trust_region_radius = 1e-32;
  o->min_relative_decrease = 1e-3;
  o->max_num_consecutive_invalid_steps = 5;
  o->jacobi_scaling = 1;
}

extern "C" int psfm_traj_optimize_device(const double* d_uv12, const double* d_ref1, const double* d_ref2,
                                         const double* d_scale, const float* d_flow12, int32_t n, int32_t w,
                                         int32_t h, const psfm_traj_options* opts, double* d_out_uv12,
                                         psfm_traj_summary* summary, void* stream) {
  return guard("psfm_traj_optimize_device", [&]() -> int {
    if (summary) memset(summary, 0, sizeof(*summary));
    if (n < 0 || w <= 0 || h <= 0) { set_error("psfm_traj_optimize: bad sizes"); return PSFM_ERR_INVALID; }
    if (n == 0) return PSFM_OK;
    int rc = require_device("psfm_traj_optimize_device");
    if (rc != PSFM_OK) return rc;
    return traj::solve_device(d_uv12, d_ref1, d_ref2, d_scale, d_flow12, n, w, h, opts, d_out_uv12, summary,
                              (cudaStream_t)stream);
  });
}

extern "C" int psfm_traj_optimize(const double* uv12, const double* ref1, const double* ref2, const double* scale,
                                  const float* flow12, int32_t n, int32_t w, int32_t h,
                                  const psfm_traj_options* opts, double* out_uv12, psfm_traj_summary* summary) {
  return guard("psfm_traj_optimize", [&]() -> int {
    if (summary) memset(summary, 0, sizeof(*summary));
    if (n < 0 || w <= 0 || h <= 0) { set_error("psfm_traj_optimize: bad sizes"); return PSFM_ERR_INVALID; }
    if (n == 0) return PSFM_OK;
    int rc = require_device("psfm_traj_optimize");
    if (rc != PSFM_OK) return rc;
    traj::Workspace& ws = traj::g_ws;
    std::lock_guard<std::mutex> lock(ws.mu);
    const auto t0 = std::chrono::steady_clock::now();
    ws.ensure((size_t)n, (size_t)(n + traj::CH - 1) / traj::CH);
    const size_t nf = 2 * (size_t)w * h;
    if (nf > ws.cap_flow) { ws.flow.alloc(nf); ws.cap_flow = nf; }
    cudaStream_t st = ws.stream;
    ws.in_uv.upload(uv12, 4 * (size_t)n, st);
    ws.in_ref1.upload(ref1, 2 * (size_t)n, st);
    ws.in_ref2.upload(ref2, 2 * (size_t)n, st);
    ws.in_scale.upload(scale, (size_t)n, st);
    ws.flow.upload(flow12, nf, st);
    rc = traj::launch_solve(ws, ws.in_uv.p, ws.in_ref1.p, ws.in_ref2.p, ws.in_scale.p, ws.flow.p, n, w, h, opts,
                            ws.out.p, summary, st);
    if (rc != PSFM_OK) return rc;
    PSFM_CUDA(cudaMemcpyAsync(out_uv12, ws.out.p, sizeof(double) * 4 * (size_t)n, cudaMemcpyDeviceToHost, st));
    PSFM_CUDA(cudaStreamSynchronize(st));
    if (summary)
      summary->total_ms = 1e3 * std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    return PSFM_OK;
  });
}
