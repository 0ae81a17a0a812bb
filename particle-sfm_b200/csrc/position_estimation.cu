// position_estimation.cu — the global position estimation of the global mapper, method "lud": image orientations and
// pair translation directions in, one camera centre per image out (DESIGN.md §4.6).
//
// Reference: GlobalMapper::EstimatePositions (sfm/global_mapper.cc:111-132) with the default method "lud":
// LeastUnsquaredDeviationPositionEstimator::EstimatePositions (global/least_unsquared_deviation_position_estimator.cc
// :92-178, use_scale_constraints = false), which solves min |A x|_1 subject to every pair scale >= 1 with Theia's
// ConstrainedL1Solver (its defaults are in position_recalled.cuh); then RegisterAllImages (:140-160) sets
// tvec = -R c.  The restatement is oracle/position_oracle.py.
//
// Unknowns x = [c (3 per view, the gauge view fixed at 0); s_k per pair].  Pair k (images 1, 2) gives three L1 rows
// c1 - c2 - s_k d_k, d_k = R2' t_k, and one inequality row s_k >= 1; ADMM works on the stacked matrix A~ = [A; G],
// b~ = [0; 1].  The scale block of A~'A~ is diagonal, D_k = |d_k|^2 + 1, so the x update is reduced to the positions:
//   S = sum_k W_k (x) (e1 - e2)(e1 - e2)',  W_k = I3 - d_k d_k' / D_k    (a 3 x 3-block graph Laplacian)
//   c = S^-1 (r_c - C D^-1 r_s),  s_k = (r_s,k + d_k'(c1 - c2)) / D_k
// S is SPD exactly when the used pairs form one connected graph, and rho is fixed, so S is built, factored and
// inverted once per call.
// Device:
//   once        k_pos_pair (d_k, D_k, the off-diagonal 3 x 3 blocks of S: pairs are unique, no sums) -> k_pos_img
//               (diagonal blocks and the first right-hand side, fixed-order CSR gather) -> dense_cholesky_launch
//               (k_chol_blocked) -> k_pos_inverse (multi-CTA: each CTA solves 8 identity columns through L and L')
//   per ADMM    k_pos_gemv (c = S^-1 r, one warp per row, fixed-order reduction) -> k_pos_admm_pair (scale
//   iteration   back-substitution, A~x, over-relaxation, z and u updates, the pair's share of the stopping test and
//               of the next right-hand side) -> k_pos_admm_img (fixed-order gather of the reduced right-hand side,
//               the position parts of A~'(z - z_old) and A~'u) -> k_pos_check (one CTA: Theia's stopping test, sets
//               the done flag)
// Iterations are queued kChunk at a time behind the done flag (kernels queued past convergence return at once); the
// host reads the control block once per chunk.  No floating-point atomics: two calls return bit-identical results.
// The explicit inverse replaces the rotation stage's one-CTA triangular solves: those read the 8 n^2 bytes of the
// factor through one SM on every iteration, the GEMV spreads the same bytes over every SM.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <numeric>
#include <vector>

#include "dense_chol.cuh"
#include "pair_inputs.h"
#include "position_recalled.cuh"
#include "psfm_common.cuh"
#include "quat.cuh"

namespace {

using namespace psfm;
using namespace psfm::quat;

constexpr int kMaxUnknowns = 8190;      // n = 3 (V - 1): the rotation stage's dense-factor bound
constexpr int kChunk = 32;              // ADMM iterations queued between two reads of the done flag
constexpr int kInvCols = 8;             // identity columns per CTA of k_pos_inverse (one warp each)

struct Ctl {
  int done, count, failed;
  double r_norm, primal_eps, s_norm, dual_eps;
};

__device__ inline double pos_of(const double* c, int v, int k) { return v == 0 ? 0.0 : c[3 * (v - 1) + k]; }

// W = I - d d' / D, entry (i, j)
__device__ inline double w_entry(const double* d, double D, int i, int j) { return (i == j ? 1.0 : 0.0) - d[i] * d[j] / D; }

// per pair: d = R2' t (GetRotatedTranslation), D = |d|^2 + 1, the off-diagonal block -W of S (lower triangle), the
// first right-hand side share (z = u = 0: r_s = 1, w = d r_s / D)
__global__ void k_pos_pair(int R, const int* __restrict__ pa, const int* __restrict__ pb, const double* __restrict__ tvec,
                           const double* __restrict__ q2, double* __restrict__ dvec, double* __restrict__ Dk,
                           double* __restrict__ rs, double* __restrict__ w, double* __restrict__ S, int lda) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= R) return;
  double d[3];
  qrotate(qinv(qnormalize(load_q(q2 + 4 * (size_t)k))), tvec + 3 * (size_t)k, d);
  const double D = d[0] * d[0] + d[1] * d[1] + d[2] * d[2] + 1.0;
#pragma unroll
  for (int i = 0; i < 3; ++i) { dvec[3 * k + i] = d[i]; w[3 * k + i] = d[i] / D; }
  Dk[k] = D;
  rs[k] = 1.0;
  const int a = pa[k], b = pb[k];
  if (a == 0 || b == 0) return;
  const int hi = max(a, b) - 1, lo = min(a, b) - 1;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) S[(size_t)(3 * hi + i) * lda + 3 * lo + j] = -w_entry(d, D, i, j);
}

// per non-gauge view: the diagonal block sum W_k (lower triangle) and the first reduced right-hand side
// sum sigma w_k (sigma = +1 at image 1, -1 at image 2), over its incident pairs in CSR order
__global__ void k_pos_img(int V, const int* __restrict__ inc_ptr, const int* __restrict__ inc, const double* __restrict__ dvec,
                          const double* __restrict__ Dk, const double* __restrict__ w, double* __restrict__ S, int lda,
                          double* __restrict__ rhs) {
  const int v = 1 + blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  double B[3][3] = {{0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}}, r[3] = {0.0, 0.0, 0.0};
  for (int e = inc_ptr[v]; e < inc_ptr[v + 1]; ++e) {
    const int k = inc[e] >> 1;
    const double sg = (inc[e] & 1) ? 1.0 : -1.0;
    const double* d = dvec + 3 * k;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      r[i] += sg * w[3 * k + i];
#pragma unroll
      for (int j = 0; j < 3; ++j) B[i][j] += w_entry(d, Dk[k], i, j);
    }
  }
  const int o = 3 * (v - 1);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    rhs[o + i] = r[i];
#pragma unroll
    for (int j = 0; j <= i; ++j) S[(size_t)(o + i) * lda + o + j] = B[i][j];
  }
}

// multi-CTA: X = S^-1 from the factor dense_cholesky_launch leaves (L in Ld / Lp).  CTA b solves the identity
// columns j0 = 8 b .. j0 + 7 through L y = e_j, L' x = y; warp r owns column j0 + r in the diagonal-block solves.
// X is [n][n], column j at X + j n.  A failed factorisation marks the run failed and done.
__global__ void __launch_bounds__(256) k_pos_inverse(int n, const double* __restrict__ Ld, const double* __restrict__ Lp,
                                                     double* __restrict__ X, const int* chol_fail, Ctl* ctl) {
  constexpr int CB = kDenseCholBlock, NR = kInvCols, NG = 256 / CB;
  __shared__ double sL[CB][CB + 1];
  __shared__ double sy[CB][NR];
  __shared__ double sacc[NG][CB][NR];
  const int tid = threadIdx.x, lane = tid & 31, wp = tid >> 5;
  if (*chol_fail) {
    if (blockIdx.x == 0 && tid == 0) { ctl->failed = 1; ctl->done = 1; }
    return;
  }
  const int j0 = blockIdx.x * NR, nr = min(NR, n - j0);
  const int np = dense_chol_panels(n), rmax = dense_chol_rmax(n);
  for (int r = 0; r < nr; ++r)
    for (int i = tid; i < n; i += blockDim.x) X[(size_t)(j0 + r) * n + i] = (i == j0 + r) ? 1.0 : 0.0;
  __syncthreads();
  // forward: L y = e_j; rows above j0 stay zero, so the sweep starts at j0's panel
  for (int p = j0 / CB; p < np; ++p) {
    const int c0 = p * CB, w = min(CB, n - c0), c1 = c0 + w;
    for (int t = tid; t < CB * CB; t += blockDim.x) sL[t / CB][t % CB] = Ld[(size_t)p * CB * CB + t];
    __syncthreads();
    if (wp < NR) {
      double y = 0.0;
      double* col = X + (size_t)(j0 + wp) * n;
      if (wp < nr && lane < w) y = col[c0 + lane];
      for (int j = 0; j < w; ++j) {
        if (lane == j) y /= sL[j][j];
        const double v = __shfl_sync(0xffffffffu, y, j);
        if (lane > j) y -= sL[lane][j] * v;
      }
      if (wp < nr && lane < w) col[c0 + lane] = y;
      sy[lane][wp] = (wp < nr && lane < w) ? y : 0.0;
    }
    __syncthreads();
    for (int i = c1 + tid; i < n; i += blockDim.x) {
      const double* l = Lp + ((size_t)p * rmax + (i - c1)) * CB;
      double s[NR];
#pragma unroll
      for (int r = 0; r < NR; ++r) s[r] = 0.0;
#pragma unroll 4
      for (int m = 0; m < CB; ++m) {
        const double lm = l[m];
#pragma unroll
        for (int r = 0; r < NR; ++r) s[r] += lm * sy[m][r];
      }
      for (int r = 0; r < nr; ++r) X[(size_t)(j0 + r) * n + i] -= s[r];
    }
    __syncthreads();
  }
  // backward: L' x = y, panel by panel from the end
  for (int p = np - 1; p >= 0; --p) {
    const int c0 = p * CB, w = min(CB, n - c0), c1 = c0 + w;
    for (int t = tid; t < CB * CB; t += blockDim.x) sL[t / CB][t % CB] = Ld[(size_t)p * CB * CB + t];
    const int c = tid % CB, g = tid / CB;
    double s[NR];
#pragma unroll
    for (int r = 0; r < NR; ++r) s[r] = 0.0;
    if (c < w)
      for (int i = c1 + g; i < n; i += NG) {
        const double l = Lp[((size_t)p * rmax + (i - c1)) * CB + c];
#pragma unroll
        for (int r = 0; r < NR; ++r) s[r] += (r < nr) ? l * X[(size_t)(j0 + r) * n + i] : 0.0;
      }
#pragma unroll
    for (int r = 0; r < NR; ++r) sacc[g][c][r] = s[r];
    __syncthreads();
    if (wp < nr) {
      double* col = X + (size_t)(j0 + wp) * n;
      double v = 0.0;
      if (lane < w) {
        double a = 0.0;
        for (int gg = 0; gg < NG; ++gg) a += sacc[gg][lane][wp];
        v = col[c0 + lane] - a;
      }
      for (int j = w - 1; j >= 0; --j) {
        if (lane == j) v /= sL[j][j];
        const double u = __shfl_sync(0xffffffffu, v, j);
        if (lane < j) v -= sL[j][lane] * u;
      }
      if (lane < w) col[c0 + lane] = v;
    }
    __syncthreads();
  }
}

// one warp per row: c_i = sum_j X[i][j] r_j (column i of the computed inverse stands for its row i: S is symmetric);
// lanes take j = lane, lane + 32, ... in order, then a fixed shuffle tree
__global__ void __launch_bounds__(256) k_pos_gemv(int n, const double* __restrict__ X, const double* __restrict__ r,
                                                  double* __restrict__ c, const int* done) {
  if (*done) return;
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= n) return;
  const double* x = X + (size_t)i * n;
  double s = 0.0;
  for (int j = lane; j < n; j += 32) s += x[j] * r[j];
  s = warp_sum(s);
  if (lane == 0) c[i] = s;
}

// per pair, one iteration of the ConstrainedL1Solver after its x update: the scale back-substitution, A~x (three L1
// rows, one inequality row), over-relaxation, shrinkage / projection, the u update; the pair's terms of the stopping
// test (|A~x - z - b~|^2, |A~x|^2, |z|^2, the scale rows of |rho A~'(z - z_old)|^2 and |rho A~'u|^2) and of the next
// right-hand side (r_s = -d'v_L + v_G and w = v_L + d r_s / D for v = b~ + z - u)
__global__ void k_pos_admm_pair(int R, const int* __restrict__ pa, const int* __restrict__ pb, const double* __restrict__ c,
                                const double* __restrict__ dvec, const double* __restrict__ Dk, double* __restrict__ rs,
                                double* __restrict__ w, double* __restrict__ z, double* __restrict__ u,
                                double* __restrict__ dz, double* __restrict__ scale, double* __restrict__ part, double rho,
                                double alpha, const int* done) {
  if (*done) return;
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= R) return;
  const int a = pa[k], b = pb[k];
  const double* d = dvec + 3 * k;
  const double D = Dk[k];
  double diff[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) diff[i] = pos_of(c, a, i) - pos_of(c, b, i);
  const double s = (rs[k] + (d[0] * diff[0] + d[1] * diff[1] + d[2] * diff[2])) / D;
  scale[k] = s;
  const double kappa = 1.0 / rho;
  double e2 = 0.0, ax2 = 0.0, z2 = 0.0, zn[4], un[4], dzs[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const double bb = i < 3 ? 0.0 : 1.0;
    const double ax = i < 3 ? diff[i] - s * d[i] : s;
    const double zo = z[4 * k + i];
    const double ahat = alpha * ax + (1.0 - alpha) * (zo + bb);
    const double v = ahat - bb + u[4 * k + i];
    const double znew = i < 3 ? fmax(0.0, v - kappa) - fmax(0.0, -v - kappa) : fmax(v, 0.0);
    un[i] = u[4 * k + i] + (ahat - znew - bb);
    zn[i] = znew;
    dzs[i] = znew - zo;
    const double e = ax - znew - bb;
    e2 += e * e; ax2 += ax * ax; z2 += znew * znew;
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) { z[4 * k + i] = zn[i]; u[4 * k + i] = un[i]; }
#pragma unroll
  for (int i = 0; i < 3; ++i) dz[3 * k + i] = dzs[i];
  const double sdz = rho * (dzs[3] - (d[0] * dzs[0] + d[1] * dzs[1] + d[2] * dzs[2]));
  const double su = rho * (un[3] - (d[0] * un[0] + d[1] * un[1] + d[2] * un[2]));
  part[5 * k] = e2; part[5 * k + 1] = ax2; part[5 * k + 2] = z2; part[5 * k + 3] = sdz * sdz; part[5 * k + 4] = su * su;
  double vl[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) vl[i] = zn[i] - un[i];
  const double r = (1.0 + zn[3] - un[3]) - (d[0] * vl[0] + d[1] * vl[1] + d[2] * vl[2]);
  rs[k] = r;
#pragma unroll
  for (int i = 0; i < 3; ++i) w[3 * k + i] = vl[i] + d[i] * r / D;
}

// per non-gauge view: the reduced right-hand side sum sigma w_k, |rho A'(z - z_old)|^2 and |rho A'u|^2 over its
// position rows, in CSR order
__global__ void k_pos_admm_img(int V, const int* __restrict__ inc_ptr, const int* __restrict__ inc, const double* __restrict__ w,
                               const double* __restrict__ dz, const double* __restrict__ u, double* __restrict__ rhs,
                               double* __restrict__ ipart, double rho, const int* done) {
  if (*done) return;
  const int v = 1 + blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  double r[3] = {0.0, 0.0, 0.0}, g[3] = {0.0, 0.0, 0.0}, h[3] = {0.0, 0.0, 0.0};
  for (int e = inc_ptr[v]; e < inc_ptr[v + 1]; ++e) {
    const int k = inc[e] >> 1;
    const double sg = (inc[e] & 1) ? 1.0 : -1.0;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      r[i] += sg * w[3 * k + i];
      g[i] += sg * dz[3 * k + i];
      h[i] += sg * u[4 * k + i];
    }
  }
  double ns = 0.0, nt = 0.0;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    rhs[3 * (v - 1) + i] = r[i];
    ns += (rho * g[i]) * (rho * g[i]);
    nt += (rho * h[i]) * (rho * h[i]);
  }
  ipart[2 * (v - 1)] = ns; ipart[2 * (v - 1) + 1] = nt;
}

// one CTA: fixed-order norms and the ConstrainedL1Solver stopping test; counts the iteration, sets the done flag
__global__ void __launch_bounds__(1024) k_pos_check(int R, int nv, const double* __restrict__ part,
                                                    const double* __restrict__ ipart, double abs_tol, double rel_tol,
                                                    Ctl* ctl) {
  __shared__ double sbuf[32];
  if (ctl->done) return;
  double s[5] = {0.0, 0.0, 0.0, 0.0, 0.0}, t[2] = {0.0, 0.0};
  for (int k = threadIdx.x; k < R; k += blockDim.x)
#pragma unroll
    for (int i = 0; i < 5; ++i) s[i] += part[5 * k + i];
  for (int v = threadIdx.x; v < nv; v += blockDim.x) { t[0] += ipart[2 * v]; t[1] += ipart[2 * v + 1]; }
  double S[5], T[2];
#pragma unroll
  for (int i = 0; i < 5; ++i) S[i] = block_sum(s[i], sbuf);
#pragma unroll
  for (int i = 0; i < 2; ++i) T[i] = block_sum(t[i], sbuf);
  if (threadIdx.x == 0) {
    ctl->count += 1;
    const double r_norm = sqrt(S[0]);
    const double max_norm = fmax(fmax(sqrt(S[1]), sqrt(S[2])), sqrt((double)R));     // |b~| = sqrt(R)
    const double primal_eps = sqrt(4.0 * R) * abs_tol + rel_tol * max_norm;
    const double s_norm = sqrt(T[0] + S[3]);
    const double dual_eps = sqrt(3.0 * nv + R) * abs_tol + rel_tol * sqrt(T[1] + S[4]);
    ctl->r_norm = r_norm; ctl->primal_eps = primal_eps; ctl->s_norm = s_norm; ctl->dual_eps = dual_eps;
    if (r_norm < primal_eps && s_norm < dual_eps) ctl->done = 1;
  }
}

// ---- host ----------------------------------------------------------------------------------------------------------
int find_root(std::vector<int>& parent, int v) {
  while (parent[v] != v) v = parent[v] = parent[parent[v]];
  return v;
}

}  // namespace

extern "C" void psfm_lud_default_options(psfm_lud_options* o) {
  if (!o) return;
  o->max_num_iterations = psfm::pos::kLudMaxIterations;
  o->rho = psfm::pos::kLudRho;
  o->alpha = psfm::pos::kLudAlpha;
  o->absolute_tolerance = psfm::pos::kLudAbsTolerance;
  o->relative_tolerance = psfm::pos::kLudRelTolerance;
}

extern "C" int psfm_estimate_global_positions(int32_t num_images, int64_t num_pairs, const int32_t* pair_images,
                                              const double* pair_tvec, const double* orientations,
                                              const uint8_t* has_orientation, const uint8_t* pair_used,
                                              const psfm_lud_options* opts, double* positions, uint8_t* has_position,
                                              double* image_tvec, double* scales, psfm_position_summary* summary) {
  const auto t0 = std::chrono::steady_clock::now();
  const long long launches0 = g_launch_count.load();
  const char* entry = "psfm_estimate_global_positions";
  psfm_position_summary sm;
  memset(&sm, 0, sizeof(sm));
  auto finish = [&](int rc) {
    sm.num_launches = g_launch_count.load() - launches0;
    if (summary) *summary = sm;
    return rc;
  };
  return guard(entry, [&]() -> int {
    int rc = check_sizes(entry, num_images, 0, num_pairs);
    if (rc != PSFM_OK) return rc;
    if ((num_pairs > 0 && (!pair_images || !pair_tvec || !scales)) ||
        (num_images > 0 && (!orientations || !positions || !has_position || !image_tvec)))
      return fail(entry, PSFM_ERR_INVALID, "null argument");
    psfm_lud_options o;
    psfm_lud_default_options(&o);
    if (opts) o = *opts;
    if (!(o.max_num_iterations > 0 && o.rho > 0.0 && o.alpha > 0.0 && o.alpha < 2.0 && o.absolute_tolerance > 0.0 &&
          o.relative_tolerance > 0.0 && std::isfinite(o.rho) && std::isfinite(o.absolute_tolerance) &&
          std::isfinite(o.relative_tolerance)))
      return fail(entry, PSFM_ERR_INVALID, "options fail the ConstrainedL1Solver options Check()");
    const int F = num_images, R = (int)num_pairs;
    if ((rc = check_pair_images(entry, R, pair_images, F)) != PSFM_OK) return rc;
    if ((rc = check_distinct_pairs(entry, R, pair_images)) != PSFM_OK) return rc;
    std::vector<int> used;
    for (int p = 0; p < R; ++p)
      if (!pair_used || pair_used[p]) used.push_back(p);
    if (used.empty()) return fail(entry, PSFM_ERR_INVALID, "no used image pair");
    // views: the images of the used pairs, ascending; the first is the gauge
    std::vector<int> vidx(F, -1), views;
    {
      std::vector<char> seen(F, 0);
      for (int p : used) seen[pair_images[2 * p]] = seen[pair_images[2 * p + 1]] = 1;
      for (int f = 0; f < F; ++f)
        if (seen[f]) { vidx[f] = (int)views.size(); views.push_back(f); }
    }
    for (int f : views) {
      if (has_orientation && !has_orientation[f]) return fail(entry, PSFM_ERR_INVALID, "a used pair's image has no orientation");
      for (int k = 0; k < 4; ++k)
        if (!std::isfinite(orientations[4 * (size_t)f + k])) return fail(entry, PSFM_ERR_INVALID, "a non-finite orientation");
    }
    for (int p : used)
      for (int k = 0; k < 3; ++k)
        if (!std::isfinite(pair_tvec[3 * (size_t)p + k])) return fail(entry, PSFM_ERR_INVALID, "a non-finite pair tvec");
    const int V = (int)views.size(), Ru = (int)used.size();
    {
      std::vector<int> parent(V);
      std::iota(parent.begin(), parent.end(), 0);
      int comps = V;
      for (int p : used) {
        const int a = find_root(parent, vidx[pair_images[2 * p]]), b = find_root(parent, vidx[pair_images[2 * p + 1]]);
        if (a != b) { parent[std::max(a, b)] = std::min(a, b); --comps; }
      }
      if (comps != 1) return fail(entry, PSFM_ERR_INVALID, "the used pairs do not form one connected graph (S is singular)");
    }
    const long long n_ll = 3LL * (V - 1);
    if (n_ll > kMaxUnknowns) return fail(entry, PSFM_ERR_UNSUPPORTED, "more than 2731 views (3 (V - 1) > 8190 unknowns)");
    const int n = (int)n_ll;
    if ((rc = require_device(entry)) != PSFM_OK) return rc;

    sm.gauge_image = views[0];
    sm.num_views = V;
    sm.num_pairs_used = Ru;
    std::vector<int> pa(Ru), pb(Ru);
    std::vector<double> tv(3 * (size_t)Ru), q2(4 * (size_t)Ru);
    for (int k = 0; k < Ru; ++k) {
      const int p = used[k];
      pa[k] = vidx[pair_images[2 * p]];
      pb[k] = vidx[pair_images[2 * p + 1]];
      for (int i = 0; i < 3; ++i) tv[3 * (size_t)k + i] = pair_tvec[3 * (size_t)p + i];
      for (int i = 0; i < 4; ++i) q2[4 * (size_t)k + i] = orientations[4 * (size_t)pair_images[2 * p + 1] + i];
    }
    // view -> incident pairs, in pair order; bit 0: the view is the pair's image 1 (+I in A), else image 2 (-I)
    std::vector<int> inc_ptr(V + 1, 0), inc(2 * (size_t)Ru);
    for (int k = 0; k < Ru; ++k) { ++inc_ptr[pa[k] + 1]; ++inc_ptr[pb[k] + 1]; }
    for (int v = 0; v < V; ++v) inc_ptr[v + 1] += inc_ptr[v];
    {
      std::vector<int> fill(inc_ptr.begin(), inc_ptr.end() - 1);
      for (int k = 0; k < Ru; ++k) { inc[fill[pa[k]]++] = 2 * k + 1; inc[fill[pb[k]]++] = 2 * k; }
    }
    std::vector<double> c(n), s(Ru);
    const auto t1 = std::chrono::steady_clock::now();
    sm.host_ms = std::chrono::duration<double, std::milli>(t1 - t0).count();
    const int lda = n + 1, np = dense_chol_panels(n), rmax = dense_chol_rmax(n);
    DBuf<int> d_pa, d_pb, d_inc_ptr, d_inc, d_fail;
    DBuf<double> d_tv, d_q2, d_d, d_D, d_rs, d_w, d_z, d_u, d_dz, d_s, d_part, d_ipart, d_rhs, d_c, d_S, d_xc, d_Lp, d_Ld,
        d_X;
    DBuf<unsigned int> d_bar;
    DBuf<Ctl> d_ctl;
    d_pa.alloc(Ru); d_pb.alloc(Ru); d_inc_ptr.alloc(V + 1); d_inc.alloc(2 * (size_t)Ru); d_fail.alloc(1);
    d_tv.alloc(3 * (size_t)Ru); d_q2.alloc(4 * (size_t)Ru); d_d.alloc(3 * (size_t)Ru); d_D.alloc(Ru); d_rs.alloc(Ru);
    d_w.alloc(3 * (size_t)Ru); d_z.alloc(4 * (size_t)Ru); d_u.alloc(4 * (size_t)Ru); d_dz.alloc(3 * (size_t)Ru);
    d_s.alloc(Ru); d_part.alloc(5 * (size_t)Ru); d_ipart.alloc(2 * (size_t)(V - 1)); d_rhs.alloc(n); d_c.alloc(n);
    d_S.alloc((size_t)lda * lda); d_xc.alloc(n); d_Lp.alloc((size_t)np * rmax * kDenseCholBlock);
    d_Ld.alloc((size_t)np * kDenseCholBlock * kDenseCholBlock); d_X.alloc((size_t)n * n); d_bar.alloc(1); d_ctl.alloc(1);
    d_pa.upload(pa.data(), Ru, nullptr); d_pb.upload(pb.data(), Ru, nullptr);
    d_inc_ptr.upload(inc_ptr.data(), V + 1, nullptr); d_inc.upload(inc.data(), 2 * (size_t)Ru, nullptr);
    d_tv.upload(tv.data(), tv.size(), nullptr); d_q2.upload(q2.data(), q2.size(), nullptr);
    d_z.zero(nullptr); d_u.zero(nullptr); d_ctl.zero(nullptr);
    PSFM_CUDA(cudaMemsetAsync(d_S.p, 0, sizeof(double) * (size_t)lda * lda, nullptr));
    Ctl* ctl = d_ctl.p;
    Event ev[4];
    PSFM_CUDA(cudaEventRecord(ev[0], nullptr));
    k_pos_pair<<<grid_of(Ru), 256>>>(Ru, d_pa.p, d_pb.p, d_tv.p, d_q2.p, d_d.p, d_D.p, d_rs.p, d_w.p, d_S.p, lda);
    PSFM_LAUNCH_CHECK();
    k_pos_img<<<grid_of(V - 1), 256>>>(V, d_inc_ptr.p, d_inc.p, d_d.p, d_D.p, d_w.p, d_S.p, lda, d_rhs.p);
    PSFM_LAUNCH_CHECK();
    PSFM_CUDA(cudaEventRecord(ev[1], nullptr));
    dense_cholesky_launch(d_S.p, n, d_xc.p, d_fail.p, d_bar.p, d_Lp.p, d_Ld.p, nullptr);
    PSFM_CUDA(cudaEventRecord(ev[2], nullptr));
    k_pos_inverse<<<(n + kInvCols - 1) / kInvCols, 256>>>(n, d_Ld.p, d_Lp.p, d_X.p, d_fail.p, ctl);
    PSFM_LAUNCH_CHECK();
    PSFM_CUDA(cudaEventRecord(ev[3], nullptr));
    PSFM_CUDA(cudaEventSynchronize(ev[3]));
    float ms[3];
    for (int i = 0; i < 3; ++i) PSFM_CUDA(cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]));
    sm.build_ms = ms[0]; sm.factor_ms = ms[1]; sm.inverse_ms = ms[2];
    // ConstrainedL1Solver::Solve
    const auto t2 = std::chrono::steady_clock::now();
    const unsigned gp = grid_of(Ru), gi = grid_of(V - 1), gg = (unsigned)((n + 7) / 8);
    Ctl h;
    for (int queued = 0; queued < o.max_num_iterations;) {
      const int chunk = std::min(kChunk, o.max_num_iterations - queued);
      for (int j = 0; j < chunk; ++j) {
        k_pos_gemv<<<gg, 256>>>(n, d_X.p, d_rhs.p, d_c.p, &ctl->done);
        PSFM_LAUNCH_CHECK();
        k_pos_admm_pair<<<gp, 256>>>(Ru, d_pa.p, d_pb.p, d_c.p, d_d.p, d_D.p, d_rs.p, d_w.p, d_z.p, d_u.p, d_dz.p, d_s.p,
                                     d_part.p, o.rho, o.alpha, &ctl->done);
        PSFM_LAUNCH_CHECK();
        k_pos_admm_img<<<gi, 256>>>(V, d_inc_ptr.p, d_inc.p, d_w.p, d_dz.p, d_u.p, d_rhs.p, d_ipart.p, o.rho, &ctl->done);
        PSFM_LAUNCH_CHECK();
        k_pos_check<<<1, 1024>>>(Ru, V - 1, d_part.p, d_ipart.p, o.absolute_tolerance, o.relative_tolerance, ctl);
        PSFM_LAUNCH_CHECK();
      }
      queued += chunk;
      sm.admm_iterations_queued = queued;
      PSFM_CUDA(cudaMemcpy(&h, ctl, sizeof(Ctl), cudaMemcpyDeviceToHost));
      if (h.failed) {
        set_error("psfm_estimate_global_positions: the factorisation of S failed (not numerically positive definite)");
        return finish(PSFM_ERR_INVALID);
      }
      if (h.done) break;
    }
    PSFM_CUDA(cudaMemcpy(c.data(), d_c.p, sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost));
    PSFM_CUDA(cudaMemcpy(s.data(), d_s.p, sizeof(double) * (size_t)Ru, cudaMemcpyDeviceToHost));
    sm.admm_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t2).count();
    sm.admm_iterations = h.count;
    sm.converged = h.done;
    sm.primal_residual = h.r_norm; sm.primal_tolerance = h.primal_eps;
    sm.dual_residual = h.s_norm; sm.dual_tolerance = h.dual_eps;
    // outputs; RegisterAllImages: tvec = -QuaternionRotatePoint(q, c)
    for (int f = 0; f < F; ++f) {
      has_position[f] = 0;
      for (int k = 0; k < 3; ++k) positions[3 * (size_t)f + k] = image_tvec[3 * (size_t)f + k] = 0.0;
    }
    for (int p = 0; p < R; ++p) scales[p] = 0.0;
    for (int k = 0; k < Ru; ++k) scales[used[k]] = s[k];
    for (int v = 0; v < V; ++v) {
      const int f = views[v];
      double* cf = positions + 3 * (size_t)f;
      for (int k = 0; k < 3; ++k) cf[k] = v == 0 ? 0.0 : c[3 * (v - 1) + k];
      double t[3];
      qrotate(load_q(orientations + 4 * (size_t)f), cf, t);
      for (int k = 0; k < 3; ++k) image_tvec[3 * (size_t)f + k] = -t[k];
      has_position[f] = 1;
    }
    return finish(PSFM_OK);
  }, finish);
}

// test entry: the stage's explicit inverse of one SPD matrix, dense_cholesky_launch then k_pos_inverse, failure through
// Ctl.failed
extern "C" int psfm_spd_inverse(const double* A, int32_t n, double* X) {
  return guard("psfm_spd_inverse", [&]() -> int {
    if (!A || !X) { set_error("psfm_spd_inverse: null argument"); return PSFM_ERR_INVALID; }
    if (n < 1 || n > kMaxUnknowns) {
      set_error("psfm_spd_inverse: needs 1 <= n <= 8190 (the stage's bound)");
      return PSFM_ERR_INVALID;
    }
    const int rc = require_device("psfm_spd_inverse");
    if (rc != PSFM_OK) return rc;
    const int lda = n + 1, np = dense_chol_panels(n), rmax = dense_chol_rmax(n);
    DBuf<double> d_S, d_xc, d_Lp, d_Ld, d_X;
    DBuf<int> d_fail;
    DBuf<unsigned int> d_bar;
    DBuf<Ctl> d_ctl;
    d_S.alloc((size_t)lda * lda); d_xc.alloc(n); d_Lp.alloc((size_t)np * rmax * kDenseCholBlock);
    d_Ld.alloc((size_t)np * kDenseCholBlock * kDenseCholBlock); d_X.alloc((size_t)n * n);
    d_fail.alloc(1); d_bar.alloc(1); d_ctl.alloc(1);
    d_S.zero(nullptr); d_ctl.zero(nullptr);
    PSFM_CUDA(cudaMemcpy2DAsync(d_S.p, sizeof(double) * lda, A, sizeof(double) * n, sizeof(double) * n, n,
                                cudaMemcpyHostToDevice, nullptr));
    dense_cholesky_launch(d_S.p, n, d_xc.p, d_fail.p, d_bar.p, d_Lp.p, d_Ld.p, nullptr);
    k_pos_inverse<<<(n + kInvCols - 1) / kInvCols, 256>>>(n, d_Ld.p, d_Lp.p, d_X.p, d_fail.p, d_ctl.p);
    PSFM_LAUNCH_CHECK();
    Ctl h;
    PSFM_CUDA(cudaMemcpy(&h, d_ctl.p, sizeof(Ctl), cudaMemcpyDeviceToHost));
    if (h.failed) { set_error("psfm_spd_inverse: matrix is not positive definite"); return PSFM_ERR_INVALID; }
    PSFM_CUDA(cudaMemcpy(X, d_X.p, sizeof(double) * (size_t)n * n, cudaMemcpyDeviceToHost));
    return PSFM_OK;
  });
}
