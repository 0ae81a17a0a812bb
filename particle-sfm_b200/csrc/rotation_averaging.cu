// rotation_averaging.cu — the global rotation averaging of the global mapper: pair relative rotations in, one
// orientation per image out (SURVEY.md §8(f), DESIGN.md §4.5).
//
// Reference: EstimateGlobalRotations (global/robust_rotation_estimator.cc:310-331).  The restatement is
// oracle/rotation_oracle.py; the constants recalled from Theia's L1Solver are in rotation_recalled.cuh.
//
// The reference solves with A, the 3R x 3(F-1) matrix of +-I blocks (pair p: -I at image 1, +I at image 2, the gauge
// image's column removed).  Every pair's three rows carry one weight, so A'WA = (B'WB) (x) I3 with B the signed
// pair-image incidence matrix: one (F-1) x (F-1) graph Laplacian factor serves the three components.
// Host (O(R log R) integer work, F quaternion products): validation, the pose filter, components by union-find,
// Kruskal, chaining along the tree from the gauge image, an image -> incident-pair CSR in pair order.
// Device, per L1 round (one host read per round):
//   once      k_lap_pair + k_lap_img (unweighted Laplacian) -> dense_cholesky_launch (k_chol_blocked), kept for
//             every ADMM iteration of every round
//   per ADMM  k_trsv (one CTA: L, L' solves, 3 right-hand sides) -> k_admm_pair (A x, over-relaxation, shrinkage,
//   iteration the u update) -> k_admm_img (A'(b + z - u) for the next iteration, A'(z - z_old), A'u) ->
//             k_admm_check (one CTA: fixed-order norms, Theia's stopping test, sets the round's done flag)
//   end       k_update (one CTA: R <- R q(x), mean step norm) -> k_residual
// IRLS, per iteration (a host read every kIrlsChunk iterations): k_lap_pair (weight sigma / (e^2 + sigma^2)^2,
// off-diagonal entries, w r) -> k_lap_img (diagonal, A'W r) -> k_chol_blocked -> k_trsv -> k_update -> k_residual.
// Iterations queued past convergence see the done flag and return at once (k_chol_blocked stops at the zeroed
// matrix's first pivot).  Then k_filter (FilterViewPairsFromOrientation); the second pruning runs on the host.
// Every sum has a fixed order (CSR gathers, one-CTA reductions, no floating-point atomics): results are
// bit-identical run to run.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <numeric>
#include <vector>

#include "dense_chol.cuh"
#include "psfm_common.cuh"
#include "rotation_recalled.cuh"

namespace {

using namespace psfm;
using namespace psfm::rot;

constexpr int kMaxComponentImages = 8192;   // dense factor + its panels: 2 x 8191^2 doubles, about 1.1 GB
constexpr int kIrlsChunk = 8;               // IRLS iterations queued between two reads of the done flag
constexpr double kDegToRad = 0.017453292519943295;   // COLMAP DegToRad

struct Ctl {
  int admm_done, admm_count, irls_done, irls_count, failed;
  double avg_step;
};

// ---- COLMAP / Ceres quaternion helpers (w, x, y, z) --------------------------------------------------------------
struct Quat {
  double w, x, y, z;
};

__host__ __device__ inline Quat qmul(const Quat& a, const Quat& b) {     // a (x) b, Eigen's Hamilton product
  return {a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
          a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x, a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w};
}
__host__ __device__ inline Quat qnormalize(const Quat& q) {               // NormalizeQuaternion
  const double n = sqrt(q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z);
  if (n == 0.0) return {1.0, 0.0, 0.0, 0.0};
  return {q.w / n, q.x / n, q.y / n, q.z / n};
}
__host__ __device__ inline Quat qconcat(const Quat& q1, const Quat& q2) {   // ConcatenateQuaternions: q2 (x) q1
  return qnormalize(qmul(qnormalize(q2), qnormalize(q1)));
}
__host__ __device__ inline Quat qinv(const Quat& q) { return {q.w, -q.x, -q.y, -q.z}; }   // InvertQuaternion
__host__ __device__ inline Quat aa_to_quat(double a0, double a1, double a2) {          // ceres::AngleAxisToQuaternion
  const double t2 = a0 * a0 + a1 * a1 + a2 * a2;
  if (t2 > 0.0) {
    const double t = sqrt(t2), h = 0.5 * t, k = sin(h) / t;
    return {cos(h), a0 * k, a1 * k, a2 * k};
  }
  return {1.0, 0.5 * a0, 0.5 * a1, 0.5 * a2};
}
__host__ __device__ inline void quat_to_aa(const Quat& q, double* a) {                 // ceres::QuaternionToAngleAxis
  const double s2 = q.x * q.x + q.y * q.y + q.z * q.z;
  double k = 2.0;
  if (s2 > 0.0) {
    const double s = sqrt(s2), c = q.w;
    const double two_theta = 2.0 * (c < 0.0 ? atan2(-s, -c) : atan2(s, c));
    k = two_theta / s;
  }
  a[0] = q.x * k; a[1] = q.y * k; a[2] = q.z * k;
}
__device__ inline Quat load_q(const double* q) { return {q[0], q[1], q[2], q[3]}; }

// QuaternionToRotationMatrix (normalised, Eigen's toRotationMatrix) and RotationMatrixToQuaternion (Eigen's
// Quaterniond(Matrix3d)): the chaining along the spanning tree (ComputeOrientation) works on matrices
void quat_to_matrix(const Quat& q0, double R[3][3]) {
  const Quat q = qnormalize(q0);
  const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
  const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w, txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
  const double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
  R[0][0] = 1 - (tyy + tzz); R[0][1] = txy - twz; R[0][2] = txz + twy;
  R[1][0] = txy + twz; R[1][1] = 1 - (txx + tzz); R[1][2] = tyz - twx;
  R[2][0] = txz - twy; R[2][1] = tyz + twx; R[2][2] = 1 - (txx + tyy);
}
Quat matrix_to_quat(const double R[3][3]) {
  const double tr = R[0][0] + R[1][1] + R[2][2];
  double q[4];
  if (tr > 0) {
    double s = std::sqrt(tr + 1.0);
    q[0] = 0.5 * s;
    s = 0.5 / s;
    q[1] = (R[2][1] - R[1][2]) * s; q[2] = (R[0][2] - R[2][0]) * s; q[3] = (R[1][0] - R[0][1]) * s;
  } else {
    int i = 0;
    if (R[1][1] > R[0][0]) i = 1;
    if (R[2][2] > R[i][i]) i = 2;
    const int j = (i + 1) % 3, k = (i + 2) % 3;
    double s = std::sqrt(R[i][i] - R[j][j] - R[k][k] + 1.0);
    q[1 + i] = 0.5 * s;
    s = 0.5 / s;
    q[0] = (R[k][j] - R[j][k]) * s; q[1 + j] = (R[j][i] + R[i][j]) * s; q[1 + k] = (R[k][i] + R[i][k]) * s;
  }
  return {q[0], q[1], q[2], q[3]};
}

// ---- kernels (images by compact index c, c = 0 the gauge; unknown c - 1 for c >= 1) -------------------------------

// per pair: weight (1, or the IRLS weight of its residual), w r, and its off-diagonal Laplacian entry
__global__ void k_lap_pair(int R, const int* __restrict__ pa, const int* __restrict__ pb, const double* __restrict__ res,
                           double sigma, int weighted, double* __restrict__ A, int lda, double* __restrict__ w,
                           double* __restrict__ wr, const int* skip) {
  if (skip && *skip) return;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= R) return;
  double wt = 1.0;
  if (weighted) {
    const double e2 = res[3 * p] * res[3 * p] + res[3 * p + 1] * res[3 * p + 1] + res[3 * p + 2] * res[3 * p + 2];
    const double t = e2 + sigma * sigma;
    wt = sigma / (t * t);
  }
  w[p] = wt;
#pragma unroll
  for (int k = 0; k < 3; ++k) wr[3 * p + k] = wt * res[3 * p + k];
  const int a = pa[p] - 1, b = pb[p] - 1;
  if (a >= 0 && b >= 0) A[(size_t)max(a, b) * lda + min(a, b)] = -wt;
}

// per non-gauge image: the Laplacian diagonal and A'W r, over its incident pairs in CSR order
__global__ void k_lap_img(int nc, const int* __restrict__ inc_ptr, const int* __restrict__ inc, const double* __restrict__ w,
                          const double* __restrict__ wr, double* __restrict__ A, int lda, double* __restrict__ rhs,
                          const int* skip) {
  if (skip && *skip) return;
  const int c = 1 + blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= nc) return;
  double d = 0.0, g0 = 0.0, g1 = 0.0, g2 = 0.0;
  for (int e = inc_ptr[c]; e < inc_ptr[c + 1]; ++e) {
    const int p = inc[e] >> 1;
    const double s = (inc[e] & 1) ? 1.0 : -1.0;
    d += w[p];
    g0 += s * wr[3 * p]; g1 += s * wr[3 * p + 1]; g2 += s * wr[3 * p + 2];
  }
  A[(size_t)(c - 1) * lda + (c - 1)] = d;
  rhs[3 * (c - 1)] = g0; rhs[3 * (c - 1) + 1] = g1; rhs[3 * (c - 1) + 2] = g2;
}

// one CTA: x = (L L')^-1 b for three interleaved right-hand sides ([n][3]), L as dense_cholesky_launch leaves it.
// A failed factorisation marks the run failed and stops both loops.
__global__ void __launch_bounds__(1024) k_trsv(int n, const double* __restrict__ Ld, const double* __restrict__ Lp,
                                               const double* __restrict__ b, double* __restrict__ x, const int* chol_fail,
                                               Ctl* ctl, const int* skip) {
  constexpr int CB = kDenseCholBlock;
  __shared__ double sL[CB][CB + 1];
  __shared__ double sy[CB][3];
  __shared__ double sacc[CB][CB][3];
  if (*skip) return;
  const int tid = threadIdx.x, lane = tid & 31;
  if (*chol_fail) {
    if (tid == 0) { ctl->failed = 1; ctl->admm_done = 1; ctl->irls_done = 1; }
    return;
  }
  const int np = dense_chol_panels(n), rmax = dense_chol_rmax(n);
  for (int i = tid; i < 3 * n; i += blockDim.x) x[i] = b[i];
  __syncthreads();
  // forward: L y = b, panel by panel
  for (int p = 0; p < np; ++p) {
    const int c0 = p * CB, w = min(CB, n - c0), c1 = c0 + w;
    for (int t = tid; t < CB * CB; t += blockDim.x) sL[t / CB][t % CB] = Ld[(size_t)p * CB * CB + t];
    __syncthreads();
    if (tid < CB) {
      double y0 = 0.0, y1 = 0.0, y2 = 0.0;
      if (lane < w) { y0 = x[3 * (c0 + lane)]; y1 = x[3 * (c0 + lane) + 1]; y2 = x[3 * (c0 + lane) + 2]; }
      for (int j = 0; j < w; ++j) {
        if (lane == j) { const double d = sL[j][j]; y0 /= d; y1 /= d; y2 /= d; }
        const double v0 = __shfl_sync(0xffffffffu, y0, j), v1 = __shfl_sync(0xffffffffu, y1, j),
                     v2 = __shfl_sync(0xffffffffu, y2, j);
        if (lane > j) { const double l = sL[lane][j]; y0 -= l * v0; y1 -= l * v1; y2 -= l * v2; }
      }
      if (lane < w) { x[3 * (c0 + lane)] = y0; x[3 * (c0 + lane) + 1] = y1; x[3 * (c0 + lane) + 2] = y2; }
      sy[lane][0] = y0; sy[lane][1] = y1; sy[lane][2] = y2;     // zero past w
    }
    __syncthreads();
    for (int i = c1 + tid; i < n; i += blockDim.x) {
      const double* l = Lp + ((size_t)p * rmax + (i - c1)) * CB;
      double s0 = 0.0, s1 = 0.0, s2 = 0.0;
#pragma unroll 8
      for (int m = 0; m < CB; ++m) {
        const double lm = l[m];
        s0 += lm * sy[m][0]; s1 += lm * sy[m][1]; s2 += lm * sy[m][2];
      }
      x[3 * i] -= s0; x[3 * i + 1] -= s1; x[3 * i + 2] -= s2;
    }
    __syncthreads();
  }
  // backward: L' x = y, panel by panel from the end
  for (int p = np - 1; p >= 0; --p) {
    const int c0 = p * CB, w = min(CB, n - c0), c1 = c0 + w;
    for (int t = tid; t < CB * CB; t += blockDim.x) sL[t / CB][t % CB] = Ld[(size_t)p * CB * CB + t];
    const int c = tid % CB, g = tid / CB;
    double s0 = 0.0, s1 = 0.0, s2 = 0.0;
    if (c < w)
      for (int i = c1 + g; i < n; i += CB) {
        const double l = Lp[((size_t)p * rmax + (i - c1)) * CB + c];
        s0 += l * x[3 * i]; s1 += l * x[3 * i + 1]; s2 += l * x[3 * i + 2];
      }
    sacc[g][c][0] = s0; sacc[g][c][1] = s1; sacc[g][c][2] = s2;
    __syncthreads();
    if (tid < CB) {
      double v0 = 0.0, v1 = 0.0, v2 = 0.0;
      if (lane < w) {
        double a0 = 0.0, a1 = 0.0, a2 = 0.0;
        for (int gg = 0; gg < CB; ++gg) { a0 += sacc[gg][lane][0]; a1 += sacc[gg][lane][1]; a2 += sacc[gg][lane][2]; }
        v0 = x[3 * (c0 + lane)] - a0; v1 = x[3 * (c0 + lane) + 1] - a1; v2 = x[3 * (c0 + lane) + 2] - a2;
      }
      for (int j = w - 1; j >= 0; --j) {
        if (lane == j) { const double d = sL[j][j]; v0 /= d; v1 /= d; v2 /= d; }
        const double u0 = __shfl_sync(0xffffffffu, v0, j), u1 = __shfl_sync(0xffffffffu, v1, j),
                     u2 = __shfl_sync(0xffffffffu, v2, j);
        if (lane < j) { const double l = sL[j][lane]; v0 -= l * u0; v1 -= l * u1; v2 -= l * u2; }
      }
      if (lane < w) { x[3 * (c0 + lane)] = v0; x[3 * (c0 + lane) + 1] = v1; x[3 * (c0 + lane) + 2] = v2; }
    }
    __syncthreads();
  }
}

__device__ inline double step_of(const double* x, int c, int k) { return c == 0 ? 0.0 : x[3 * (c - 1) + k]; }

// per pair, one ADMM iteration of Theia's L1Solver after its x update: A x, over-relaxation, shrinkage, the u update,
// and the pair's terms of the stopping test (|Ax - z - b|^2, |Ax|^2, |z|^2, |b|^2)
__global__ void k_admm_pair(int R, const int* __restrict__ pa, const int* __restrict__ pb, const double* __restrict__ x,
                            const double* __restrict__ bvec, double* __restrict__ z, double* __restrict__ u,
                            double* __restrict__ dz, double* __restrict__ part, const int* skip) {
  if (*skip) return;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= R) return;
  const int a = pa[p], b = pb[p];
  const double kappa = 1.0 / kAdmmRho;
  double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int i = 3 * p + k;
    const double ax = step_of(x, b, k) - step_of(x, a, k);
    const double bb = bvec[i], zo = z[i];
    const double ahat = kAdmmAlpha * ax + (1.0 - kAdmmAlpha) * (zo + bb);
    const double v = ahat - bb + u[i];
    const double zn = fmax(0.0, v - kappa) - fmax(0.0, -v - kappa);
    u[i] += ahat - zn - bb;
    z[i] = zn;
    dz[i] = zn - zo;
    const double e = ax - zn - bb;
    s0 += e * e; s1 += ax * ax; s2 += zn * zn; s3 += bb * bb;
  }
  part[4 * p] = s0; part[4 * p + 1] = s1; part[4 * p + 2] = s2; part[4 * p + 3] = s3;
}

// per non-gauge image: A'(b + z - u) (the next x update's right-hand side), |rho A'(z - z_old)|^2, |rho A'u|^2
__global__ void k_admm_img(int nc, const int* __restrict__ inc_ptr, const int* __restrict__ inc, const double* __restrict__ bvec,
                           const double* __restrict__ z, const double* __restrict__ u, const double* __restrict__ dz,
                           double* __restrict__ atv, double* __restrict__ ipart, const int* skip) {
  if (*skip) return;
  const int c = 1 + blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= nc) return;
  double g[3] = {0.0, 0.0, 0.0}, s[3] = {0.0, 0.0, 0.0}, t[3] = {0.0, 0.0, 0.0};
  for (int e = inc_ptr[c]; e < inc_ptr[c + 1]; ++e) {
    const int p = inc[e] >> 1;
    const double sg = (inc[e] & 1) ? 1.0 : -1.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int i = 3 * p + k;
      g[k] += sg * (bvec[i] + z[i] - u[i]);
      s[k] += sg * dz[i];
      t[k] += sg * u[i];
    }
  }
  double ns = 0.0, nt = 0.0;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    atv[3 * (c - 1) + k] = g[k];
    ns += (kAdmmRho * s[k]) * (kAdmmRho * s[k]);
    nt += (kAdmmRho * t[k]) * (kAdmmRho * t[k]);
  }
  ipart[2 * (c - 1)] = ns; ipart[2 * (c - 1) + 1] = nt;
}

// one CTA: fixed-order norms and Theia's stopping test; counts the iteration, sets the round's done flag
__global__ void __launch_bounds__(1024) k_admm_check(int R, int n, const double* __restrict__ part,
                                                     const double* __restrict__ ipart, Ctl* ctl) {
  __shared__ double sbuf[32];
  if (ctl->admm_done) return;
  double s[4] = {0.0, 0.0, 0.0, 0.0}, t[2] = {0.0, 0.0};
  for (int p = threadIdx.x; p < R; p += blockDim.x)
#pragma unroll
    for (int k = 0; k < 4; ++k) s[k] += part[4 * p + k];
  for (int i = threadIdx.x; i < n; i += blockDim.x) { t[0] += ipart[2 * i]; t[1] += ipart[2 * i + 1]; }
  double S[4], T[2];
#pragma unroll
  for (int k = 0; k < 4; ++k) S[k] = block_sum(s[k], sbuf);
#pragma unroll
  for (int k = 0; k < 2; ++k) T[k] = block_sum(t[k], sbuf);
  if (threadIdx.x == 0) {
    ctl->admm_count += 1;
    const double r_norm = sqrt(S[0]);
    const double max_norm = fmax(fmax(sqrt(S[1]), sqrt(S[2])), sqrt(S[3]));
    const double primal_eps = sqrt(3.0 * R) * kAdmmAbsTolerance + kAdmmRelTolerance * max_norm;
    const double dual_eps = sqrt(3.0 * n) * kAdmmAbsTolerance + kAdmmRelTolerance * sqrt(T[1]);
    if (r_norm < primal_eps && sqrt(T[0]) < dual_eps) ctl->admm_done = 1;
  }
}

// one CTA: UpdateGlobalRotations (R <- ConcatenateQuaternions(q(x), R)) and ComputeAverageStepSize; in IRLS mode
// also counts the iteration and sets its done flag
__global__ void __launch_bounds__(1024) k_update(int nc, const double* __restrict__ x, double* __restrict__ Rq, Ctl* ctl,
                                                 int irls, double threshold) {
  __shared__ double sbuf[32];
  if (irls && ctl->irls_done) return;
  double s = 0.0;
  for (int c = 1 + threadIdx.x; c < nc; c += blockDim.x) {
    const double* xi = x + 3 * (c - 1);
    const Quat q = qconcat(aa_to_quat(xi[0], xi[1], xi[2]), load_q(Rq + 4 * c));
    Rq[4 * c] = q.w; Rq[4 * c + 1] = q.x; Rq[4 * c + 2] = q.y; Rq[4 * c + 3] = q.z;
    s += sqrt(xi[0] * xi[0] + xi[1] * xi[1] + xi[2] * xi[2]);
  }
  s = block_sum(s, sbuf);
  if (threadIdx.x == 0) {
    const double avg = s / (nc - 1);
    ctl->avg_step = avg;
    if (irls) {
      ctl->irls_count += 1;
      if (avg < threshold) ctl->irls_done = 1;
    }
  }
}

// per pair, ComputeResiduals: the angle-axis of R2^-1 R12 R1
__global__ void k_residual(int R, const int* __restrict__ pa, const int* __restrict__ pb, const double* __restrict__ rq,
                           const double* __restrict__ Rq, double* __restrict__ res, const int* skip) {
  if (skip && *skip) return;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= R) return;
  Quat q = qconcat(load_q(Rq + 4 * pa[p]), load_q(rq + 4 * p));
  q = qconcat(q, qinv(load_q(Rq + 4 * pb[p])));
  quat_to_aa(q, res + 3 * p);
}

// per pair, FilterViewPairsFromOrientation's AngularDifferenceIsAcceptable
__global__ void k_filter(int R, const int* __restrict__ pa, const int* __restrict__ pb, const double* __restrict__ rq,
                         const double* __restrict__ Rq, double sq_max, unsigned char* __restrict__ kept) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= R) return;
  const Quat composed = qconcat(qinv(load_q(Rq + 4 * pa[p])), load_q(Rq + 4 * pb[p]));
  const Quat loop = qconcat(composed, qinv(load_q(rq + 4 * p)));
  double a[3];
  quat_to_aa(loop, a);
  kept[p] = (a[0] * a[0] + a[1] * a[1] + a[2] * a[2]) <= sq_max;
}

// ---- host graph work ---------------------------------------------------------------------------------------------
struct UnionFind {
  std::vector<int> parent;
  explicit UnionFind(int n) : parent(n) { std::iota(parent.begin(), parent.end(), 0); }
  int find(int v) {
    while (parent[v] != v) v = parent[v] = parent[parent[v]];
    return v;
  }
  bool unite(int a, int b) {
    a = find(a); b = find(b);
    if (a == b) return false;
    if (a > b) std::swap(a, b);
    parent[b] = a;                 // the root is the smallest image of its component
    return true;
  }
};

// RemoveDisconnectedViewPairs over the listed pairs: the largest component (ties: the one holding the smallest
// image index); returns the kept pairs and marks its images in `in_comp`
std::vector<int> largest_component(int F, const int32_t* pair_images, const std::vector<int>& pairs,
                                   std::vector<char>& in_comp) {
  UnionFind uf(F);
  std::vector<int> size(F, 0);
  std::vector<char> seen(F, 0);
  for (int p : pairs) { uf.unite(pair_images[2 * p], pair_images[2 * p + 1]); seen[pair_images[2 * p]] = seen[pair_images[2 * p + 1]] = 1; }
  for (int f = 0; f < F; ++f) if (seen[f]) ++size[uf.find(f)];
  int best = -1;
  for (int f = 0; f < F; ++f)          // roots are smallest members: ascending f meets components by smallest image
    if (seen[f] && uf.find(f) == f && (best < 0 || size[f] > size[best])) best = f;
  in_comp.assign(F, 0);
  std::vector<int> kept;
  if (best < 0) return kept;
  for (int f = 0; f < F; ++f) in_comp[f] = seen[f] && uf.find(f) == best;
  for (int p : pairs) if (in_comp[pair_images[2 * p]]) kept.push_back(p);
  return kept;
}

int rot_fail(int code, const std::string& msg) {
  set_error("psfm_estimate_global_rotations: " + msg);
  return code;
}

inline unsigned grid_of(long long n) { return (unsigned)std::max<long long>(1, (n + 255) / 256); }

}  // namespace

extern "C" void psfm_rotation_default_options(psfm_rotation_options* o) {
  if (!o) return;
  o->max_num_l1_iterations = 5;
  o->l1_step_convergence_threshold = 0.001;
  o->max_num_irls_iterations = 100;
  o->irls_step_convergence_threshold = 0.001;
  o->irls_loss_parameter_sigma = 5.0 * kDegToRad;
  o->rotation_filter_max_degrees = 5.0;
}

extern "C" int psfm_estimate_global_rotations(int32_t num_images, int64_t num_pairs, const int32_t* pair_images,
                                              const double* qvec, const int32_t* num_correspondences,
                                              const uint8_t* has_pose, const psfm_rotation_options* opts,
                                              double* orientations, uint8_t* has_orientation, uint8_t* pair_kept,
                                              psfm_rotation_summary* summary) {
  const auto t0 = std::chrono::steady_clock::now();
  const long long launches0 = g_launch_count.load();
  if (num_images < 0 || num_pairs < 0) return rot_fail(PSFM_ERR_INVALID, "negative size");
  if (num_pairs > 0x7fffffffLL) return rot_fail(PSFM_ERR_INVALID, "more than 2^31 - 1 pairs");
  if ((num_pairs > 0 && (!pair_images || !qvec || !num_correspondences || !pair_kept)) ||
      (num_images > 0 && (!orientations || !has_orientation)))
    return rot_fail(PSFM_ERR_INVALID, "null argument");
  psfm_rotation_options o;
  psfm_rotation_default_options(&o);
  if (opts) o = *opts;
  if (!(o.max_num_l1_iterations > 0 && o.l1_step_convergence_threshold > 0.0 && o.max_num_irls_iterations > 0 &&
        o.irls_step_convergence_threshold > 0.0 && o.irls_loss_parameter_sigma > 0.0 && o.rotation_filter_max_degrees > 0.0))
    return rot_fail(PSFM_ERR_INVALID, "options fail RobustRotationEstimator::Options::Check()");
  const int F = num_images, R = (int)num_pairs;
  {
    std::vector<uint64_t> keys(R);
    for (int p = 0; p < R; ++p) {
      const int a = pair_images[2 * p], b = pair_images[2 * p + 1];
      if (a < 0 || a >= F || b < 0 || b >= F) return rot_fail(PSFM_ERR_INVALID, "an image index is outside [0, num_images)");
      if (a == b) return rot_fail(PSFM_ERR_INVALID, "a pair of an image with itself");
      keys[p] = ((uint64_t)std::min(a, b) << 32) | (uint64_t)std::max(a, b);
    }
    std::sort(keys.begin(), keys.end());
    if (std::adjacent_find(keys.begin(), keys.end()) != keys.end())
      return rot_fail(PSFM_ERR_INVALID, "an unordered image pair is listed twice");
  }
  if (o.max_num_l1_iterations > PSFM_ROTATION_MAX_L1_ROUNDS)
    return rot_fail(PSFM_ERR_UNSUPPORTED, "max_num_l1_iterations above PSFM_ROTATION_MAX_L1_ROUNDS");

  psfm_rotation_summary sm;
  memset(&sm, 0, sizeof(sm));
  sm.gauge_image = -1;
  for (int f = 0; f < F; ++f) { has_orientation[f] = 0; for (int k = 0; k < 4; ++k) orientations[4 * f + k] = 0.0; }
  for (int p = 0; p < R; ++p) pair_kept[p] = 0;
  auto finish = [&](int rc) {
    sm.num_launches = g_launch_count.load() - launches0;
    if (summary) *summary = sm;
    return rc;
  };
  // AllPairs(only_with_pose), then the first RemoveDisconnectedViewPairs
  std::vector<int> posed;
  for (int p = 0; p < R; ++p) {
    bool ok = !has_pose || has_pose[p];
    for (int k = 0; k < 4; ++k) ok = ok && std::isfinite(qvec[4 * p + k]);
    if (ok) posed.push_back(p);
  }
  std::vector<char> in_comp;
  const std::vector<int> cp = largest_component(F, pair_images, posed, in_comp);
  if (cp.empty()) {
    set_error("psfm_estimate_global_rotations: no image pair with a pose");
    return finish(PSFM_NO_ROTATIONS);
  }
  std::vector<int> cidx(F, -1), cimg;
  for (int f = 0; f < F; ++f) if (in_comp[f]) { cidx[f] = (int)cimg.size(); cimg.push_back(f); }
  const int nc = (int)cimg.size(), n = nc - 1, Rc = (int)cp.size();
  if (nc > kMaxComponentImages) return rot_fail(PSFM_ERR_UNSUPPORTED, "more than 8192 images in the kept component");
  sm.gauge_image = cimg[0];
  sm.num_images_connected = nc;
  sm.num_pairs_connected = Rc;
  std::vector<int> pa(Rc), pb(Rc);
  std::vector<double> rq(4 * (size_t)Rc);
  for (int i = 0; i < Rc; ++i) {
    pa[i] = cidx[pair_images[2 * cp[i]]];
    pb[i] = cidx[pair_images[2 * cp[i] + 1]];
    for (int k = 0; k < 4; ++k) rq[4 * i + k] = qvec[4 * (size_t)cp[i] + k];
  }
  // OrientationsFromMaximumSpanningTree: Kruskal on (-num_correspondences, image 1, image 2), then chaining from
  // the gauge image (on a tree the traversal order does not change the result)
  std::vector<int> order(Rc);
  std::iota(order.begin(), order.end(), 0);
  std::sort(order.begin(), order.end(), [&](int i, int j) {
    const int ni = num_correspondences[cp[i]], nj = num_correspondences[cp[j]];
    if (ni != nj) return ni > nj;
    if (pa[i] != pa[j]) return pa[i] < pa[j];
    return pb[i] < pb[j];
  });
  std::vector<std::vector<int>> tree(nc);
  {
    UnionFind uf(nc);
    for (int i : order)
      if (uf.unite(pa[i], pb[i])) { tree[pa[i]].push_back(i); tree[pb[i]].push_back(i); }
  }
  std::vector<double> Rq(4 * (size_t)nc, 0.0);
  {
    std::vector<char> done(nc, 0);
    std::vector<int> queue(1, 0);
    Rq[0] = 1.0;
    done[0] = 1;
    for (size_t h = 0; h < queue.size(); ++h) {
      const int s = queue[h];
      double Rs[3][3], Rr[3][3], Rn[3][3];
      quat_to_matrix({Rq[4 * s], Rq[4 * s + 1], Rq[4 * s + 2], Rq[4 * s + 3]}, Rs);
      for (int i : tree[s]) {
        const bool src_first = pa[i] == s;
        const int t = src_first ? pb[i] : pa[i];
        if (done[t]) continue;
        quat_to_matrix({rq[4 * i], rq[4 * i + 1], rq[4 * i + 2], rq[4 * i + 3]}, Rr);
        for (int r = 0; r < 3; ++r)
          for (int c = 0; c < 3; ++c) {
            double v = 0.0;
            for (int k = 0; k < 3; ++k) v += (src_first ? Rr[r][k] : Rr[k][r]) * Rs[k][c];
            Rn[r][c] = v;
          }
        const Quat q = matrix_to_quat(Rn);
        Rq[4 * t] = q.w; Rq[4 * t + 1] = q.x; Rq[4 * t + 2] = q.y; Rq[4 * t + 3] = q.z;
        done[t] = 1;
        queue.push_back(t);
      }
    }
  }
  // image -> incident pairs, in pair order; bit 0: the image is the pair's image 2 (+I in A), else image 1 (-I)
  std::vector<int> inc_ptr(nc + 1, 0), inc(2 * (size_t)Rc);
  for (int i = 0; i < Rc; ++i) { ++inc_ptr[pa[i] + 1]; ++inc_ptr[pb[i] + 1]; }
  for (int c = 0; c < nc; ++c) inc_ptr[c + 1] += inc_ptr[c];
  {
    std::vector<int> fill(inc_ptr.begin(), inc_ptr.end() - 1);
    for (int i = 0; i < Rc; ++i) { inc[fill[pa[i]]++] = 2 * i; inc[fill[pb[i]]++] = 2 * i + 1; }
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return rot_fail(PSFM_ERR_NO_DEVICE, "no CUDA device available (this library has no CPU path)");
  }
  const auto t1 = std::chrono::steady_clock::now();
  std::vector<unsigned char> kept(Rc);
  try {
    const int lda = n + 1, np = dense_chol_panels(n), rmax = dense_chol_rmax(n);
    DBuf<int> d_pa, d_pb, d_inc_ptr, d_inc, d_fail;
    DBuf<double> d_rq, d_R, d_res, d_z, d_u, d_dz, d_w, d_wr, d_part, d_ipart, d_atv, d_x, d_A, d_xc, d_Lp, d_Ld;
    DBuf<unsigned int> d_bar;
    DBuf<Ctl> d_ctl;
    DBuf<unsigned char> d_kept;
    d_pa.alloc(Rc); d_pb.alloc(Rc); d_inc_ptr.alloc(nc + 1); d_inc.alloc(2 * (size_t)Rc); d_fail.alloc(1);
    d_rq.alloc(4 * (size_t)Rc); d_R.alloc(4 * (size_t)nc); d_res.alloc(3 * (size_t)Rc); d_z.alloc(3 * (size_t)Rc);
    d_u.alloc(3 * (size_t)Rc); d_dz.alloc(3 * (size_t)Rc); d_w.alloc(Rc); d_wr.alloc(3 * (size_t)Rc);
    d_part.alloc(4 * (size_t)Rc); d_ipart.alloc(2 * (size_t)n); d_atv.alloc(3 * (size_t)n); d_x.alloc(3 * (size_t)n);
    d_A.alloc((size_t)lda * lda); d_xc.alloc(n); d_Lp.alloc((size_t)np * rmax * kDenseCholBlock);
    d_Ld.alloc((size_t)np * kDenseCholBlock * kDenseCholBlock); d_bar.alloc(1); d_ctl.alloc(1); d_kept.alloc(Rc);
    d_pa.upload(pa.data(), Rc, nullptr); d_pb.upload(pb.data(), Rc, nullptr);
    d_inc_ptr.upload(inc_ptr.data(), nc + 1, nullptr); d_inc.upload(inc.data(), 2 * (size_t)Rc, nullptr);
    d_rq.upload(rq.data(), 4 * (size_t)Rc, nullptr); d_R.upload(Rq.data(), 4 * (size_t)nc, nullptr);
    d_ctl.zero(nullptr);
    Ctl* ctl = d_ctl.p;
    const unsigned gp = grid_of(Rc), gi = grid_of(n);
    auto factor = [&](bool weighted, const int* skip) {
      PSFM_CUDA(cudaMemsetAsync(d_A.p, 0, sizeof(double) * (size_t)lda * lda, nullptr));
      k_lap_pair<<<gp, 256>>>(Rc, d_pa.p, d_pb.p, d_res.p, o.irls_loss_parameter_sigma, weighted, d_A.p, lda, d_w.p,
                              d_wr.p, skip);
      PSFM_LAUNCH_CHECK();
      k_lap_img<<<gi, 256>>>(nc, d_inc_ptr.p, d_inc.p, d_w.p, d_wr.p, d_A.p, lda, d_atv.p, skip);
      PSFM_LAUNCH_CHECK();
      dense_cholesky_launch(d_A.p, n, d_xc.p, d_fail.p, d_bar.p, d_Lp.p, d_Ld.p, nullptr);
    };
    auto read_ctl = [&]() {
      Ctl h;
      PSFM_CUDA(cudaMemcpy(&h, ctl, sizeof(Ctl), cudaMemcpyDeviceToHost));
      return h;
    };
    // ComputeResiduals of the spanning-tree orientations; L1Solver factors A'A once
    k_residual<<<gp, 256>>>(Rc, d_pa.p, d_pb.p, d_rq.p, d_R.p, d_res.p, nullptr);
    PSFM_LAUNCH_CHECK();
    factor(false, nullptr);
    // SolveL1Regression
    int cap = 5;
    for (int round = 0; round < o.max_num_l1_iterations; ++round) {
      PSFM_CUDA(cudaMemsetAsync(d_z.p, 0, sizeof(double) * 3 * (size_t)Rc, nullptr));
      PSFM_CUDA(cudaMemsetAsync(d_u.p, 0, sizeof(double) * 3 * (size_t)Rc, nullptr));
      PSFM_CUDA(cudaMemsetAsync(d_dz.p, 0, sizeof(double) * 3 * (size_t)Rc, nullptr));
      PSFM_CUDA(cudaMemsetAsync(&ctl->admm_done, 0, 2 * sizeof(int), nullptr));     // admm_done, admm_count
      k_admm_img<<<gi, 256>>>(nc, d_inc_ptr.p, d_inc.p, d_res.p, d_z.p, d_u.p, d_dz.p, d_atv.p, d_ipart.p, &ctl->admm_done);
      PSFM_LAUNCH_CHECK();
      for (int it = 0; it < cap; ++it) {
        k_trsv<<<1, 1024>>>(n, d_Ld.p, d_Lp.p, d_atv.p, d_x.p, d_fail.p, ctl, &ctl->admm_done);
        PSFM_LAUNCH_CHECK();
        k_admm_pair<<<gp, 256>>>(Rc, d_pa.p, d_pb.p, d_x.p, d_res.p, d_z.p, d_u.p, d_dz.p, d_part.p, &ctl->admm_done);
        PSFM_LAUNCH_CHECK();
        k_admm_img<<<gi, 256>>>(nc, d_inc_ptr.p, d_inc.p, d_res.p, d_z.p, d_u.p, d_dz.p, d_atv.p, d_ipart.p, &ctl->admm_done);
        PSFM_LAUNCH_CHECK();
        k_admm_check<<<1, 1024>>>(Rc, n, d_part.p, d_ipart.p, ctl);
        PSFM_LAUNCH_CHECK();
      }
      k_update<<<1, 1024>>>(nc, d_x.p, d_R.p, ctl, 0, 0.0);
      PSFM_LAUNCH_CHECK();
      k_residual<<<gp, 256>>>(Rc, d_pa.p, d_pb.p, d_rq.p, d_R.p, d_res.p, nullptr);
      PSFM_LAUNCH_CHECK();
      const Ctl h = read_ctl();
      if (h.failed) { set_error("psfm_estimate_global_rotations: the L1 system's factorisation failed"); return finish(PSFM_NO_ROTATIONS); }
      sm.num_l1_rounds = round + 1;
      sm.admm_iterations[round] = h.admm_count;
      sm.l1_final_step = h.avg_step;
      if (h.avg_step <= o.l1_step_convergence_threshold) break;
      cap *= 2;
    }
    // SolveIRLS
    for (int it = 0; it < o.max_num_irls_iterations;) {
      const int chunk = std::min(kIrlsChunk, o.max_num_irls_iterations - it);
      for (int j = 0; j < chunk; ++j) {
        factor(true, &ctl->irls_done);
        k_trsv<<<1, 1024>>>(n, d_Ld.p, d_Lp.p, d_atv.p, d_x.p, d_fail.p, ctl, &ctl->irls_done);
        PSFM_LAUNCH_CHECK();
        k_update<<<1, 1024>>>(nc, d_x.p, d_R.p, ctl, 1, o.irls_step_convergence_threshold);
        PSFM_LAUNCH_CHECK();
        k_residual<<<gp, 256>>>(Rc, d_pa.p, d_pb.p, d_rq.p, d_R.p, d_res.p, &ctl->irls_done);
        PSFM_LAUNCH_CHECK();
      }
      it += chunk;
      const Ctl h = read_ctl();
      if (h.failed) { set_error("psfm_estimate_global_rotations: the IRLS system's factorisation failed"); return finish(PSFM_NO_ROTATIONS); }
      sm.num_irls_iterations = h.irls_count;
      sm.irls_final_step = h.avg_step;
      if (h.irls_done) break;
    }
    const double rad = o.rotation_filter_max_degrees * kDegToRad;
    k_filter<<<gp, 256>>>(Rc, d_pa.p, d_pb.p, d_rq.p, d_R.p, rad * rad, d_kept.p);
    PSFM_LAUNCH_CHECK();
    PSFM_CUDA(cudaMemcpy(Rq.data(), d_R.p, sizeof(double) * 4 * (size_t)nc, cudaMemcpyDeviceToHost));
    PSFM_CUDA(cudaMemcpy(kept.data(), d_kept.p, Rc, cudaMemcpyDeviceToHost));
  } catch (const CudaFail& f) { return finish(f.code); }
  const auto t2 = std::chrono::steady_clock::now();
  // the second RemoveDisconnectedViewPairs; every image of the first component keeps its orientation
  for (int c = 0; c < nc; ++c) {
    has_orientation[cimg[c]] = 1;
    for (int k = 0; k < 4; ++k) orientations[4 * (size_t)cimg[c] + k] = Rq[4 * c + k];
  }
  std::vector<int> filtered;
  for (int i = 0; i < Rc; ++i) if (kept[i]) filtered.push_back(cp[i]);
  std::vector<char> in_kept;
  const std::vector<int> fin = largest_component(F, pair_images, filtered, in_kept);
  for (int p : fin) pair_kept[p] = 1;
  sm.num_pairs_kept = (int)fin.size();
  sm.num_images_kept = (int)std::count(in_kept.begin(), in_kept.end(), 1);
  const auto t3 = std::chrono::steady_clock::now();
  const auto ms = [](auto a, auto b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
  sm.host_ms = ms(t0, t1) + ms(t2, t3);
  sm.device_ms = ms(t1, t2);
  return finish(PSFM_OK);
}
