// verification.cu — the two-view geometric verification of `colmap matches_importer --match_type pairs`: raw matches
// in, each pair's config, F, H and inlier matches out (DESIGN.md §4.8).
//
// Reference: TwoViewGeometryVerifier -> TwoViewGeometry::Estimate -> EstimateUncalibrated (SIMPLE_PINHOLE cameras
// without a prior focal length): LORANSAC<seven-point F, eight-point F> on the squared Sampson error,
// LORANSAC<normalised DLT H, same> on the squared transfer error, the config rule, F's inliers, DetectWatermark with
// LORANSAC<translation, translation> (verification_recalled.cuh).  The restatement is oracle/verification_oracle.py.
//
// Device (R pairs, M raw matches):
//   gather   k_gather: each match's two keypoints as one float4 (x1, y1, x2, y2), 16 B per match
//   verify   k_verify: one CTA per pair.  The leader thread draws each trial's sample and builds its models (the
//            seven-point null space by Householder QR of A', never A'A; the cubic by one closed-form root, deflation
//            and the stable quadratic; the DLT likewise);
//            the CTA scores all models of the sample in one sweep over the pair's matches (per-thread partials, then a
//            fixed-order block reduction); the leader applies the support comparison, the dynamic trial bound and the
//            stopping test in model order.  Local optimisation sweeps the best model's inliers for their moments and
//            the R factor of the normalised rows (Givens rotations, never A'A), takes R's smallest right singular
//            vector with the one-sided Jacobi of dlt.cuh, and scores the local model.  Then F's inliers are compacted
//            in match order, the watermark test and its translation LORANSAC run on them, and the config is decided.
//   compact  k_compact: the inlier matches packed by the host's prefix sum of the per-pair counts
// Trials run in the sequential order, so every scored trial is a trial of the reference loop (no trial is scored and
// discarded).  Three launches per call with pairs, none without; no floating-point atomics: two calls are
// bit-identical.  Memory: 16 B per match for the gathered points, 4 B for the inlier list, 8 B for the output.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <vector>

#include "dlt.cuh"
#include "match_table.cuh"
#include "pair_inputs.h"
#include "psfm_common.cuh"
#include "verification_recalled.cuh"

namespace {

using namespace psfm;
using namespace psfm::ver;
typedef unsigned long long u64;

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
enum { kKindF = 0, kKindH = 1, kKindW = 2 };
enum { kUndefined = 0, kDegenerate = 1, kUncalibrated = 3, kPlanarOrPanoramic = 6, kWatermark = 7 };

struct Args {
  int R;
  const long long* mptr;           // [R + 1]
  const float4* pts;               // [M] gathered (x1, y1, x2, y2)
  const int2* sizes;               // [R][2] camera (width, height) of image 1, of image 2
  int* inl_idx;                    // [M] per pair at mptr[p]: F's inliers (indices into the pair's matches)
  int* config;                     // [R]
  double* F;                       // [R][9] stored form
  double* H;                       // [R][9]
  long long* count;                // [R] inliers
  int* trials;                     // [R][3]
  int* rounds;                     // [R][3]
  double thr;                      // max_error^2
  double confidence, multiplier;
  long long max_trials[3];         // per kind, after the constructor's cap
  long long min_trials;
  int min_num_inliers;
  double max_H_ratio;
  int detect_watermark;
  double wm_ratio, wm_border;
  u64 seed;
};

// ---- sampler: SplitMix64 streams keyed by (seed, pair, kind, trial) -------------------------------------------------
constexpr u64 kGolden = 0x9E3779B97F4A7C15ull;

__device__ __forceinline__ u64 mix64(u64 z) {
  z ^= z >> 30; z *= 0xBF58476D1CE4E5B9ull;
  z ^= z >> 27; z *= 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

__device__ void draw_sample(u64 seed, u64 pair, u64 kind, u64 trial, unsigned n, int k, int* idx) {
  u64 s = mix64(seed + kGolden * (pair + 1));
  s = mix64(s + kGolden * (kind + 1));
  s = mix64(s + kGolden * (trial + 1));
  int got = 0;
  while (got < k) {
    s += kGolden;
    const int i = (int)(((mix64(s) >> 32) * (u64)n) >> 32);
    bool dup = false;
    for (int j = 0; j < got; ++j) dup |= idx[j] == i;
    if (!dup) idx[got++] = i;
  }
}

// ---- residuals ------------------------------------------------------------------------------------------------------
template <int KIND>
__device__ __forceinline__ double residual(const double* f, float4 p) {
  const double X = p.x, Y = p.y, U = p.z, V = p.w;
  if (KIND == kKindF) {                        // ComputeSquaredSampsonError
    const double e0 = f[0] * X + f[1] * Y + f[2];
    const double e1 = f[3] * X + f[4] * Y + f[5];
    const double e2 = f[6] * X + f[7] * Y + f[8];
    const double t0 = f[0] * U + f[3] * V + f[6];
    const double t1 = f[1] * U + f[4] * V + f[7];
    const double c = U * e0 + V * e1 + e2;
    return c * c / (e0 * e0 + e1 * e1 + t0 * t0 + t1 * t1);
  } else if (KIND == kKindH) {                 // squared transfer error in image 2
    const double inv = 1.0 / (f[6] * X + f[7] * Y + f[8]);
    const double d0 = U - (f[0] * X + f[1] * Y + f[2]) * inv;
    const double d1 = V - (f[3] * X + f[4] * Y + f[5]) * inv;
    return d0 * d0 + d1 * d1;
  } else {                                     // translation
    const double d0 = U - (X + f[0]), d1 = V - (Y + f[1]);
    return d0 * d0 + d1 * d1;
  }
}

// ---- minimal estimators (one thread) --------------------------------------------------------------------------------
// null space of the M x 9 system A (M < 9) from the Householder QR of A': the last 9 - M columns of Q
template <int M>
__device__ void null_space_qr(double (&B)[9][M], double (*out)[9]) {   // B = A' (destroyed)
  double beta[M];
#pragma unroll
  for (int j = 0; j < M; ++j) {
    double nrm = 0.0;
#pragma unroll
    for (int i = 0; i < 9; ++i)
      if (i >= j) nrm += B[i][j] * B[i][j];
    nrm = sqrt(nrm);
    if (nrm == 0.0) { beta[j] = 0.0; continue; }
    const double alpha = B[j][j] >= 0.0 ? -nrm : nrm;
    B[j][j] -= alpha;
    double vtv = 0.0;
#pragma unroll
    for (int i = 0; i < 9; ++i)
      if (i >= j) vtv += B[i][j] * B[i][j];
    beta[j] = 2.0 / vtv;
#pragma unroll
    for (int c = j + 1; c < M; ++c) {
      double d = 0.0;
#pragma unroll
      for (int i = 0; i < 9; ++i)
        if (i >= j) d += B[i][j] * B[i][c];
      d *= beta[j];
#pragma unroll
      for (int i = 0; i < 9; ++i)
        if (i >= j) B[i][c] -= d * B[i][j];
    }
  }
#pragma unroll
  for (int k = M; k < 9; ++k) {
    double x[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) x[i] = i == k ? 1.0 : 0.0;
#pragma unroll
    for (int j = M - 1; j >= 0; --j) {
      double d = 0.0;
#pragma unroll
      for (int i = 0; i < 9; ++i)
        if (i >= j) d += B[i][j] * x[i];
      d *= beta[j];
#pragma unroll
      for (int i = 0; i < 9; ++i)
        if (i >= j) x[i] -= d * B[i][j];
    }
#pragma unroll
    for (int i = 0; i < 9; ++i) out[k - M][i] = x[i];
  }
}

__device__ __forceinline__ double det3(const double* f) {
  return f[0] * (f[4] * f[8] - f[5] * f[7]) - f[1] * (f[3] * f[8] - f[5] * f[6]) + f[2] * (f[3] * f[7] - f[4] * f[6]);
}

// one Newton step, kept only when it lowers |p|: at a near-multiple root p' is rounding noise and the step can jump far
__device__ __forceinline__ double newton_step(double c3, double c2, double c1, double c0, double x) {
  const double f = ((c3 * x + c2) * x + c1) * x + c0;
  const double df = (3.0 * c3 * x + 2.0 * c2) * x + c1;
  if (df == 0.0) return x;
  const double y = x - f / df;
  const double g = ((c3 * y + c2) * y + c1) * y + c0;
  return fabs(g) < fabs(f) ? y : x;
}

// the roots of a x^2 + b x + c (a != 0) for a discriminant d >= 0: h = -(b + sign(b) sqrt(d)) / 2 adds magnitudes, so
// neither h / a nor c / h cancels
__device__ __forceinline__ void stable_quadratic(double a, double b, double c, double d, double* x) {
  const double h = -0.5 * (b + copysign(sqrt(d), b));
  x[0] = h / a;
  x[1] = h != 0.0 ? c / h : 0.0;
}

// Real roots of c3 x^3 + c2 x^2 + c1 x + c0, one Newton step each (oracle: cubic_real_roots).  One real root r comes
// from the depressed cubic's closed form: Cardano with the two cube roots added without cancellation, or the
// trigonometric form's largest-magnitude root.  After its Newton step r is deflated out, from the constant term when it
// is the largest root and from the leading term otherwise (the stable direction each way), and the quadratic left
// decides whether there are two more real roots and gives them in the stable form.  The depressed form yields no other
// root: once c3 is small its shift -c2 / 3 c3 swamps the moderate roots, and its discriminant cancels.
__device__ int cubic_real_roots(double c3, double c2, double c1, double c0, double* x) {
  if (c3 == 0.0) {
    if (c2 == 0.0) {
      if (c1 == 0.0) return 0;
      x[0] = -c0 / c1;
      return 1;
    }
    const double d = c1 * c1 - 4.0 * c2 * c0;
    if (d < 0.0) return 0;
    stable_quadratic(c2, c1, c0, d, x);
    return 2;
  }
  const double b = c2 / c3, c = c1 / c3, d = c0 / c3;
  const double p = c - b * b / 3.0;
  const double q = 2.0 * b * b * b / 27.0 - b * c / 3.0 + d;
  const double disc = (q / 2.0) * (q / 2.0) + (p / 3.0) * (p / 3.0) * (p / 3.0);
  const double shift = -b / 3.0;
  double r = shift;
  if (disc > 0.0) {
    const double A = -copysign(cbrt(fabs(q) / 2.0 + sqrt(disc)), q);
    r = (A != 0.0 ? A - p / (3.0 * A) : 0.0) + shift;
  } else if (p != 0.0) {
    const double rr = 2.0 * sqrt(-p / 3.0);
    const double a = 3.0 * q / (2.0 * p) * sqrt(-3.0 / p);
    const double phi = acos(fmin(1.0, fmax(-1.0, a))) / 3.0;
    r = 0.0;
    for (int k = 0; k < 3; ++k) {
      const double t = rr * cos(phi - 2.0 * M_PI * k / 3.0) + shift;
      if (fabs(t) > fabs(r)) r = t;
    }
  }
  r = newton_step(c3, c2, c1, c0, r);
  x[0] = r;
  // c3 x^2 + e1 x + e0 = p(x) / (x - r); r is the largest root when |c3 r^3| >= |c0| = |c3 r r1 r2|
  const bool backward = r != 0.0 && fabs(c3 * r * r * r) >= fabs(c0);
  double e1, e0;
  if (backward) { e0 = -c0 / r; e1 = (e0 - c1) / r; }
  else { e1 = c2 + c3 * r; e0 = c1 + e1 * r; }
  const double dq = e1 * e1 - 4.0 * c3 * e0;
  if (dq < 0.0) return 1;
  stable_quadratic(c3, e1, e0, dq, x + 1);
  x[1] = newton_step(c3, c2, c1, c0, x[1]);
  x[2] = newton_step(c3, c2, c1, c0, x[2]);
  return 3;
}

__device__ bool lex_less(const double* u, const double* v) {
  for (int i = 0; i < 9; ++i)
    if (u[i] != v[i]) return u[i] < v[i];
  return false;
}

// FundamentalMatrixSevenPointEstimator on raw pixels; models scaled to F(2,2) = 1 and ordered by (F00, F01, ...)
__device__ __noinline__ int seven_point(const float4* p, double (*models)[9]) {
  double B[9][7];
#pragma unroll
  for (int i = 0; i < 7; ++i) {
    const double x0 = p[i].x, y0 = p[i].y, x1 = p[i].z, y1 = p[i].w;
    B[0][i] = x1 * x0; B[1][i] = x1 * y0; B[2][i] = x1;
    B[3][i] = y1 * x0; B[4][i] = y1 * y0; B[5][i] = y1;
    B[6][i] = x0; B[7][i] = y0; B[8][i] = 1.0;
  }
  double ns[2][9];
  null_space_qr<7>(B, ns);
  const double* a = ns[0];
  const double* b = ns[1];
  double t1[9], tm[9];
  for (int i = 0; i < 9; ++i) { t1[i] = a[i] + b[i]; tm[i] = -a[i] + b[i]; }
  const double d0 = det3(b), d1 = det3(t1), dm = det3(tm), c3 = det3(a);
  const double c2 = 0.5 * (d1 + dm) - d0;
  const double c1 = 0.5 * (d1 - dm) - c3;
  // det(lam a + b) = c3 lam^3 + c2 lam^2 + c1 lam + d0; when |c3| < |d0| the pencil is solved as det(a + mu b) =
  // d0 mu^3 + c1 mu^2 + c2 mu + c3 instead, whose leading coefficient is the larger one (mu = 0 is F = a, lam = inf)
  const bool flip = fabs(c3) < fabs(d0);
  double lam[3];
  const int nr = flip ? cubic_real_roots(d0, c1, c2, c3, lam) : cubic_real_roots(c3, c2, c1, d0, lam);
  int nm = 0;
  for (int r = 0; r < nr; ++r) {
    double F[9], nrm = 0.0;
    for (int i = 0; i < 9; ++i) { F[i] = flip ? a[i] + lam[r] * b[i] : lam[r] * a[i] + b[i]; nrm += F[i] * F[i]; }
    if (fabs(F[8] / sqrt(nrm)) < kMinF22) continue;
    const double s = F[8];
    for (int i = 0; i < 9; ++i) F[i] /= s;
    int pos = nm;                              // insertion in (F00, F01, ...) order
    while (pos > 0 && lex_less(F, models[pos - 1])) {
      for (int i = 0; i < 9; ++i) models[pos][i] = models[pos - 1][i];
      --pos;
    }
    for (int i = 0; i < 9; ++i) models[pos][i] = F[i];
    ++nm;
  }
  return nm;
}

// CenterAndNormalizeImagePoints of k points: scale s and centroid c (T = [s 0 -s cx; 0 s -s cy; 0 0 1])
template <int K>
__device__ void normalize_points(const double (&x)[K], const double (&y)[K], double& s, double& cx, double& cy) {
  cx = 0.0; cy = 0.0;
  for (int i = 0; i < K; ++i) { cx += x[i]; cy += y[i]; }
  cx /= K; cy /= K;
  double r = 0.0;
  for (int i = 0; i < K; ++i) r += (x[i] - cx) * (x[i] - cx) + (y[i] - cy) * (y[i] - cy);
  s = sqrt(2.0) / sqrt(r / K);
}

// H = T2^-1 Hn T1 with T = [s 0 -s cx; 0 s -s cy; 0 0 1]
__device__ void denormalize_h(const double* hn, double s1, double c1x, double c1y, double s2, double c2x, double c2y, double* H) {
  double A[9];                                 // Hn T1
  for (int r = 0; r < 3; ++r) {
    A[3 * r + 0] = hn[3 * r + 0] * s1;
    A[3 * r + 1] = hn[3 * r + 1] * s1;
    A[3 * r + 2] = -s1 * c1x * hn[3 * r + 0] - s1 * c1y * hn[3 * r + 1] + hn[3 * r + 2];
  }
  const double i2 = 1.0 / s2;                  // T2^-1 = [1/s 0 cx; 0 1/s cy; 0 0 1]
  for (int c = 0; c < 3; ++c) {
    H[c] = i2 * A[c] + c2x * A[6 + c];
    H[3 + c] = i2 * A[3 + c] + c2y * A[6 + c];
    H[6 + c] = A[6 + c];
  }
}

// HomographyMatrixEstimator on 4 points: normalised DLT, null vector by Householder QR
__device__ __noinline__ int homography_minimal(const float4* p, double* H) {
  double x1[4], y1[4], x2[4], y2[4];
  for (int i = 0; i < 4; ++i) { x1[i] = p[i].x; y1[i] = p[i].y; x2[i] = p[i].z; y2[i] = p[i].w; }
  double s1, c1x, c1y, s2, c2x, c2y;
  normalize_points<4>(x1, y1, s1, c1x, c1y);
  normalize_points<4>(x2, y2, s2, c2x, c2y);
  double B[9][8];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const double a0 = (x1[i] - c1x) * s1, a1 = (y1[i] - c1y) * s1, d0 = (x2[i] - c2x) * s2, d1 = (y2[i] - c2y) * s2;
    const int r = 2 * i, q = 2 * i + 1;
    B[0][r] = -a0; B[1][r] = -a1; B[2][r] = -1.0; B[3][r] = 0.0; B[4][r] = 0.0; B[5][r] = 0.0;
    B[6][r] = a0 * d0; B[7][r] = a1 * d0; B[8][r] = d0;
    B[0][q] = 0.0; B[1][q] = 0.0; B[2][q] = 0.0; B[3][q] = -a0; B[4][q] = -a1; B[5][q] = -1.0;
    B[6][q] = a0 * d1; B[7][q] = a1 * d1; B[8][q] = d1;
  }
  double ns[1][9];
  null_space_qr<8>(B, ns);
  denormalize_h(ns[0], s1, c1x, c1y, s2, c2x, c2y, H);
  return 1;
}

// ---- block-level pieces -----------------------------------------------------------------------------------------------
struct Shared {
  double models[3][9];
  double best[9];
  double local[9];
  double red[kWarps][45];
  double tot[45];
  double G[81], GV[81];            // the local step's 9 x 9 R factor and its right singular vectors (leader only)
  double lnull[9], lnorm[6];       // the local step's normalised null vector and (s1, c1x, c1y, s2, c2x, c2y)
  double best_sum;
  long long best_n;
  long long dyn;
  int idx[8];
  int nm;
  int have_best;
  int flag_better, flag_lo, flag_stop, abort_;
  int trials, rounds;
  int wsum[kWarps];
};

// sum of N per-thread values over the CTA in a fixed order; the totals land in s.tot (all threads see them)
template <int N>
__device__ void block_reduce(double (&v)[N], Shared& s) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < N; ++k) {
    const double w = warp_sum(v[k]);
    if (lane == 0) s.red[wid][k] = w;
  }
  __syncthreads();
  if (threadIdx.x < N) {
    double t = 0.0;
    for (int w = 0; w < kWarps; ++w) t += s.red[w][threadIdx.x];
    s.tot[threadIdx.x] = t;
  }
  __syncthreads();
}

template <int KIND>
__device__ __forceinline__ float4 point(const float4* pts, const int* list, int i) {
  return KIND == kKindW ? pts[list[i]] : pts[i];
}

// inlier counts and residual sums of nm models (nm <= 3) in one sweep: s.tot[m] counts, s.tot[3 + m] sums
template <int KIND>
__device__ void score(const double (*models)[9], int nm, const float4* pts, const int* list, int n, double thr, Shared& s) {
  double v[6] = {0, 0, 0, 0, 0, 0};
  double m[3][9];
  for (int k = 0; k < nm; ++k)
    for (int i = 0; i < 9; ++i) m[k][i] = models[k][i];
  for (int i = threadIdx.x; i < n; i += kThreads) {
    const float4 p = point<KIND>(pts, list, i);
#pragma unroll
    for (int k = 0; k < 3; ++k)
      if (k < nm) {
        const double r = residual<KIND>(m[k], p);
        if (r <= thr) { v[k] += 1.0; v[3 + k] += r; }
      }
  }
  block_reduce<6>(v, s);
}

// The local step's R factor: the 9 x 9 upper triangle of the normalised design matrix's QR, packed by rows.  Solving R
// instead of the Gram matrix A'A keeps the null vector's error proportional to A's condition number, not its square.
__device__ __forceinline__ constexpr int tri(int j, int k) { return j * (17 - j) / 2 + k; }

// fold the row r (zero before column j0) into R by Givens rotations, column by column; r is destroyed
__device__ __forceinline__ void givens_fold(double (&R)[45], double (&r)[9], int j0) {
#pragma unroll
  for (int j = 0; j < 9; ++j) {
    if (j < j0) continue;
    const double b = r[j];
    if (b == 0.0) continue;
    const double a = R[tri(j, j)];
    const double h = sqrt(a * a + b * b), c = a / h, sn = b / h;
    R[tri(j, j)] = h;
#pragma unroll
    for (int k = j + 1; k < 9; ++k) {
      const double x = R[tri(j, k)], y = r[k];
      R[tri(j, k)] = c * x + sn * y; r[k] = c * y - sn * x;
    }
  }
}

// fold the triangle of lane + o into this lane's (a shuffle tree: lane 0 ends with the warp's triangle).  Every lane
// folds at once, so the rows go last to first: folding row i changes rows i .. 8 only, and row i of the source lane is
// still its own when it is read.
__device__ __forceinline__ void givens_merge_down(double (&R)[45], int o) {
#pragma unroll
  for (int i = 8; i >= 0; --i) {
    double r[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) r[k] = k < i ? 0.0 : __shfl_down_sync(0xffffffffu, R[tri(i, k)], o);
    givens_fold(R, r, i);
  }
}

template <int KIND>
__device__ __noinline__ void local_model(Shared& s, double s1, double c1x, double c1y, double s2, double c2x, double c2y);

// the local estimator on the inliers of s.best: eight-point F, normalised DLT H, or the mean translation; s.local
template <int KIND>
__device__ void local_estimate(const float4* pts, const int* list, int n, double thr, Shared& s) {
  double best[9];
  for (int i = 0; i < 9; ++i) best[i] = s.best[i];
  {                                                      // moments: count, sum x1, y1, x2, y2
    double v[5] = {0, 0, 0, 0, 0};
    for (int i = threadIdx.x; i < n; i += kThreads) {
      const float4 p = point<KIND>(pts, list, i);
      if (residual<KIND>(best, p) <= thr) { v[0] += 1.0; v[1] += p.x; v[2] += p.y; v[3] += p.z; v[4] += p.w; }
    }
    block_reduce<5>(v, s);
  }
  const double cnt = s.tot[0];
  const double c1x = s.tot[1] / cnt, c1y = s.tot[2] / cnt, c2x = s.tot[3] / cnt, c2y = s.tot[4] / cnt;
  if (KIND == kKindW) {
    if (threadIdx.x == 0) { s.local[0] = c2x - c1x; s.local[1] = c2y - c1y; }
    __syncthreads();
    return;
  }
  {                                                      // RMS distances to the centroids
    double v[2] = {0, 0};
    for (int i = threadIdx.x; i < n; i += kThreads) {
      const float4 p = point<KIND>(pts, list, i);
      if (residual<KIND>(best, p) <= thr) {
        v[0] += (p.x - c1x) * (p.x - c1x) + (p.y - c1y) * (p.y - c1y);
        v[1] += (p.z - c2x) * (p.z - c2x) + (p.w - c2y) * (p.w - c2y);
      }
    }
    block_reduce<2>(v, s);
  }
  const double s1 = sqrt(2.0) / sqrt(s.tot[0] / cnt), s2 = sqrt(2.0) / sqrt(s.tot[1] / cnt);
  {                                                      // R factor of the normalised rows
    double R[45];
#pragma unroll
    for (int k = 0; k < 45; ++k) R[k] = 0.0;
    for (int i = threadIdx.x; i < n; i += kThreads) {
      const float4 p = point<KIND>(pts, list, i);
      if (!(residual<KIND>(best, p) <= thr)) continue;
      const double a0 = (p.x - c1x) * s1, a1 = (p.y - c1y) * s1, d0 = (p.z - c2x) * s2, d1 = (p.w - c2y) * s2;
      if (KIND == kKindF) {
        double r[9] = {d0 * a0, d0 * a1, d0, d1 * a0, d1 * a1, d1, a0, a1, 1.0};
        givens_fold(R, r, 0);
      } else {
        double r[9] = {-a0, -a1, -1.0, 0.0, 0.0, 0.0, a0 * d0, a1 * d0, d0};
        double q[9] = {0.0, 0.0, 0.0, -a0, -a1, -1.0, a0 * d1, a1 * d1, d1};
        givens_fold(R, r, 0);
        givens_fold(R, q, 3);
      }
    }
    for (int o = 16; o > 0; o >>= 1) givens_merge_down(R, o);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (lane == 0)
#pragma unroll
      for (int k = 0; k < 45; ++k) s.red[wid][k] = R[k];
    __syncthreads();
  }
  if (threadIdx.x == 0) local_model<KIND>(s, s1, c1x, c1y, s2, c2x, c2y);
  __syncthreads();
}

// the leader's part of the local step: the warps' R factors (s.red) folded in warp order, the right singular vector of
// the smallest singular value of R, the rank-2 constraint for F, denormalised into s.local
template <int KIND>
__device__ __noinline__ void local_model(Shared& s, double s1, double c1x, double c1y, double s2, double c2x, double c2y) {
  {
    double R[45];
    for (int k = 0; k < 45; ++k) R[k] = s.red[0][k];
    for (int w = 1; w < kWarps; ++w)
      for (int i = 0; i < 9; ++i) {
        double r[9];
        for (int k = 0; k < 9; ++k) r[k] = k < i ? 0.0 : s.red[w][tri(i, k)];
        givens_fold(R, r, i);
      }
    for (int u = 0; u < 9; ++u)
      for (int w = 0; w < 9; ++w) s.G[9 * u + w] = w < u ? 0.0 : R[tri(u, w)];
    const int mn9 = one_sided_jacobi_mem(s.G, s.GV, 9);
    double f[9];
    for (int i = 0; i < 9; ++i) f[i] = s.GV[9 * i + mn9];
    for (int i = 0; i < 9; ++i) s.lnull[i] = f[i];
    s.lnorm[0] = s1; s.lnorm[1] = c1x; s.lnorm[2] = c1y; s.lnorm[3] = s2; s.lnorm[4] = c2x; s.lnorm[5] = c2y;
    if (KIND == kKindF) {
      double A[3][3], V[3][3];                           // rank 2: the smallest singular value set to zero
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) A[r][c] = f[3 * r + c];
      one_sided_jacobi<3>(A, V);
      int mn = 0;
      double nmin = A[0][0] * A[0][0] + A[1][0] * A[1][0] + A[2][0] * A[2][0];
      for (int j = 1; j < 3; ++j) {
        const double nj = A[0][j] * A[0][j] + A[1][j] * A[1][j] + A[2][j] * A[2][j];
        if (nj < nmin) { nmin = nj; mn = j; }
      }
      double Fn[3][3];
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) {
          double t = 0.0;
          for (int j = 0; j < 3; ++j)
            if (j != mn) t += A[r][j] * V[c][j];
          Fn[r][c] = t;
        }
      // F = T2' Fn T1
      double T1[3][3] = {{s1, 0.0, -s1 * c1x}, {0.0, s1, -s1 * c1y}, {0.0, 0.0, 1.0}};
      double T2[3][3] = {{s2, 0.0, -s2 * c2x}, {0.0, s2, -s2 * c2y}, {0.0, 0.0, 1.0}};
      double Y[3][3];
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) Y[r][c] = Fn[r][0] * T1[0][c] + Fn[r][1] * T1[1][c] + Fn[r][2] * T1[2][c];
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) s.local[3 * r + c] = T2[0][r] * Y[0][c] + T2[1][r] * Y[1][c] + T2[2][r] * Y[2][c];
    } else {
      denormalize_h(f, s1, c1x, c1y, s2, c2x, c2y, s.local);
    }
  }
}

struct Report {
  int success;
  long long num_inliers;
  int trials, rounds, have_model;
};

// LORANSAC<Estimator, LocalEstimator>::Estimate for one pair and one kind, the whole CTA; the best model is in s.best
template <int KIND>
__device__ Report loransac(const Args& a, int pair, const float4* pts, const int* list, int n, long long max_trials, Shared& s) {
  constexpr int K = KIND == kKindF ? kSevenPointSamples : KIND == kKindH ? kHomographySamples : kTranslationSamples;
  constexpr int LK = KIND == kKindF ? kEightPointSamples : K;
  Report rep = {0, 0, 0, 0, 0};
  __syncthreads();
  if (n < K) return rep;
  if (threadIdx.x == 0) {
    s.best_n = 0; s.best_sum = 1.7976931348623157e308; s.have_best = 0; s.dyn = max_trials;
    s.abort_ = 0; s.trials = 0; s.rounds = 0;
  }
  __syncthreads();
  for (long long trial = 0; trial < max_trials; ++trial) {
    __syncthreads();                           // every thread has read the previous sample's shared state
    if (threadIdx.x == 0) {
      draw_sample(a.seed, (u64)pair, (u64)KIND, (u64)trial, (unsigned)n, K, s.idx);
      float4 p[K];
      for (int i = 0; i < K; ++i) p[i] = point<KIND>(pts, list, s.idx[i]);
      if (KIND == kKindF) {
        s.nm = seven_point(p, s.models);
      } else if (KIND == kKindH) {
        s.nm = homography_minimal(p, s.models[0]);
      } else {
        s.models[0][0] = (double)p[0].z - (double)p[0].x;
        s.models[0][1] = (double)p[0].w - (double)p[0].y;
        s.nm = 1;
      }
      s.trials = (int)(trial + 1);
    }
    __syncthreads();
    const int nm = s.nm;
    if (nm == 0) continue;
    score<KIND>(s.models, nm, pts, list, n, a.thr, s);
    double cnt[3], sum[3];
    for (int k = 0; k < 3; ++k) { cnt[k] = s.tot[k]; sum[k] = s.tot[3 + k]; }
    __syncthreads();
    for (int mi = 0; mi < nm; ++mi) {
      if (threadIdx.x == 0) {
        const long long ni = (long long)cnt[mi];
        const bool better = ni > s.best_n || (ni == s.best_n && sum[mi] < s.best_sum);
        s.flag_better = better;
        s.flag_lo = better && ni > K && ni >= LK;
        if (better) {
          s.best_n = ni; s.best_sum = sum[mi]; s.have_best = 1;
          for (int i = 0; i < 9; ++i) s.best[i] = s.models[mi][i];
        }
      }
      __syncthreads();
      const int better = s.flag_better, lo = s.flag_lo;
      if (lo) {
        for (int r = 0; r < kMaxNumLocalTrials; ++r) {
          __syncthreads();
          const long long prev = s.best_n;
          local_estimate<KIND>(pts, list, n, a.thr, s);
          score<KIND>(&s.local, 1, pts, list, n, a.thr, s);
          if (threadIdx.x == 0) {
            const long long li = (long long)s.tot[0];
            const double ls = s.tot[3];
            if (li > s.best_n || (li == s.best_n && ls < s.best_sum)) {
              s.best_n = li; s.best_sum = ls;
              for (int i = 0; i < 9; ++i) s.best[i] = s.local[i];
            }
            s.rounds += 1;
            s.flag_stop = s.best_n <= prev;
          }
          __syncthreads();
          if (s.flag_stop) break;
        }
      }
      if (threadIdx.x == 0) {
        if (better) s.dyn = compute_num_trials(s.best_n, n, K, a.confidence, a.multiplier);
        if (trial >= s.dyn && trial >= a.min_trials) s.abort_ = 1;
      }
      __syncthreads();
      if (s.abort_) break;
    }
    if (s.abort_) break;
  }
  __syncthreads();
  rep.success = s.best_n >= K;
  rep.num_inliers = s.best_n;
  rep.trials = s.trials;
  rep.rounds = s.rounds;
  rep.have_model = s.have_best;
  return rep;
}

// the stored form of F or H: unit Frobenius norm, the largest-magnitude entry positive (the first on a tie)
__device__ void store_model(const double* m, int have, double* out) {
  if (!have) {
    for (int i = 0; i < 9; ++i) out[i] = 0.0;
    return;
  }
  double nrm = 0.0;
  for (int i = 0; i < 9; ++i) nrm += m[i] * m[i];
  nrm = sqrt(nrm);
  int big = 0;
  for (int i = 1; i < 9; ++i)
    if (fabs(m[i]) > fabs(m[big])) big = i;
  const double sg = m[big] / nrm < 0.0 ? -1.0 : 1.0;
  for (int i = 0; i < 9; ++i) out[i] = sg * (m[i] / nrm);
}

__global__ void k_gather(int R, const long long* __restrict__ mptr, const int2* __restrict__ pairs,
                         const long long* __restrict__ kp_ptr, const float2* __restrict__ kps, const uint2* __restrict__ m,
                         float4* __restrict__ pts) {
  const int p = blockIdx.x;
  if (p >= R) return;
  const long long o1 = kp_ptr[pairs[p].x], o2 = kp_ptr[pairs[p].y];
  for (long long i = mptr[p] + threadIdx.x; i < mptr[p + 1]; i += blockDim.x) {
    const uint2 mm = m[i];
    const float2 a = kps[o1 + mm.x], b = kps[o2 + mm.y];
    pts[i] = make_float4(a.x, a.y, b.x, b.y);
  }
}

__global__ void __launch_bounds__(kThreads) k_verify(Args a) {
  __shared__ Shared s;
  const int p = blockIdx.x;
  if (p >= a.R) return;
  const long long base = a.mptr[p];
  const int n = (int)(a.mptr[p + 1] - base);
  const float4* pts = a.pts + base;
  int* list = a.inl_idx + base;
  double Fm[9], Hm[9];
  if (n < a.min_num_inliers) {
    if (threadIdx.x == 0) {
      a.config[p] = kUndefined;
      for (int i = 0; i < 9; ++i) { a.F[9 * p + i] = 0.0; a.H[9 * p + i] = 0.0; }
      a.count[p] = 0;
      for (int k = 0; k < 3; ++k) { a.trials[3 * p + k] = 0; a.rounds[3 * p + k] = 0; }
    }
    return;
  }
  const Report fr = loransac<kKindF>(a, p, pts, nullptr, n, a.max_trials[kKindF], s);
  for (int i = 0; i < 9; ++i) Fm[i] = s.best[i];
  __syncthreads();
  const Report hr = loransac<kKindH>(a, p, pts, nullptr, n, a.max_trials[kKindH], s);
  for (int i = 0; i < 9; ++i) Hm[i] = s.best[i];
  __syncthreads();
  int config;
  const long long mi = a.min_num_inliers;
  if ((!fr.success && !hr.success) || (fr.num_inliers < mi && hr.num_inliers < mi)) {
    config = kDegenerate;
  } else {
    const double ratio = fr.num_inliers ? (double)hr.num_inliers / (double)fr.num_inliers : INFINITY;
    config = ratio > a.max_H_ratio ? kPlanarOrPanoramic : kUncalibrated;
  }
  // F's inliers in match order (a stable block-wide compaction)
  long long cnt = 0;
  if (config != kDegenerate && fr.success) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (int c0 = 0; c0 < n; c0 += kThreads) {
      const int i = c0 + threadIdx.x;
      const bool in = i < n && residual<kKindF>(Fm, pts[i]) <= a.thr;
      const unsigned ball = __ballot_sync(0xffffffffu, in);
      if (lane == 0) s.wsum[wid] = __popc(ball);
      __syncthreads();
      int off = 0;
      for (int w = 0; w < wid; ++w) off += s.wsum[w];
      int total = 0;
      for (int w = 0; w < kWarps; ++w) total += s.wsum[w];
      if (in) list[cnt + off + __popc(ball & ((1u << lane) - 1u))] = i;
      cnt += total;
      __syncthreads();
    }
  }
  int wtrials = 0, wrounds = 0;
  if (config != kDegenerate && fr.success && a.detect_watermark && cnt > 0) {
    // DetectWatermark: F's inliers outside the inner box of both images
    const int2 sz1 = a.sizes[2 * p], sz2 = a.sizes[2 * p + 1];
    const double m1 = a.wm_border * sqrt((double)sz1.x * sz1.x + (double)sz1.y * sz1.y);
    const double m2 = a.wm_border * sqrt((double)sz2.x * sz2.x + (double)sz2.y * sz2.y);
    double v[1] = {0.0};
    for (int j = threadIdx.x; j < cnt; j += kThreads) {
      const float4 q = pts[list[j]];
      const bool in1 = q.x >= m1 && q.x <= sz1.x - m1 && q.y >= m1 && q.y <= sz1.y - m1;
      const bool in2 = q.z >= m2 && q.z <= sz2.x - m2 && q.w >= m2 && q.w <= sz2.y - m2;
      if (!in1 && !in2) v[0] += 1.0;
    }
    block_reduce<1>(v, s);
    const double border = s.tot[0];
    __syncthreads();
    if (!(border / (double)cnt < a.wm_ratio)) {
      const Report wr = loransac<kKindW>(a, p, pts, list, (int)cnt, a.max_trials[kKindW], s);
      wtrials = wr.trials; wrounds = wr.rounds;
      if ((double)wr.num_inliers / (double)cnt >= a.wm_ratio) config = kWatermark;
    }
  }
  if (threadIdx.x == 0) {
    a.config[p] = config;
    store_model(Fm, fr.have_model, a.F + 9 * p);
    store_model(Hm, hr.have_model, a.H + 9 * p);
    a.count[p] = cnt;
    a.trials[3 * p] = fr.trials; a.trials[3 * p + 1] = hr.trials; a.trials[3 * p + 2] = wtrials;
    a.rounds[3 * p] = fr.rounds; a.rounds[3 * p + 1] = hr.rounds; a.rounds[3 * p + 2] = wrounds;
  }
}

__global__ void k_compact(int R, const long long* __restrict__ mptr, const long long* __restrict__ iptr,
                          const int* __restrict__ inl_idx, const uint2* __restrict__ m, uint2* __restrict__ out) {
  const int p = blockIdx.x;
  if (p >= R) return;
  const long long b = mptr[p], o = iptr[p], n = iptr[p + 1] - iptr[p];
  for (long long j = threadIdx.x; j < n; j += blockDim.x) out[o + j] = m[b + inl_idx[b + j]];
}

// psfm_verification_local_model: one local step of k_verify on one point stream, through the same Shared layout;
// out = the normalised null vector (9), (s1, c1x, c1y, s2, c2x, c2y) (6), the denormalised local model (9)
template <int KIND>
__global__ void __launch_bounds__(kThreads) k_local_model(const float4* __restrict__ pts, int n,
                                                           const double* __restrict__ best, double thr, double* out) {
  __shared__ Shared s;
  if (threadIdx.x < 9) s.best[threadIdx.x] = best[threadIdx.x];
  __syncthreads();
  local_estimate<KIND>(pts, nullptr, n, thr, s);
  if (threadIdx.x < 9) {
    out[threadIdx.x] = s.lnull[threadIdx.x];
    out[15 + threadIdx.x] = s.local[threadIdx.x];
  }
  if (threadIdx.x < 6) out[9 + threadIdx.x] = s.lnorm[threadIdx.x];
}

// psfm_verification_minimal / psfm_verification_cubic: one sample (one cubic) per thread through the functions
// k_verify calls
constexpr int kMinimalBlock = 128;

template <int KIND>
__global__ void __launch_bounds__(kMinimalBlock) k_minimal(const float4* __restrict__ pts, long long count,
                                                           double* __restrict__ models, int* __restrict__ num_models) {
  const long long t = blockIdx.x * (long long)kMinimalBlock + threadIdx.x;
  if (t >= count) return;
  constexpr int K = KIND == kKindF ? kSevenPointSamples : kHomographySamples;
  float4 p[K];
  for (int i = 0; i < K; ++i) p[i] = pts[K * t + i];
  double m[3][9];
  const int nm = KIND == kKindF ? seven_point(p, m) : homography_minimal(p, m[0]);
  constexpr int NM = KIND == kKindF ? 3 : 1;
  for (int k = 0; k < NM; ++k)
    for (int i = 0; i < 9; ++i) models[(NM * t + k) * 9 + i] = k < nm ? m[k][i] : 0.0;
  num_models[t] = nm;
}

__global__ void __launch_bounds__(kMinimalBlock) k_cubic(const double* __restrict__ coeffs, long long count,
                                                         double* __restrict__ roots, int* __restrict__ num_roots) {
  const long long t = blockIdx.x * (long long)kMinimalBlock + threadIdx.x;
  if (t >= count) return;
  const double* c = coeffs + 4 * t;
  double x[3] = {0.0, 0.0, 0.0};
  num_roots[t] = cubic_real_roots(c[0], c[1], c[2], c[3], x);
  for (int i = 0; i < 3; ++i) roots[3 * t + i] = x[i];
}

}  // namespace

extern "C" void psfm_verification_default_options(psfm_verification_options* o) {
  if (!o) return;
  o->max_error = 4.0;
  o->confidence = 0.999;
  o->max_num_trials = 20000;
  o->min_num_trials = 0;
  o->min_inlier_ratio = 0.1;
  o->min_num_inliers = 15;
  o->dyn_num_trials_multiplier = 3.0;
  o->max_H_inlier_ratio = 0.8;
  o->detect_watermark = 1;
  o->watermark_min_inlier_ratio = 0.7;
  o->watermark_border_size = 0.1;
  o->random_seed = 0;
}

namespace {

// TwoViewGeometry::Options::Check() on the options (NULL: the defaults)
int check_options(const char* entry, const psfm_verification_options* opts, psfm_verification_options* o) {
  psfm_verification_default_options(o);
  if (opts) *o = *opts;
  if (!(o->max_error > 0 && o->confidence >= 0 && o->confidence <= 1 && o->min_inlier_ratio >= 0 &&
        o->min_inlier_ratio <= 1 && o->min_num_trials >= 0 && o->min_num_trials <= o->max_num_trials &&
        o->min_num_inliers >= 0 && o->dyn_num_trials_multiplier > 0 && o->max_H_inlier_ratio >= 0 &&
        o->watermark_min_inlier_ratio >= 0 && o->watermark_min_inlier_ratio <= 1 && o->watermark_border_size >= 0 &&
        o->watermark_border_size <= 1 && std::isfinite(o->max_error) && std::isfinite(o->dyn_num_trials_multiplier) &&
        std::isfinite(o->max_H_inlier_ratio)))
    return fail(entry, PSFM_ERR_INVALID, "options fail the TwoViewGeometry::Options Check()");
  return PSFM_OK;
}

// the pairs whose two cameras both have a prior focal length go to EstimateCalibrated, which is not supported
int check_prior_focal_length(const char* entry, int R, const int32_t* pair_images, const int32_t* image_camera,
                             const uint8_t* prior_focal_length) {
  if (prior_focal_length)
    for (int p = 0; p < R; ++p)
      if (prior_focal_length[image_camera[pair_images[2 * p]]] && prior_focal_length[image_camera[pair_images[2 * p + 1]]])
        return fail(entry, PSFM_ERR_UNSUPPORTED,
                    "both cameras of a pair have a prior focal length (EstimateCalibrated is not supported)");
  return PSFM_OK;
}

// The graph both entries verify.  Host copies of keypoint_ptr, pair_images and match_ptr; keypoints and matches on the
// host (uploaded here) unless `table` holds every array on the device already.
struct Graph {
  int num_images = 0, R = 0;
  long long K = 0, M = 0;
  const int64_t* keypoint_ptr = nullptr;
  const float* keypoints = nullptr;
  const int32_t* pair_images = nullptr;
  const int64_t* match_ptr = nullptr;
  const uint32_t* matches = nullptr;
  const psfm_match_table* table = nullptr;
};

// Everything after the host checks: gather, LORANSAC per pair, compaction and the copies back.
int verify_graph(const char* entry, std::chrono::steady_clock::time_point t0, long long launches0, const Graph& g,
                 const int32_t* image_camera, const int32_t* camera_size, const psfm_verification_options& o,
                 int32_t* config, double* F, double* E, double* H, int64_t* inlier_ptr, uint32_t* inlier_matches,
                 int32_t* pair_trials, psfm_verification_summary* summary) {
  const int R = g.R;
  const long long M = g.M;
  psfm_verification_summary sm;
  memset(&sm, 0, sizeof(sm));
  inlier_ptr[0] = 0;
  if (R == 0) {
    sm.host_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (summary) *summary = sm;
    return PSFM_OK;
  }
  int rc = require_device(entry);
  if (rc != PSFM_OK) return rc;
  std::vector<int> sizes(4 * (size_t)R);
  for (int p = 0; p < R; ++p)
    for (int k = 0; k < 2; ++k) {
      const int c = image_camera[g.pair_images[2 * p + k]];
      sizes[4 * p + 2 * k] = camera_size[2 * c];
      sizes[4 * p + 2 * k + 1] = camera_size[2 * c + 1];
    }
  sm.host_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  Event ev[4];
  DBuf<long long> up_kp_ptr, up_mptr, d_iptr, d_count;
  DBuf<float2> up_kps;
  DBuf<int2> up_pairs, d_sizes;
  DBuf<uint2> up_m, d_out;
  DBuf<float4> d_pts;
  DBuf<int> d_inl, d_config, d_trials, d_rounds;
  DBuf<double> d_F, d_H;
  const long long *kp_ptr, *mptr;
  const float2* kps;
  const int2* pairs;
  const uint2* m;
  if (g.table) {
    kp_ptr = g.table->d_keypoint_ptr.p; kps = g.table->keypoints.p; mptr = g.table->d_match_ptr.p;
    pairs = g.table->pairs.p; m = g.table->matches.p;
  } else {
    up_kp_ptr.alloc(g.num_images + 1); up_kps.alloc(g.K); up_mptr.alloc(R + 1); up_pairs.alloc(R); up_m.alloc(M);
    up_kp_ptr.upload(reinterpret_cast<const long long*>(g.keypoint_ptr), g.num_images + 1, nullptr);
    up_kps.upload(reinterpret_cast<const float2*>(g.keypoints), g.K, nullptr);
    up_mptr.upload(reinterpret_cast<const long long*>(g.match_ptr), R + 1, nullptr);
    up_pairs.upload(reinterpret_cast<const int2*>(g.pair_images), R, nullptr);
    up_m.upload(reinterpret_cast<const uint2*>(g.matches), M, nullptr);
    kp_ptr = up_kp_ptr.p; kps = up_kps.p; mptr = up_mptr.p; pairs = up_pairs.p; m = up_m.p;
  }
  d_iptr.alloc(R + 1); d_count.alloc(R); d_sizes.alloc(2 * (size_t)R); d_pts.alloc(M); d_inl.alloc(M);
  d_config.alloc(R); d_trials.alloc(3 * (size_t)R); d_rounds.alloc(3 * (size_t)R); d_F.alloc(9 * (size_t)R);
  d_H.alloc(9 * (size_t)R);
  d_sizes.upload(reinterpret_cast<const int2*>(sizes.data()), 2 * (size_t)R, nullptr);
  PSFM_CUDA(cudaEventRecord(ev[0], nullptr));
  k_gather<<<R, 256>>>(R, mptr, pairs, kp_ptr, kps, m, d_pts.p);
  PSFM_LAUNCH_CHECK();
  PSFM_CUDA(cudaEventRecord(ev[1], nullptr));
  Args a;
  a.R = R; a.mptr = mptr; a.pts = d_pts.p; a.sizes = d_sizes.p; a.inl_idx = d_inl.p; a.config = d_config.p;
  a.F = d_F.p; a.H = d_H.p; a.count = d_count.p; a.trials = d_trials.p; a.rounds = d_rounds.p;
  a.thr = o.max_error * o.max_error;
  a.confidence = o.confidence; a.multiplier = o.dyn_num_trials_multiplier;
  const int ks[3] = {kSevenPointSamples, kHomographySamples, kTranslationSamples};
  for (int k = 0; k < 3; ++k) {
    const double ratio = k == kKindW ? o.watermark_min_inlier_ratio : o.min_inlier_ratio;
    const long long cap = compute_num_trials((long long)(ratio * kCapNumSamples), kCapNumSamples, ks[k], o.confidence,
                                             o.dyn_num_trials_multiplier);
    a.max_trials[k] = std::min<long long>(o.max_num_trials, cap);
  }
  a.min_trials = o.min_num_trials; a.min_num_inliers = o.min_num_inliers; a.max_H_ratio = o.max_H_inlier_ratio;
  a.detect_watermark = o.detect_watermark != 0; a.wm_ratio = o.watermark_min_inlier_ratio;
  a.wm_border = o.watermark_border_size; a.seed = (u64)o.random_seed;
  k_verify<<<R, kThreads>>>(a);
  PSFM_LAUNCH_CHECK();
  PSFM_CUDA(cudaEventRecord(ev[2], nullptr));
  std::vector<long long> cnt(R);
  PSFM_CUDA(cudaMemcpy(cnt.data(), d_count.p, sizeof(long long) * R, cudaMemcpyDeviceToHost));
  for (int p = 0; p < R; ++p) inlier_ptr[p + 1] = inlier_ptr[p] + cnt[p];
  const long long N = inlier_ptr[R];
  d_iptr.upload(reinterpret_cast<const long long*>(inlier_ptr), R + 1, nullptr);
  d_out.alloc(N);
  k_compact<<<R, 256>>>(R, mptr, d_iptr.p, d_inl.p, m, d_out.p);
  PSFM_LAUNCH_CHECK();
  PSFM_CUDA(cudaEventRecord(ev[3], nullptr));
  PSFM_CUDA(cudaEventSynchronize(ev[3]));
  if (N) PSFM_CUDA(cudaMemcpy(inlier_matches, d_out.p, sizeof(uint2) * N, cudaMemcpyDeviceToHost));
  PSFM_CUDA(cudaMemcpy(config, d_config.p, sizeof(int) * R, cudaMemcpyDeviceToHost));
  PSFM_CUDA(cudaMemcpy(F, d_F.p, sizeof(double) * 9 * R, cudaMemcpyDeviceToHost));
  PSFM_CUDA(cudaMemcpy(H, d_H.p, sizeof(double) * 9 * R, cudaMemcpyDeviceToHost));
  memset(E, 0, sizeof(double) * 9 * (size_t)R);
  std::vector<int> tr(3 * (size_t)R), rd(3 * (size_t)R);
  PSFM_CUDA(cudaMemcpy(tr.data(), d_trials.p, sizeof(int) * 3 * R, cudaMemcpyDeviceToHost));
  PSFM_CUDA(cudaMemcpy(rd.data(), d_rounds.p, sizeof(int) * 3 * R, cudaMemcpyDeviceToHost));
  if (pair_trials) memcpy(pair_trials, tr.data(), sizeof(int) * 3 * (size_t)R);
  for (int p = 0; p < R; ++p) {
    for (int k = 0; k < 3; ++k) {
      sm.num_trials[k] += tr[3 * p + k];
      sm.num_local_rounds[k] += rd[3 * p + k];
    }
    if (config[p] >= 0 && config[p] < 8) sm.num_config[config[p]] += 1;
  }
  for (int k = 0; k < 3; ++k) sm.num_trials_scored[k] = sm.num_trials[k];
  float ms[3];
  for (int i = 0; i < 3; ++i) PSFM_CUDA(cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]));
  sm.gather_ms = ms[0]; sm.ransac_ms = ms[1]; sm.compact_ms = ms[2];
  sm.num_launches = g_launch_count.load() - launches0;
  if (summary) *summary = sm;
  return PSFM_OK;
}

}  // namespace

extern "C" int psfm_verify_two_view_geometries(int32_t num_images, const int64_t* keypoint_ptr, const float* keypoints,
                                               const int32_t* image_camera, int32_t num_cameras, const int32_t* camera_size,
                                               const uint8_t* prior_focal_length, int64_t num_pairs,
                                               const int32_t* pair_images, const int64_t* match_ptr, const uint32_t* matches,
                                               const psfm_verification_options* opts, int32_t* config, double* F, double* E,
                                               double* H, int64_t* inlier_ptr, uint32_t* inlier_matches,
                                               int32_t* pair_trials, psfm_verification_summary* summary) {
  return guard("psfm_verify_two_view_geometries", [&]() -> int {
    const auto t0 = std::chrono::steady_clock::now();
    const long long launches0 = g_launch_count.load();
    const char* entry = "psfm_verify_two_view_geometries";
    int rc = check_sizes(entry, num_images, num_cameras, num_pairs);
    if (rc != PSFM_OK) return rc;
    if (!keypoint_ptr || (num_images > 0 && !image_camera) || (num_cameras > 0 && !camera_size) ||
        (num_pairs > 0 && (!pair_images || !match_ptr || !config || !F || !E || !H)) || !inlier_ptr)
      return fail(entry, PSFM_ERR_INVALID, "null argument");
    psfm_verification_options o;
    if ((rc = check_options(entry, opts, &o)) != PSFM_OK) return rc;
    const int Fimg = num_images, R = (int)num_pairs;
    if ((rc = check_keypoint_ptr(entry, Fimg, keypoint_ptr)) != PSFM_OK) return rc;
    const long long K = keypoint_ptr[Fimg];
    if (K > 0 && !keypoints) return fail(entry, PSFM_ERR_INVALID, "null argument");
    if ((rc = check_image_cameras(entry, Fimg, image_camera, num_cameras)) != PSFM_OK) return rc;
    if ((rc = check_camera_sizes(entry, num_cameras, camera_size)) != PSFM_OK) return rc;
    long long M = 0;
    if (R > 0) {
      if ((rc = check_match_ptr(entry, "match_ptr", R, match_ptr)) != PSFM_OK) return rc;
      for (int p = 0; p < R; ++p)
        if (match_ptr[p + 1] - match_ptr[p] > 0x7fffffffLL)
          return fail(entry, PSFM_ERR_UNSUPPORTED, "a pair with 2^31 or more matches");
      if ((rc = check_pair_images(entry, R, pair_images, Fimg)) != PSFM_OK) return rc;
      if ((rc = check_distinct_pairs(entry, R, pair_images)) != PSFM_OK) return rc;
      M = match_ptr[R];
      if (M > 0 && (!matches || !inlier_matches)) return fail(entry, PSFM_ERR_INVALID, "null argument");
      if ((rc = check_match_keypoints(entry, R, pair_images, keypoint_ptr, match_ptr, matches)) != PSFM_OK) return rc;
      if ((rc = check_prior_focal_length(entry, R, pair_images, image_camera, prior_focal_length)) != PSFM_OK) return rc;
    }
    Graph g;
    g.num_images = Fimg; g.R = R; g.K = K; g.M = M;
    g.keypoint_ptr = keypoint_ptr; g.keypoints = keypoints; g.pair_images = pair_images; g.match_ptr = match_ptr;
    g.matches = matches;
    return verify_graph(entry, t0, launches0, g, image_camera, camera_size, o, config, F, E, H, inlier_ptr, inlier_matches,
                        pair_trials, summary);
  });
}

extern "C" int psfm_match_table_verify(const psfm_match_table* t, const int32_t* image_camera, int32_t num_cameras,
                                       const int32_t* camera_size, const uint8_t* prior_focal_length,
                                       const psfm_verification_options* opts, int32_t* config, double* F, double* E,
                                       double* H, int64_t* inlier_ptr, uint32_t* inlier_matches, int32_t* pair_trials,
                                       psfm_verification_summary* summary) {
  return guard("psfm_match_table_verify", [&]() -> int {
    const auto t0 = std::chrono::steady_clock::now();
    const long long launches0 = g_launch_count.load();
    const char* entry = "psfm_match_table_verify";
    if (!t) return fail(entry, PSFM_ERR_INVALID, "null argument");
    int rc = check_sizes(entry, t->num_images, num_cameras, t->num_pairs);
    if (rc != PSFM_OK) return rc;
    const int R = (int)t->num_pairs;
    if ((t->num_images > 0 && !image_camera) || (num_cameras > 0 && !camera_size) ||
        (R > 0 && (!config || !F || !E || !H)) || !inlier_ptr || (t->num_matches > 0 && !inlier_matches))
      return fail(entry, PSFM_ERR_INVALID, "null argument");
    psfm_verification_options o;
    if ((rc = check_options(entry, opts, &o)) != PSFM_OK) return rc;
    if ((rc = check_image_cameras(entry, t->num_images, image_camera, num_cameras)) != PSFM_OK) return rc;
    if ((rc = check_camera_sizes(entry, num_cameras, camera_size)) != PSFM_OK) return rc;
    for (int p = 0; p < R; ++p)
      if (t->match_ptr[p + 1] - t->match_ptr[p] > 0x7fffffffLL)
        return fail(entry, PSFM_ERR_UNSUPPORTED, "a pair with 2^31 or more matches");
    if ((rc = check_prior_focal_length(entry, R, t->pair_images.data(), image_camera, prior_focal_length)) != PSFM_OK)
      return rc;
    Graph g;
    g.num_images = t->num_images; g.R = R; g.K = t->num_keypoints; g.M = t->num_matches;
    g.keypoint_ptr = reinterpret_cast<const int64_t*>(t->keypoint_ptr.data());
    g.match_ptr = reinterpret_cast<const int64_t*>(t->match_ptr.data());
    g.pair_images = t->pair_images.data();
    g.table = t;
    return verify_graph(entry, t0, launches0, g, image_camera, camera_size, o, config, F, E, H, inlier_ptr, inlier_matches,
                        pair_trials, summary);
  });
}

extern "C" int psfm_verification_local_model(int32_t kind, const float* points, int64_t n, const double* best,
                                             double max_squared_error, double* null_vector, double* normalization,
                                             double* local_model) {
  const char* entry = "psfm_verification_local_model";
  return guard(entry, [&]() -> int {
    if (!points || !best || !null_vector || !normalization || !local_model) return fail(entry, PSFM_ERR_INVALID, "null argument");
    if (kind != kKindF && kind != kKindH) return fail(entry, PSFM_ERR_INVALID, "kind must be 0 (F) or 1 (H)");
    if (n < 1 || n > 0x7fffffffLL) return fail(entry, PSFM_ERR_INVALID, "needs 1 <= n < 2^31");
    if (!(max_squared_error >= 0.0)) return fail(entry, PSFM_ERR_INVALID, "max_squared_error must be >= 0");
    const int rc = require_device(entry);
    if (rc != PSFM_OK) return rc;
    DBuf<float4> d_pts;
    DBuf<double> d_best, d_out;
    d_pts.alloc(n); d_best.alloc(9); d_out.alloc(24);
    d_pts.upload(reinterpret_cast<const float4*>(points), n, nullptr);
    d_best.upload(best, 9, nullptr);
    if (kind == kKindF) k_local_model<kKindF><<<1, kThreads>>>(d_pts.p, (int)n, d_best.p, max_squared_error, d_out.p);
    else k_local_model<kKindH><<<1, kThreads>>>(d_pts.p, (int)n, d_best.p, max_squared_error, d_out.p);
    PSFM_LAUNCH_CHECK();
    double out[24];
    PSFM_CUDA(cudaMemcpy(out, d_out.p, sizeof(out), cudaMemcpyDeviceToHost));
    memcpy(null_vector, out, 9 * sizeof(double));
    memcpy(normalization, out + 9, 6 * sizeof(double));
    memcpy(local_model, out + 15, 9 * sizeof(double));
    return PSFM_OK;
  });
}

extern "C" int psfm_verification_minimal(int32_t kind, const float* points, int64_t count, double* models,
                                         int32_t* num_models) {
  const char* entry = "psfm_verification_minimal";
  return guard(entry, [&]() -> int {
    if (!points || !models || !num_models) return fail(entry, PSFM_ERR_INVALID, "null argument");
    if (kind != kKindF && kind != kKindH) return fail(entry, PSFM_ERR_INVALID, "kind must be 0 (F) or 1 (H)");
    if (count < 1 || count > (1LL << 24)) return fail(entry, PSFM_ERR_INVALID, "needs 1 <= count <= 2^24");
    const int rc = require_device(entry);
    if (rc != PSFM_OK) return rc;
    const long long k = kind == kKindF ? kSevenPointSamples : kHomographySamples, nm = kind == kKindF ? 3 : 1;
    DBuf<float4> d_pts;
    DBuf<double> d_models;
    DBuf<int> d_num;
    d_pts.alloc(k * count); d_models.alloc(9 * nm * count); d_num.alloc(count);
    d_pts.upload(reinterpret_cast<const float4*>(points), k * count, nullptr);
    const unsigned grid = (unsigned)((count + kMinimalBlock - 1) / kMinimalBlock);
    if (kind == kKindF) k_minimal<kKindF><<<grid, kMinimalBlock>>>(d_pts.p, count, d_models.p, d_num.p);
    else k_minimal<kKindH><<<grid, kMinimalBlock>>>(d_pts.p, count, d_models.p, d_num.p);
    PSFM_LAUNCH_CHECK();
    PSFM_CUDA(cudaMemcpy(models, d_models.p, sizeof(double) * 9 * nm * count, cudaMemcpyDeviceToHost));
    PSFM_CUDA(cudaMemcpy(num_models, d_num.p, sizeof(int) * count, cudaMemcpyDeviceToHost));
    return PSFM_OK;
  });
}

extern "C" int psfm_verification_cubic(const double* coeffs, int64_t count, double* roots, int32_t* num_roots) {
  const char* entry = "psfm_verification_cubic";
  return guard(entry, [&]() -> int {
    if (!coeffs || !roots || !num_roots) return fail(entry, PSFM_ERR_INVALID, "null argument");
    if (count < 1 || count > (1LL << 24)) return fail(entry, PSFM_ERR_INVALID, "needs 1 <= count <= 2^24");
    const int rc = require_device(entry);
    if (rc != PSFM_OK) return rc;
    DBuf<double> d_c, d_x;
    DBuf<int> d_n;
    d_c.alloc(4 * count); d_x.alloc(3 * count); d_n.alloc(count);
    d_c.upload(coeffs, 4 * count, nullptr);
    k_cubic<<<(unsigned)((count + kMinimalBlock - 1) / kMinimalBlock), kMinimalBlock>>>(d_c.p, count, d_x.p, d_n.p);
    PSFM_LAUNCH_CHECK();
    PSFM_CUDA(cudaMemcpy(roots, d_x.p, sizeof(double) * 3 * count, cudaMemcpyDeviceToHost));
    PSFM_CUDA(cudaMemcpy(num_roots, d_n.p, sizeof(int) * count, cudaMemcpyDeviceToHost));
    return PSFM_OK;
  });
}
