// dlt.cuh — the triangulation pieces shared by the two-view relative pose (two_view.cu), the multi-view DLT of
// init_geometry.cu and the triangulation of every registered image (triangulation.cu), and the null-vector solve of
// the verification's local step (verification.cu).  psfm_null_vectors (dlt.cu) runs each solver alone for the tests.
#pragma once
#include <cmath>

namespace psfm {

constexpr double kJacobiTol = 1e-15;     // columns p, q count as orthogonal when |a_p . a_q| <= tol |a_p| |a_q|

// one-sided (Hestenes) Jacobi: A <- A V with mutually orthogonal columns, V orthogonal; column j of A then has the
// norm of a singular value and V(:, j) is its right singular vector.  Working on A, not A'A, keeps the relative
// accuracy of the small singular values.
template <int N>
__device__ __forceinline__ void one_sided_jacobi(double (&A)[N][N], double (&V)[N][N]) {
#pragma unroll
  for (int i = 0; i < N; ++i)
#pragma unroll
    for (int j = 0; j < N; ++j) V[i][j] = i == j ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 40; ++sweep) {
    bool rotated = false;
#pragma unroll
    for (int p = 0; p < N - 1; ++p)
#pragma unroll
      for (int q = p + 1; q < N; ++q) {
        double alpha = 0.0, beta = 0.0, gamma = 0.0;
#pragma unroll
        for (int k = 0; k < N; ++k) {
          alpha += A[k][p] * A[k][p];
          beta += A[k][q] * A[k][q];
          gamma += A[k][p] * A[k][q];
        }
        if (!(fabs(gamma) > kJacobiTol * sqrt(alpha * beta))) continue;
        rotated = true;
        const double zeta = (beta - alpha) / (2.0 * gamma);
        const double t = (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
#pragma unroll
        for (int k = 0; k < N; ++k) {
          const double ap = A[k][p], aq = A[k][q];
          A[k][p] = c * ap - s * aq; A[k][q] = s * ap + c * aq;
          const double vp = V[k][p], vq = V[k][q];
          V[k][p] = c * vp - s * vq; V[k][q] = s * vp + c * vq;
        }
      }
    if (!rotated) break;
  }
}

// TriangulatePoint's null vector: the right singular vector of the smallest singular value of the 4 x 4 DLT matrix A
// (destroyed), before hnormalisation
__device__ __forceinline__ void dlt_null_vector_4x4(double (&A)[4][4], double (&v)[4]) {
  double V[4][4];
  one_sided_jacobi<4>(A, V);
  int best = 0;
  double bn = A[0][0] * A[0][0] + A[1][0] * A[1][0] + A[2][0] * A[2][0] + A[3][0] * A[3][0];
#pragma unroll
  for (int j = 1; j < 4; ++j) {
    const double nj = A[0][j] * A[0][j] + A[1][j] * A[1][j] + A[2][j] * A[2][j] + A[3][j] * A[3][j];
    if (nj < bn) { bn = nj; best = j; }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    double x = V[i][0];
#pragma unroll
    for (int j = 1; j < 4; ++j)
      if (j == best) x = V[i][j];
    v[i] = x;
  }
}

// TriangulatePoint's solve: dlt_null_vector_4x4, hnormalized
__device__ __forceinline__ void dlt_point_4x4(double (&A)[4][4], double* X) {
  double v[4];
  dlt_null_vector_4x4(A, v);
  X[0] = v[0] / v[3]; X[1] = v[1] / v[3]; X[2] = v[2] / v[3];
}

// eigenvector of the smallest eigenvalue of a symmetric N x N matrix (full storage, destroyed): cyclic Jacobi
template <int N>
__device__ __forceinline__ void smallest_eigenvector(double (&A)[N][N], double (&v)[N]) {
  double V[N][N];
#pragma unroll
  for (int i = 0; i < N; ++i)
#pragma unroll
    for (int j = 0; j < N; ++j) V[i][j] = i == j ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 30; ++sweep) {
    double off = 0.0, dia = 0.0;
#pragma unroll
    for (int i = 0; i < N; ++i) {
      dia += A[i][i] * A[i][i];
#pragma unroll
      for (int j = i + 1; j < N; ++j) off += A[i][j] * A[i][j];
    }
    if (!(off > 1e-34 * dia)) break;
#pragma unroll
    for (int p = 0; p < N - 1; ++p)
#pragma unroll
      for (int q = p + 1; q < N; ++q) {
        const double apq = A[p][q];
        if (apq == 0.0) continue;
        const double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
        const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
#pragma unroll
        for (int k = 0; k < N; ++k) {       // A <- A J (columns p, q)
          const double akp = A[k][p], akq = A[k][q];
          A[k][p] = c * akp - s * akq; A[k][q] = s * akp + c * akq;
        }
#pragma unroll
        for (int k = 0; k < N; ++k) {       // A <- J' A (rows p, q)
          const double apk = A[p][k], aqk = A[q][k];
          A[p][k] = c * apk - s * aqk; A[q][k] = s * apk + c * aqk;
        }
#pragma unroll
        for (int k = 0; k < N; ++k) {
          const double vkp = V[k][p], vkq = V[k][q];
          V[k][p] = c * vkp - s * vkq; V[k][q] = s * vkp + c * vkq;
        }
      }
  }
  int best = 0;
#pragma unroll
  for (int i = 1; i < N; ++i)
    if (A[i][i] < A[best][best]) best = i;
#pragma unroll
  for (int i = 0; i < N; ++i) {
    double x = V[i][0];
#pragma unroll
    for (int j = 1; j < N; ++j)
      if (j == best) x = V[i][j];
    v[i] = x;
  }
}

// one_sided_jacobi with A (n x n row-major, destroyed) and V (n x n) in memory, for a caller that cannot hold 2 n^2
// doubles in registers (the 9 x 9 R factors of verification.cu's local step); returns the index of the column of A V
// with the smallest norm, whose column of V is the right singular vector of A's smallest singular value
__device__ inline int one_sided_jacobi_mem(double* A, double* V, int n) {
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < n; ++j) V[i * n + j] = i == j ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 40; ++sweep) {
    bool rotated = false;
    for (int p = 0; p < n - 1; ++p)
      for (int q = p + 1; q < n; ++q) {
        double alpha = 0.0, beta = 0.0, gamma = 0.0;
        for (int k = 0; k < n; ++k) {
          alpha += A[k * n + p] * A[k * n + p];
          beta += A[k * n + q] * A[k * n + q];
          gamma += A[k * n + p] * A[k * n + q];
        }
        if (!(fabs(gamma) > kJacobiTol * sqrt(alpha * beta))) continue;
        rotated = true;
        const double zeta = (beta - alpha) / (2.0 * gamma);
        const double t = (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
        for (int k = 0; k < n; ++k) {
          const double ap = A[k * n + p], aq = A[k * n + q];
          A[k * n + p] = c * ap - s * aq; A[k * n + q] = s * ap + c * aq;
          const double vp = V[k * n + p], vq = V[k * n + q];
          V[k * n + p] = c * vp - s * vq; V[k * n + q] = s * vp + c * vq;
        }
      }
    if (!rotated) break;
  }
  int best = 0;
  double bn = 0.0;
  for (int j = 0; j < n; ++j) {
    double nj = 0.0;
    for (int k = 0; k < n; ++k) nj += A[k * n + j] * A[k * n + j];
    if (j == 0 || nj < bn) { bn = nj; best = j; }
  }
  return best;
}

// TriangulateMultiViewPoint's accumulation of one view: A += (P - r r' P)' (P - r r' P), r = (x, y, 1) / |(x, y, 1)|,
// P row-major 3 x 4
__device__ __forceinline__ void multi_view_accumulate(const double* P, double x, double y, double (&A)[4][4]) {
  const double inv = 1.0 / sqrt(x * x + y * y + 1.0);
  const double r[3] = {x * inv, y * inv, inv};
  double T[3][4];
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const double d = r[0] * P[c] + r[1] * P[4 + c] + r[2] * P[8 + c];
#pragma unroll
    for (int k = 0; k < 3; ++k) T[k][c] = P[4 * k + c] - r[k] * d;
  }
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) A[a][b] += T[0][a] * T[0][b] + T[1][a] * T[1][b] + T[2][a] * T[2][b];
}

// CalculateTriangulationAngle(c1, c2, X), law-of-cosines form
__device__ __forceinline__ double triangulation_angle(const double* c1, const double* c2, const double* X) {
  const double e0 = c1[0] - c2[0], e1 = c1[1] - c2[1], e2 = c1[2] - c2[2];
  const double b2 = e0 * e0 + e1 * e1 + e2 * e2;
  const double a0 = X[0] - c1[0], a1 = X[1] - c1[1], a2 = X[2] - c1[2];
  const double r1 = a0 * a0 + a1 * a1 + a2 * a2;
  const double d0 = X[0] - c2[0], d1 = X[1] - c2[1], d2 = X[2] - c2[2];
  const double r2 = d0 * d0 + d1 * d1 + d2 * d2;
  const double den = 2.0 * sqrt(r1 * r2);
  if (den == 0.0) return 0.0;
  const double a = fabs(acos((r1 + r2 - b2) / den)), b = M_PI - a;
  return b < a ? b : a;                        // std::min: a NaN angle stays NaN
}

}  // namespace psfm
