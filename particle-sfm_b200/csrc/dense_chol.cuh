// dense_chol.cuh — the BA solver's blocked Cholesky (k_chol_blocked, ba_schur_explicit.cuh) on a dense SPD system,
// for units outside the BA solver.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace psfm {

constexpr int kDenseCholBlock = 32;     // k_chol_blocked's panel width (CB)

// Rows of the factor kept per panel: every row below the panel plus the solved rhs row.
__host__ __device__ inline int dense_chol_rmax(int ns) { return ns + 1; }
__host__ __device__ inline int dense_chol_panels(int ns) { return (ns + kDenseCholBlock - 1) / kDenseCholBlock; }

// Factors the ns x ns SPD matrix in A ([ns + 1][ns + 1] row-major, lda = ns + 1: the lower triangle of rows 0 .. ns-1,
// row ns the right-hand side b; A is overwritten) and solves A x = b into x [ns].  *fail = 1 on a non-positive pivot.
// bar: one device counter.  The factor L stays behind, panel p covering columns c0 = 32 p .. c1 = min(c0 + 32, ns):
//   L[i][c0 + k] = Ld[(p * 32 + (i - c0)) * 32 + k]          for c0 <= i < c1   (Ld: [panels][32][32], lower)
//   L[i][c0 + k] = Lp[(p * rmax + (i - c1)) * 32 + k]        for c1 <= i < ns   (Lp: [panels][rmax][32])
// Ld and Lp hold dense_chol_panels(ns) * 32 * 32 and dense_chol_panels(ns) * dense_chol_rmax(ns) * 32 doubles.
// One cooperative launch on stream st, counted by launch_count().
void dense_cholesky_launch(double* A, int ns, double* x, int* fail, unsigned int* bar, double* Lp, double* Ld,
                           cudaStream_t st);

}  // namespace psfm
