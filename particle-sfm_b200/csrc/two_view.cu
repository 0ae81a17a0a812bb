// two_view.cu — the relative pose of every verified image pair at once (SURVEY.md §8(f) row f-4).
//
// Reference: gcolmap's DatabaseCache::Load(..., relative_pose = true) (base/database_cache.cc:206-228) runs
// TwoViewGeometry::EstimateRelativePose (estimators/two_view_geometry.cc:172-239) as one ThreadPool task per pair:
// PoseFromEssentialMatrix (CALIBRATED, UNCALIBRATED with E = K2' F K1) or PoseFromHomographyMatrix (PLANAR,
// PANORAMIC, PLANAR_OR_PANORAMIC) over all inlier matches, CheckCheirality of every candidate, the median
// triangulation angle of the chosen candidate's points.  The restatement is oracle/two_view_oracle.py.
// Pipeline (R pairs, N inlier matches in total):
//   1. k_candidates  per pair: E or the normalised H, its 3 x 3 SVD (one-sided Jacobi), up to 4 candidates (R, t,
//                    max_depth = 1000 |R' t|, |R(:, 2)|)
//   2. k_cheirality  per match: both keypoints normalised from the keypoint table, per candidate the two-view DLT
//                    by a one-sided Jacobi SVD of the 4 x 4 matrix A itself (not of A'A, whose condition number
//                    is the square of A's: the tiny baselines of adjacent video frames put many points near
//                    max_depth), both depth tests; a 4-bit pass mask per match, and per (pair, candidate) counts by
//                    warp-aggregated integer atomics (deterministic)
//   3. k_choose      per pair: the candidate by the reference's tie rules, qvec, tvec, config, num_points3D
//   4. k_angles      per kept match of the chosen candidate: X again (same device function), its triangulation
//                    angle, compacted with its pair index
//   5. radix sorts   by angle, then stably by pair: every pair's angles in one sorted run
//   6. k_median      per pair: COLMAP's Median of its run
// Defined corners (the reference's own behaviour there is not usable):
//   * candidate order of an essential matrix: its SVD is not unique (sigma1 = sigma2 for an exact essential matrix;
//     u3 and v3 have no common sign when sigma3 = 0), so the order is fixed on the candidates: t has its
//     largest-magnitude component positive (ties to the lower index), R1 is the rotation of larger trace (equal
//     traces keep the SVD's order).  Only ties between candidate counts see it.
//   * no homography candidate keeps a point (a pure rotation has one candidate with t = 0, so max_depth = 0): the
//     reference reads an unset R; here candidate 0, tri_angle 0.
// Memory: 8 bytes per match (its indices) and 1 byte (its mask) during steps 2-4, 24 bytes per kept match in the
// sorts (the matches are released before them): about 21 GB at the DAVIS shape (636 M matches).
#include <algorithm>
#include <vector>

#include "dlt.cuh"
#include "pair_inputs.h"
#include "psfm_common.cuh"
#include "radix_sort.cuh"

namespace {

using namespace psfm;
typedef unsigned long long u64;

constexpr int kCand = 4;
constexpr int kCandStride = 16;          // doubles per candidate: R[9], t[3], max_depth, |R(:, 2)|, 2 unused
constexpr double kEps = 2.220446049250313e-16;
// TriangulatePoint with P1 = [I|0], P2 = [R|t] (c = R[9], t[3]), hnormalized
__device__ __forceinline__ void triangulate(const double* c, double x1, double y1, double x2, double y2, double* X) {
  double A[4][4] = {{-1.0, 0.0, x1, 0.0},
                    {0.0, -1.0, y1, 0.0},
                    {x2 * c[6] - c[0], x2 * c[7] - c[1], x2 * c[8] - c[2], x2 * c[11] - c[9]},
                    {y2 * c[6] - c[3], y2 * c[7] - c[4], y2 * c[8] - c[5], y2 * c[11] - c[10]}};
  dlt_point_4x4(A, X);
}

// CheckCheirality's two CalculateDepth tests of one correspondence
__device__ __forceinline__ bool in_front(const double* c, const double* X) {
  const double d1 = X[2];
  if (!(d1 > kEps && d1 < c[12])) return false;
  const double d2 = (c[6] * X[0] + c[7] * X[1] + c[8] * X[2] + c[11]) * c[13];
  return d2 > kEps && d2 < c[12];
}

__device__ __forceinline__ double det3(const double* M) {
  return M[0] * (M[4] * M[8] - M[5] * M[7]) - M[1] * (M[3] * M[8] - M[5] * M[6]) + M[2] * (M[3] * M[7] - M[4] * M[6]);
}

// singular values (descending, stable) of a row-major 3 x 3 M; with U and V (row-major, columns = singular vectors)
__device__ __forceinline__ void svd3(const double* M, double* sigma, double* U, double* V) {
  double A[3][3], Vj[3][3];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) A[r][c] = M[3 * r + c];
  one_sided_jacobi<3>(A, Vj);
  double s[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) s[j] = sqrt(A[0][j] * A[0][j] + A[1][j] * A[1][j] + A[2][j] * A[2][j]);
  int o[3] = {0, 1, 2};
  if (s[o[1]] > s[o[0]]) { const int x = o[0]; o[0] = o[1]; o[1] = x; }
  if (s[o[2]] > s[o[1]]) { const int x = o[1]; o[1] = o[2]; o[2] = x; }
  if (s[o[1]] > s[o[0]]) { const int x = o[0]; o[0] = o[1]; o[1] = x; }
  for (int j = 0; j < 3; ++j) {
    const int k = o[j];
    sigma[j] = s[k];
    for (int r = 0; r < 3; ++r) {
      V[3 * r + j] = Vj[r][k];
      if (U) U[3 * r + j] = A[r][k] / s[k];
    }
  }
}

__device__ __forceinline__ void store_candidate(double* c, const double* R, const double* t) {
  for (int i = 0; i < 9; ++i) c[i] = R[i];
  c[9] = t[0]; c[10] = t[1]; c[11] = t[2];
  const double r0 = R[0] * t[0] + R[3] * t[1] + R[6] * t[2], r1 = R[1] * t[0] + R[4] * t[1] + R[7] * t[2],
               r2 = R[2] * t[0] + R[5] * t[1] + R[8] * t[2];
  c[12] = 1000.0 * sqrt(r0 * r0 + r1 * r1 + r2 * r2);
  c[13] = sqrt(R[2] * R[2] + R[5] * R[5] + R[8] * R[8]);
  c[14] = c[15] = 0.0;
}

// DecomposeEssentialMatrix and the candidate order of the header comment; returns the number of candidates (4)
__device__ int essential_candidates(const double* E, double* cand) {
  double sigma[3], U[9], V[9];
  svd3(E, sigma, U, V);
  // u3 = u1 x u2: U is a rotation; its third column is free in sign when sigma3 = 0 anyway
  U[2] = U[3] * U[7] - U[6] * U[4];
  U[5] = U[6] * U[1] - U[0] * U[7];
  U[8] = U[0] * U[4] - U[3] * U[1];
  if (det3(V) < 0)
    for (int i = 0; i < 9; ++i) V[i] = -V[i];
  // R1 = U W V' = u1 v2' - u2 v1' + u3 v3',  R2 = U W' V' = u2 v1' - u1 v2' + u3 v3'
  double R1[9], R2[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      const double a = U[3 * r] * V[3 * c + 1] - U[3 * r + 1] * V[3 * c], b = U[3 * r + 2] * V[3 * c + 2];
      R1[3 * r + c] = a + b;
      R2[3 * r + c] = b - a;
    }
  double t[3] = {U[2], U[5], U[8]};
  const double n = sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
  int big = 0;
  for (int i = 0; i < 3; ++i) {
    t[i] /= n;
    if (fabs(t[i]) > fabs(t[big])) big = i;
  }
  if (t[big] < 0) { t[0] = -t[0]; t[1] = -t[1]; t[2] = -t[2]; }
  const double* Ra = R1;
  const double* Rb = R2;
  if (R2[0] + R2[4] + R2[8] > R1[0] + R1[4] + R1[8]) { Ra = R2; Rb = R1; }
  const double mt[3] = {-t[0], -t[1], -t[2]};
  store_candidate(cand, Ra, t);
  store_candidate(cand + kCandStride, Rb, t);
  store_candidate(cand + 2 * kCandStride, Ra, mt);
  store_candidate(cand + 3 * kCandStride, Rb, mt);
  return 4;
}

__device__ __forceinline__ double opposite_of_minor(const double* S, int row, int col) {
  const int c1 = col == 0 ? 1 : 0, c2 = col == 2 ? 1 : 2, r1 = row == 0 ? 1 : 0, r2 = row == 2 ? 1 : 2;
  return S[3 * r1 + c2] * S[3 * r2 + c1] - S[3 * r1 + c1] * S[3 * r2 + c2];
}

__device__ __forceinline__ double sign_of(double x) { return (double)((0.0 < x) - (x < 0.0)); }

// R = Hn (I - (2 / v) ts n'), t = R ts
__device__ __forceinline__ void homography_rotation(const double* Hn, const double* ts, const double* nv, double v, double* R,
                                                    double* t) {
  double B[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) B[3 * r + c] = (r == c ? 1.0 : 0.0) - (2.0 / v) * ts[r] * nv[c];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) R[3 * r + c] = Hn[3 * r] * B[c] + Hn[3 * r + 1] * B[3 + c] + Hn[3 * r + 2] * B[6 + c];
  for (int r = 0; r < 3; ++r) t[r] = R[3 * r] * ts[0] + R[3 * r + 1] * ts[1] + R[3 * r + 2] * ts[2];
}

// DecomposeHomographyMatrix (K = SIMPLE_PINHOLE (f, cx, cy)); returns the number of candidates (1 or 4)
__device__ int homography_candidates(const double* H, const double* k1, const double* k2, double* cand) {
  // Hn = K2^-1 H K1
  double HK[9], Hn[9];
  for (int r = 0; r < 3; ++r) {
    HK[3 * r] = H[3 * r] * k1[0];
    HK[3 * r + 1] = H[3 * r + 1] * k1[0];
    HK[3 * r + 2] = H[3 * r] * k1[1] + H[3 * r + 1] * k1[2] + H[3 * r + 2];
  }
  for (int c = 0; c < 3; ++c) {
    Hn[c] = (HK[c] - k2[1] * HK[6 + c]) / k2[0];
    Hn[3 + c] = (HK[3 + c] - k2[2] * HK[6 + c]) / k2[0];
    Hn[6 + c] = HK[6 + c];
  }
  double sigma[3], V[9];
  svd3(Hn, sigma, nullptr, V);
  for (int i = 0; i < 9; ++i) Hn[i] /= sigma[1];
  if (det3(Hn) < 0)
    for (int i = 0; i < 9; ++i) Hn[i] = -Hn[i];
  double S[9], inf = 0.0;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      S[3 * r + c] = Hn[r] * Hn[c] + Hn[3 + r] * Hn[3 + c] + Hn[6 + r] * Hn[6 + c] - (r == c ? 1.0 : 0.0);
      inf = fmax(inf, fabs(S[3 * r + c]));
    }
  if (inf < 1e-3) {
    const double z[3] = {0.0, 0.0, 0.0};
    store_candidate(cand, Hn, z);
    return 1;
  }
  const double M00 = opposite_of_minor(S, 0, 0), M11 = opposite_of_minor(S, 1, 1), M22 = opposite_of_minor(S, 2, 2);
  const double rt00 = sqrt(M00), rt11 = sqrt(M11), rt22 = sqrt(M22);
  const double e12 = sign_of(opposite_of_minor(S, 1, 2)), e02 = sign_of(opposite_of_minor(S, 0, 2)),
               e01 = sign_of(opposite_of_minor(S, 0, 1));
  int idx = 0;
  if (fabs(S[4]) > fabs(S[0])) idx = 1;
  if (fabs(S[8]) > fabs(S[4 * idx])) idx = 2;
  double np1[3], np2[3];
  if (idx == 0) {
    np1[0] = S[0]; np2[0] = S[0];
    np1[1] = S[1] + rt22; np2[1] = S[1] - rt22;
    np1[2] = S[2] + e12 * rt11; np2[2] = S[2] - e12 * rt11;
  } else if (idx == 1) {
    np1[0] = S[1] + rt22; np2[0] = S[1] - rt22;
    np1[1] = S[4]; np2[1] = S[4];
    np1[2] = S[5] - e02 * rt00; np2[2] = S[5] + e02 * rt00;
  } else {
    np1[0] = S[2] + e01 * rt11; np2[0] = S[2] - e01 * rt11;
    np1[1] = S[5] + rt00; np2[1] = S[5] - rt00;
    np1[2] = S[8]; np2[2] = S[8];
  }
  const double trS = S[0] + S[4] + S[8];
  const double v = 2.0 * sqrt(1.0 + trS - M00 - M11 - M22);
  const double esii = sign_of(S[4 * idx]);
  const double r = sqrt(2.0 + trS + v), nt = sqrt(2.0 + trS - v);
  const double l1 = sqrt(np1[0] * np1[0] + np1[1] * np1[1] + np1[2] * np1[2]),
               l2 = sqrt(np2[0] * np2[0] + np2[1] * np2[1] + np2[2] * np2[2]);
  double n1[3], n2[3], t1s[3], t2s[3];
  for (int i = 0; i < 3; ++i) { n1[i] = np1[i] / l1; n2[i] = np2[i] / l2; }
  const double half_nt = 0.5 * nt, esii_r = esii * r;
  for (int i = 0; i < 3; ++i) {
    t1s[i] = half_nt * (esii_r * n2[i] - nt * n1[i]);
    t2s[i] = half_nt * (esii_r * n1[i] - nt * n2[i]);
  }
  double R1[9], R2[9], t1[3], t2[3];
  homography_rotation(Hn, t1s, n1, v, R1, t1);
  homography_rotation(Hn, t2s, n2, v, R2, t2);
  const double m1[3] = {-t1[0], -t1[1], -t1[2]}, m2[3] = {-t2[0], -t2[1], -t2[2]};
  store_candidate(cand, R1, t1);
  store_candidate(cand + kCandStride, R1, m1);
  store_candidate(cand + 2 * kCandStride, R2, t2);
  store_candidate(cand + 3 * kCandStride, R2, m2);
  return 4;
}

__device__ __forceinline__ bool is_essential(int config) { return config == 2 || config == 3; }
__device__ __forceinline__ bool is_homography(int config) { return config >= 4 && config <= 6; }

__global__ void k_candidates(int R, const int* __restrict__ pair_images, const int* __restrict__ config,
                             const double* __restrict__ E, const double* __restrict__ F, const double* __restrict__ H,
                             const int* __restrict__ image_camera, const double* __restrict__ cameras, double* __restrict__ cand,
                             int* __restrict__ ncand) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= R) return;
  const int cfg = config[p];
  const double* k1 = cameras + 3 * image_camera[pair_images[2 * p]];
  const double* k2 = cameras + 3 * image_camera[pair_images[2 * p + 1]];
  double* c = cand + (size_t)p * kCand * kCandStride;
  int n = 0;
  if (is_essential(cfg)) {
    double M[9];
    if (cfg == 2) {
      for (int i = 0; i < 9; ++i) M[i] = E[9 * (size_t)p + i];
    } else {
      // E = K2' F K1
      const double* f = F + 9 * (size_t)p;
      double FK[9];
      for (int r = 0; r < 3; ++r) {
        FK[3 * r] = f[3 * r] * k1[0];
        FK[3 * r + 1] = f[3 * r + 1] * k1[0];
        FK[3 * r + 2] = f[3 * r] * k1[1] + f[3 * r + 1] * k1[2] + f[3 * r + 2];
      }
      for (int col = 0; col < 3; ++col) {
        M[col] = k2[0] * FK[col];
        M[3 + col] = k2[0] * FK[3 + col];
        M[6 + col] = k2[1] * FK[col] + k2[2] * FK[3 + col] + FK[6 + col];
      }
    }
    n = essential_candidates(M, c);
  } else if (is_homography(cfg)) {
    n = homography_candidates(H + 9 * (size_t)p, k1, k2, c);
  }
  ncand[p] = n;
}

// pair of flat match i: the last p with iptr[p] <= i (iptr non-decreasing, iptr[0] = 0 <= i < iptr[R])
__device__ __forceinline__ int pair_of(const long long* iptr, int R, long long i) {
  int lo = 0, hi = R;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (iptr[mid] <= i) lo = mid;
    else hi = mid;
  }
  return lo;
}

// normalised keypoints (ImageToWorld) of match i of pair p
__device__ __forceinline__ void match_points(int p, long long i, const uint2* __restrict__ matches, const int* __restrict__ pair_images,
                                             const long long* __restrict__ kp_ptr, const float2* __restrict__ kps,
                                             const int* __restrict__ image_camera, const double* __restrict__ cameras, double* x) {
  const uint2 m = matches[i];
  const int a = pair_images[2 * p], b = pair_images[2 * p + 1];
  const float2 pa = kps[kp_ptr[a] + m.x], pb = kps[kp_ptr[b] + m.y];
  const double* ka = cameras + 3 * image_camera[a];
  const double* kb = cameras + 3 * image_camera[b];
  x[0] = ((double)pa.x - ka[1]) / ka[0];
  x[1] = ((double)pa.y - ka[2]) / ka[0];
  x[2] = ((double)pb.x - kb[1]) / kb[0];
  x[3] = ((double)pb.y - kb[2]) / kb[0];
}

// warps walk 32 consecutive matches at a time, so that every lane reaches the ballots
__global__ void __launch_bounds__(256) k_cheirality(long long N, const long long* __restrict__ iptr, int R,
                                                    const uint2* __restrict__ matches, const int* __restrict__ pair_images,
                                                    const long long* __restrict__ kp_ptr, const float2* __restrict__ kps,
                                                    const int* __restrict__ image_camera, const double* __restrict__ cameras,
                                                    const double* __restrict__ cand, const int* __restrict__ ncand,
                                                    unsigned char* __restrict__ mask, u64* __restrict__ counts) {
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long base = warp * 32; base < N; base += nwarps * 32) {
    const long long i = base + lane;
    const bool valid = i < N;
    int p = -1;
    unsigned bits = 0;
    if (valid) {
      p = pair_of(iptr, R, i);
      const int nc = ncand[p];
      if (nc > 0) {
        double x[4];
        match_points(p, i, matches, pair_images, kp_ptr, kps, image_camera, cameras, x);
        for (int c = 0; c < nc; ++c) {
          const double* cd = cand + ((size_t)p * kCand + c) * kCandStride;
          double X[3];
          triangulate(cd, x[0], x[1], x[2], x[3], X);
          if (in_front(cd, X)) bits |= 1u << c;
        }
      }
      mask[i] = (unsigned char)bits;
    }
    const unsigned group = __match_any_sync(0xffffffffu, p);
    const bool leader = lane == __ffs(group) - 1;
#pragma unroll
    for (int c = 0; c < kCand; ++c) {
      const unsigned k = __popc(__ballot_sync(0xffffffffu, (bits >> c) & 1u) & group);
      if (leader && valid && k) atomicAdd(counts + (size_t)p * kCand + c, (u64)k);
    }
  }
}

__device__ __forceinline__ void rotation_to_quaternion(const double* R, double* q) {
  const double tr = R[0] + R[4] + R[8];
  if (tr > 0.0) {
    double s = sqrt(tr + 1.0);
    q[0] = 0.5 * s;
    s = 0.5 / s;
    q[1] = (R[7] - R[5]) * s; q[2] = (R[2] - R[6]) * s; q[3] = (R[3] - R[1]) * s;
    return;
  }
  int i = 0;
  if (R[4] > R[0]) i = 1;
  if (R[8] > R[4 * i]) i = 2;
  const int j = (i + 1) % 3, k = (j + 1) % 3;
  double s = sqrt(R[4 * i] - R[4 * j] - R[4 * k] + 1.0);
  q[1 + i] = 0.5 * s;
  s = 0.5 / s;
  q[0] = (R[3 * k + j] - R[3 * j + k]) * s;
  q[1 + j] = (R[3 * j + i] + R[3 * i + j]) * s;
  q[1 + k] = (R[3 * k + i] + R[3 * i + k]) * s;
}

__global__ void k_choose(int R, const int* __restrict__ config, const double* __restrict__ cand, const int* __restrict__ ncand,
                         const u64* __restrict__ counts, int* __restrict__ chosen, double* __restrict__ qvec, double* __restrict__ tvec,
                         int* __restrict__ config_out, long long* __restrict__ num_points3D, unsigned char* __restrict__ estimated) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= R) return;
  const int cfg = config[p], nc = ncand[p];
  const u64* cnt = counts + (size_t)p * kCand;
  double q[4] = {0.0, 0.0, 0.0, 0.0}, t[3] = {0.0, 0.0, 0.0};
  int best = -1, out_cfg = cfg;
  u64 cur = 0;
  if (nc > 0) {
    if (is_essential(cfg)) {                   // PoseFromEssentialMatrix: >=, the later candidate wins a tie
      best = 0;
      for (int c = 0; c < nc; ++c)
        if (cnt[c] >= cur) { best = c; cur = cnt[c]; }
    } else {                                   // PoseFromHomographyMatrix: >, a candidate must keep a point
      for (int c = 0; c < nc; ++c)
        if (cnt[c] > 0 && cnt[c] > cur) { best = c; cur = cnt[c]; }
      if (best < 0) best = 0;
    }
    const double* cd = cand + ((size_t)p * kCand + best) * kCandStride;
    rotation_to_quaternion(cd, q);
    t[0] = cd[9]; t[1] = cd[10]; t[2] = cd[11];
    if (cfg == 6) out_cfg = sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]) == 0.0 ? 5 : 4;
  }
  chosen[p] = best;
  for (int i = 0; i < 4; ++i) qvec[4 * (size_t)p + i] = q[i];
  for (int i = 0; i < 3; ++i) tvec[3 * (size_t)p + i] = t[i];
  config_out[p] = out_cfg;
  num_points3D[p] = (long long)cur;
  estimated[p] = nc > 0;
}

// CalculateTriangulationAngle(0, -R' t, X)
__device__ __forceinline__ double triangulation_angle(const double* cd, const double* X) {
  const double o[3] = {0.0, 0.0, 0.0};
  const double c[3] = {-(cd[0] * cd[9] + cd[3] * cd[10] + cd[6] * cd[11]), -(cd[1] * cd[9] + cd[4] * cd[10] + cd[7] * cd[11]),
                       -(cd[2] * cd[9] + cd[5] * cd[10] + cd[8] * cd[11])};
  return psfm::triangulation_angle(o, c, X);
}

__global__ void __launch_bounds__(256) k_angles(long long N, const long long* __restrict__ iptr, int R,
                                                const uint2* __restrict__ matches, const int* __restrict__ pair_images,
                                                const long long* __restrict__ kp_ptr, const float2* __restrict__ kps,
                                                const int* __restrict__ image_camera, const double* __restrict__ cameras,
                                                const double* __restrict__ cand, const int* __restrict__ chosen,
                                                const unsigned char* __restrict__ mask, u64* __restrict__ cursor, double* __restrict__ angle, int* __restrict__ angle_pair) {
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long base = warp * 32; base < N; base += nwarps * 32) {
    const long long i = base + lane;
    int p = -1;
    bool keep = false;
    if (i < N) {
      p = pair_of(iptr, R, i);
      const int c = chosen[p];
      keep = c >= 0 && ((mask[i] >> c) & 1u);
    }
    const unsigned ballot = __ballot_sync(0xffffffffu, keep);
    if (!ballot) continue;
    u64 start = 0;
    if (lane == __ffs(ballot) - 1) start = atomicAdd(cursor, (u64)__popc(ballot));
    start = __shfl_sync(0xffffffffu, start, __ffs(ballot) - 1);
    if (keep) {
      double x[4], X[3];
      match_points(p, i, matches, pair_images, kp_ptr, kps, image_camera, cameras, x);
      const double* cd = cand + ((size_t)p * kCand + chosen[p]) * kCandStride;
      triangulate(cd, x[0], x[1], x[2], x[3], X);
      const u64 pos = start + __popc(ballot & ((1u << lane) - 1u));
      angle[pos] = triangulation_angle(cd, X);
      angle_pair[pos] = p;
    }
  }
}

// COLMAP Median of every pair's sorted run; PLANAR_OR_PANORAMIC pairs that became PANORAMIC get 0
__global__ void k_median(int R, const long long* __restrict__ run_start, const long long* __restrict__ num_points3D,
                         const int* __restrict__ config_out, const int* __restrict__ config, const double* __restrict__ sorted,
                         double* __restrict__ tri_angle) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= R) return;
  const long long n = num_points3D[p];
  double m = 0.0;
  if (n > 0 && !(config[p] == 6 && config_out[p] == 5)) {
    const double* s = sorted + run_start[p];
    const long long h = n / 2;
    m = (n & 1) ? s[h] : (s[h] + s[h - 1]) / 2.0;
  }
  tri_angle[p] = m;
}

}  // namespace

extern "C" int psfm_two_view_relative_poses(int32_t num_images, const int64_t* keypoint_ptr, const float* keypoints,
                                            const int32_t* image_camera, const double* cameras, int32_t num_cameras,
                                            int64_t num_pairs, const int32_t* pair_images, const int32_t* config,
                                            const double* E, const double* F, const double* H, const int64_t* inlier_ptr,
                                            const uint32_t* inlier_matches, double* qvec, double* tvec, double* tri_angle,
                                            int32_t* config_out, int64_t* num_points3D, uint8_t* estimated) {
  const char* entry = "psfm_two_view_relative_poses";
  return guard(entry, [&]() -> int {
    int rc = check_sizes(entry, num_images, num_cameras, num_pairs);
    if (rc != PSFM_OK) return rc;
    if (num_pairs > 0 && (!keypoint_ptr || !image_camera || !cameras || !pair_images || !config || !E || !F || !H ||
                          !inlier_ptr || !qvec || !tvec || !tri_angle || !config_out || !num_points3D || !estimated))
      return fail(entry, PSFM_ERR_INVALID, "null argument");
    const int R = (int)num_pairs;
    if (R > 0) {
      // no check_distinct_pairs: this stage accepts self pairs and repeated pairs
      if ((rc = check_keypoint_ptr(entry, num_images, keypoint_ptr)) != PSFM_OK) return rc;
      if ((rc = check_image_cameras(entry, num_images, image_camera, num_cameras)) != PSFM_OK) return rc;
      if ((rc = check_match_ptr(entry, "inlier_ptr", R, inlier_ptr)) != PSFM_OK) return rc;
      if ((rc = check_pair_images(entry, R, pair_images, num_images)) != PSFM_OK) return rc;
      if (inlier_ptr[R] > 0 && (!inlier_matches || (keypoint_ptr[num_images] > 0 && !keypoints)))
        return fail(entry, PSFM_ERR_INVALID, "null argument");
      if ((rc = check_match_keypoints(entry, R, pair_images, keypoint_ptr, inlier_ptr, inlier_matches)) != PSFM_OK) return rc;
    }
    if ((rc = require_device(entry)) != PSFM_OK) return rc;
    if (R == 0) return PSFM_OK;
    const long long N = inlier_ptr[R], K = keypoint_ptr[num_images];
    DBuf<int> d_pairs, d_config, d_cam, d_ncand, d_chosen, d_cfg_out;
    DBuf<double> d_cams, d_E, d_F, d_H, d_cand, d_q, d_t, d_tri;
    DBuf<long long> d_iptr, d_kp_ptr, d_np3;
    DBuf<u64> d_counts;
    DBuf<unsigned char> d_est;
    d_pairs.alloc(2 * (size_t)R); d_config.alloc(R); d_cam.alloc(num_images); d_cams.alloc(3 * (size_t)num_cameras);
    d_E.alloc(9 * (size_t)R); d_F.alloc(9 * (size_t)R); d_H.alloc(9 * (size_t)R);
    d_cand.alloc((size_t)R * kCand * kCandStride); d_ncand.alloc(R); d_chosen.alloc(R); d_cfg_out.alloc(R);
    d_q.alloc(4 * (size_t)R); d_t.alloc(3 * (size_t)R); d_tri.alloc(R); d_np3.alloc(R); d_est.alloc(R);
    d_counts.alloc((size_t)R * kCand);
    d_pairs.upload(pair_images, 2 * (size_t)R, nullptr); d_config.upload(config, R, nullptr);
    d_cam.upload(image_camera, num_images, nullptr); d_cams.upload(cameras, 3 * (size_t)num_cameras, nullptr);
    d_E.upload(E, 9 * (size_t)R, nullptr); d_F.upload(F, 9 * (size_t)R, nullptr); d_H.upload(H, 9 * (size_t)R, nullptr);
    d_counts.zero(nullptr);
    k_candidates<<<grid_of(R), 256>>>(R, d_pairs.p, d_config.p, d_E.p, d_F.p, d_H.p, d_cam.p, d_cams.p, d_cand.p, d_ncand.p);
    PSFM_LAUNCH_CHECK();
    DBuf<uint2> d_m;
    DBuf<float2> d_kps;
    DBuf<unsigned char> d_mask;
    if (N > 0) {                                    // with no inlier at all, only the per-pair kernels run
      d_iptr.alloc((size_t)R + 1); d_kp_ptr.alloc((size_t)num_images + 1);
      d_iptr.upload(reinterpret_cast<const long long*>(inlier_ptr), (size_t)R + 1, nullptr);
      d_kp_ptr.upload(reinterpret_cast<const long long*>(keypoint_ptr), (size_t)num_images + 1, nullptr);
      d_m.alloc(N); d_kps.alloc(K); d_mask.alloc(N);
      d_m.upload(reinterpret_cast<const uint2*>(inlier_matches), N, nullptr);
      d_kps.upload(reinterpret_cast<const float2*>(keypoints), K, nullptr);
      k_cheirality<<<grid_stride_of(N), 256>>>(N, d_iptr.p, R, d_m.p, d_pairs.p, d_kp_ptr.p, d_kps.p, d_cam.p, d_cams.p,
                                               d_cand.p, d_ncand.p, d_mask.p, d_counts.p);
      PSFM_LAUNCH_CHECK();
    }
    k_choose<<<grid_of(R), 256>>>(R, d_config.p, d_cand.p, d_ncand.p, d_counts.p, d_chosen.p, d_q.p, d_t.p, d_cfg_out.p,
                                  d_np3.p, d_est.p);
    PSFM_LAUNCH_CHECK();
    PSFM_CUDA(cudaMemcpy(qvec, d_q.p, sizeof(double) * 4 * (size_t)R, cudaMemcpyDeviceToHost));
    PSFM_CUDA(cudaMemcpy(tvec, d_t.p, sizeof(double) * 3 * (size_t)R, cudaMemcpyDeviceToHost));
    PSFM_CUDA(cudaMemcpy(config_out, d_cfg_out.p, sizeof(int) * (size_t)R, cudaMemcpyDeviceToHost));
    PSFM_CUDA(cudaMemcpy(num_points3D, d_np3.p, sizeof(long long) * (size_t)R, cudaMemcpyDeviceToHost));
    PSFM_CUDA(cudaMemcpy(estimated, d_est.p, (size_t)R, cudaMemcpyDeviceToHost));
    std::vector<long long> run_start((size_t)R + 1, 0);
    for (int p = 0; p < R; ++p) run_start[p + 1] = run_start[p] + num_points3D[p];
    const long long M = run_start[R];
    if (M == 0) {
      std::fill(tri_angle, tri_angle + R, 0.0);
      return PSFM_OK;
    }
    // kept points of the chosen candidates: angles with their pair, sorted by angle, then stably by pair
    DBuf<double> ka, kb;
    DBuf<int> va, vb;
    DBuf<u64> cursor;
    ka.alloc(M); va.alloc(M); cursor.alloc(1);
    cursor.zero(nullptr);
    k_angles<<<grid_stride_of(N), 256>>>(N, d_iptr.p, R, d_m.p, d_pairs.p, d_kp_ptr.p, d_kps.p, d_cam.p, d_cams.p, d_cand.p,
                                         d_chosen.p, d_mask.p, cursor.p, ka.p, va.p);
    PSFM_LAUNCH_CHECK();
    d_m.release(); d_mask.release(); d_kps.release();
    kb.alloc(M); vb.alloc(M);
    cub::DoubleBuffer<double> keys(ka.p, kb.p);
    cub::DoubleBuffer<int> vals(va.p, vb.p);
    sort_pairs(keys, vals, M, 64);
    cub::DoubleBuffer<int> pkeys(vals.Current(), vals.Alternate());
    cub::DoubleBuffer<double> pvals(keys.Current(), keys.Alternate());
    sort_pairs(pkeys, pvals, M, key_bits(R - 1));
    DBuf<long long> d_run;
    d_run.alloc((size_t)R + 1);
    d_run.upload(run_start.data(), (size_t)R + 1, nullptr);
    k_median<<<grid_of(R), 256>>>(R, d_run.p, d_np3.p, d_cfg_out.p, d_config.p, pvals.Current(), d_tri.p);
    PSFM_LAUNCH_CHECK();
    PSFM_CUDA(cudaMemcpy(tri_angle, d_tri.p, sizeof(double) * (size_t)R, cudaMemcpyDeviceToHost));
    return PSFM_OK;
  });
}
