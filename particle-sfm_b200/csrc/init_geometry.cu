// init_geometry.cu — the RANSAC-free, embarrassingly parallel steps that initialise HP2 (SURVEY.md §8f row f-4).
//
// Reference:
//   OptimizeRelativePositionWithKnownRotation / BatchOptimize...   sfm/gmapper/src/global/known_rotation_util.cc:107-229
//       per image pair: constraint columns c_i = R2 ((R1' f1_i) x (R2' f2_i)) (:55-79), IRLS on the null vector of
//       C diag(1/w) C' with w_i = max(|t' c_i|, 1e-7) — <= 100 iterations, stop after 10 consecutive iterations
//       whose cost change is <= 1e-5 (:116-176), sign by the cheirality majority (:85-101, :181-189; COLMAP
//       CheckCheirality / TriangulatePoint / CalculateDepth).  The reference runs one ThreadPool task per pair.
//       Two callers of one kernel, templated on its point loader: psfm_known_rotation_translations (normalised
//       points from the caller) and psfm_optimize_pairwise_translations (GlobalMapper::OptimizePairwiseTranslations,
//       sfm/global_mapper.cc:106-109: the database arrays, keypoints gathered and normalised on the device).
//   multi-view DLT of a track   COLMAP TriangulateMultiViewPoint, the estimator behind
//       IncrementalTriangulator::Create (sfm/incremental_triangulator.cc:463-548): smallest eigenvector of
//       sum (P - x x' P)' (P - x x' P).
// Here: one CTA per image pair (threads over the correspondences, fixed-order block reductions, every thread
// solves the 3 x 3 eigenproblem redundantly — no broadcast), one thread per track.  Eigenvectors by cyclic Jacobi
// rotations in fp64 (the reference uses Eigen's JacobiSVD / SelfAdjointEigenSolver: same vector up to sign and
// rounding; parity tolerance in tests/test_gpu_init.py).
#include <cmath>
#include <vector>

#include "dlt.cuh"
#include "pair_inputs.h"
#include "psfm_common.cuh"

namespace {

using namespace psfm;

// COLMAP QuaternionToRotationMatrix (w, x, y, z), normalised; row-major
__device__ __forceinline__ void quat_to_rot(const double* q, double* R) {
  const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  const double w = q[0] / n, x = q[1] / n, y = q[2] / n, z = q[3] / n;
  R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - w * z); R[2] = 2 * (x * z + w * y);
  R[3] = 2 * (x * y + w * z); R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - w * x);
  R[6] = 2 * (x * z - w * y); R[7] = 2 * (y * z + w * x); R[8] = 1 - 2 * (x * x + y * y);
}

// fixed-order block sum of NV values (blockDim.x = 128): result in every thread
template <int NV>
__device__ __forceinline__ void block_sum_all(double (&v)[NV], double* sbuf) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const double s = warp_sum(v[j]);
    if (lane == 0) sbuf[j * 32 + wid] = s;
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    double s = 0.0;
    for (int w = 0; w < nw; ++w) s += sbuf[j * 32 + w];
    v[j] = s;
  }
}

// constraint column of correspondence i: R2 ((R1' f1) x (R2' f2))
__device__ __forceinline__ void constraint(const double* R1, const double* R2, double x1, double y1, double x2, double y2, double* c) {
  const double a0 = R1[0] * x1 + R1[3] * y1 + R1[6], a1 = R1[1] * x1 + R1[4] * y1 + R1[7], a2 = R1[2] * x1 + R1[5] * y1 + R1[8];
  const double b0 = R2[0] * x2 + R2[3] * y2 + R2[6], b1 = R2[1] * x2 + R2[4] * y2 + R2[7], b2 = R2[2] * x2 + R2[5] * y2 + R2[8];
  const double k0 = a1 * b2 - a2 * b1, k1 = a2 * b0 - a0 * b2, k2 = a0 * b1 - a1 * b0;
  c[0] = R2[0] * k0 + R2[1] * k1 + R2[2] * k2;
  c[1] = R2[3] * k0 + R2[4] * k1 + R2[5] * k2;
  c[2] = R2[6] * k0 + R2[7] * k1 + R2[8] * k2;
}

// Point loaders of k_known_rotation: pair p's correspondence range and its normalised points.
// PointArrays: normalised points given by the caller (psfm_known_rotation_translations).
struct PointArrays {
  const double2* __restrict__ p1;
  const double2* __restrict__ p2;
  const int* __restrict__ ptr;
  __device__ __forceinline__ void range(int p, long long& e0, long long& e1) const { e0 = ptr[p]; e1 = ptr[p + 1]; }
  __device__ __forceinline__ void load(int, long long i, double& x1, double& y1, double& x2, double& y2) const {
    const double2 a = p1[i], b = p2[i];
    x1 = a.x; y1 = a.y; x2 = b.x; y2 = b.y;
  }
};

// MatchGather: the database arrays of psfm_two_view_relative_poses; both keypoints gathered through the match's
// indices and normalised (SIMPLE_PINHOLE ImageToWorld) with two_view.cu's expression.  An unused pair has an empty
// range.
struct MatchGather {
  const long long* __restrict__ iptr;
  const uint2* __restrict__ matches;
  const int* __restrict__ pair_images;
  const long long* __restrict__ kp_ptr;
  const float2* __restrict__ kps;
  const int* __restrict__ image_camera;
  const double* __restrict__ cameras;
  const unsigned char* __restrict__ used;     // may be null: every pair
  __device__ __forceinline__ void range(int p, long long& e0, long long& e1) const {
    e0 = iptr[p];
    e1 = (used && !used[p]) ? e0 : iptr[p + 1];
  }
  __device__ __forceinline__ void load(int p, long long i, double& x1, double& y1, double& x2, double& y2) const {
    const uint2 m = matches[i];
    const int a = pair_images[2 * p], b = pair_images[2 * p + 1];
    const float2 pa = kps[kp_ptr[a] + m.x], pb = kps[kp_ptr[b] + m.y];
    const double* ka = cameras + 3 * image_camera[a];
    const double* kb = cameras + 3 * image_camera[b];
    x1 = ((double)pa.x - ka[1]) / ka[0];
    y1 = ((double)pa.y - ka[2]) / ka[0];
    x2 = ((double)pb.x - kb[1]) / kb[0];
    y2 = ((double)pb.y - kb[2]) / kb[0];
  }
};

template <class Points>
__global__ void __launch_bounds__(128) k_known_rotation(const Points pts, const double* __restrict__ q1,
                                                        const double* __restrict__ q2, double* __restrict__ tvec, int* __restrict__ iters) {
  __shared__ double sbuf[7 * 32];
  const int pair = blockIdx.x, tid = threadIdx.x;
  long long e0, e1;
  pts.range(pair, e0, e1);
  const long long n = e1 - e0;
  double R1[9], R2[9];
  quat_to_rot(q1 + 4 * (size_t)pair, R1);
  quat_to_rot(q2 + 4 * (size_t)pair, R2);
  double pos[3] = {0.0, 0.0, 0.0};
  if (n <= 0) {
    if (tid == 0) { tvec[3 * (size_t)pair] = tvec[3 * (size_t)pair + 1] = tvec[3 * (size_t)pair + 2] = 0.0; if (iters) iters[pair] = 0; }
    return;
  }
  // IRLS (known_rotation_util.cc:132-176).  One pass per iteration: with the weights of the previous vector
  // (|pos' c_i|, 1 before the first) accumulate C diag(1 / max(w, 1e-7)) C'; the cost of the new vector is the sum
  // of the next pass's unclamped weights, so the convergence test of iteration k is evaluated at the start of k + 1.
  double cost = 0.0;
  int inner = 0, its = 0;
  bool first = true;
  double newpos[3] = {0.0, 0.0, 0.0};
  for (int it = 0; it <= 100; ++it) {
    double acc[7] = {0, 0, 0, 0, 0, 0, 0};
    for (long long i = e0 + tid; i < e1; i += 128) {
      double ax, ay, bx, by;
      pts.load(pair, i, ax, ay, bx, by);
      double c[3];
      constraint(R1, R2, ax, ay, bx, by, c);
      double w = first ? 1.0 : fabs(newpos[0] * c[0] + newpos[1] * c[1] + newpos[2] * c[2]);
      acc[6] += w;                                  // cost of newpos (unclamped)
      w = w < 1e-7 ? 1e-7 : w;
      const double iw = 1.0 / w;
      acc[0] += c[0] * c[0] * iw; acc[1] += c[0] * c[1] * iw; acc[2] += c[0] * c[2] * iw;
      acc[3] += c[1] * c[1] * iw; acc[4] += c[1] * c[2] * iw; acc[5] += c[2] * c[2] * iw;
    }
    block_sum_all<7>(acc, sbuf);
    if (!first) {
      // finish iteration `its` (its vector is newpos, its cost acc[6])
      const double new_cost = acc[6];
      const double nn = newpos[0] * newpos[0] + newpos[1] * newpos[1] + newpos[2] * newpos[2];
      const double delta = fmax(fabs(cost - new_cost), 1.0 - nn);
      inner = (delta <= 1e-5) ? inner + 1 : 0;
      cost = new_cost;
      pos[0] = newpos[0]; pos[1] = newpos[1]; pos[2] = newpos[2];
      if (its >= 100 || inner >= 10) break;
    }
    first = false;
    ++its;
    double L[3][3] = {{acc[0], acc[1], acc[2]}, {acc[1], acc[3], acc[4]}, {acc[2], acc[4], acc[5]}};
    smallest_eigenvector<3>(L, newpos);
  }
  // sign: the majority of the correspondences must triangulate in front of both cameras (P1 = [I|0], P2 = [R|t])
  double R[9];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) R[3 * r + c] = R2[3 * r] * R1[3 * c] + R2[3 * r + 1] * R1[3 * c + 1] + R2[3 * r + 2] * R1[3 * c + 2];
  const double rt0 = R[0] * pos[0] + R[3] * pos[1] + R[6] * pos[2], rt1 = R[1] * pos[0] + R[4] * pos[1] + R[7] * pos[2],
               rt2 = R[2] * pos[0] + R[5] * pos[1] + R[8] * pos[2];
  const double max_depth = 1000.0 * sqrt(rt0 * rt0 + rt1 * rt1 + rt2 * rt2);
  const double eps = 2.220446049250313e-16;
  double cnt[1] = {0.0};
  for (long long i = e0 + tid; i < e1; i += 128) {
    double ax, ay, bx, by;
    pts.load(pair, i, ax, ay, bx, by);
    // DLT rows: x1 P1[2] - P1[0], y1 P1[2] - P1[1], x2 P2[2] - P2[0], y2 P2[2] - P2[1]
    double Am[4][4] = {{-1.0, 0.0, ax, 0.0},
                       {0.0, -1.0, ay, 0.0},
                       {bx * R[6] - R[0], bx * R[7] - R[1], bx * R[8] - R[2], bx * pos[2] - pos[0]},
                       {by * R[6] - R[3], by * R[7] - R[4], by * R[8] - R[5], by * pos[2] - pos[1]}};
    double X[3];
    dlt_point_4x4(Am, X);                           // TriangulatePoint: the SVD of Am itself, never Am'Am
    const double X0 = X[0], X1 = X[1], X2 = X[2];
    const double d1 = X2;
    if (d1 > eps && d1 < max_depth) {
      const double d2 = (R[6] * X0 + R[7] * X1 + R[8] * X2 + pos[2]) * sqrt(R[2] * R[2] + R[5] * R[5] + R[8] * R[8]);
      if (d2 > eps && d2 < max_depth) cnt[0] += 1.0;
    }
  }
  block_sum_all<1>(cnt, sbuf);
  if (!(cnt[0] > (double)(n / 2))) { pos[0] = -pos[0]; pos[1] = -pos[1]; pos[2] = -pos[2]; }
  if (tid == 0) {
    tvec[3 * (size_t)pair] = pos[0]; tvec[3 * (size_t)pair + 1] = pos[1]; tvec[3 * (size_t)pair + 2] = pos[2];
    if (iters) iters[pair] = its;
  }
}

// one thread per track: A = sum (P - x x' P)' (P - x x' P), X = smallest eigenvector, dehomogenised
__global__ void __launch_bounds__(128) k_triangulate_tracks(const double* __restrict__ proj, const double2* __restrict__ xy,
                                                            const int* __restrict__ track_ptr, int ntracks, double* __restrict__ xyz) {
  const int t = blockIdx.x * 128 + threadIdx.x;
  if (t >= ntracks) return;
  double A[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) A[r][c] = 0.0;
  for (int i = track_ptr[t]; i < track_ptr[t + 1]; ++i) {
    const double2 p = xy[i];
    multi_view_accumulate(proj + 12 * (size_t)i, p.x, p.y, A);
  }
  double v[4];
  smallest_eigenvector<4>(A, v);
  xyz[3 * (size_t)t] = v[0] / v[3]; xyz[3 * (size_t)t + 1] = v[1] / v[3]; xyz[3 * (size_t)t + 2] = v[2] / v[3];
}

}  // namespace

extern "C" int psfm_known_rotation_translations(const double* points1, const double* points2, const int32_t* pair_ptr,
                                                const double* qvec1, const double* qvec2, int32_t num_pairs, double* tvec,
                                                int32_t* iterations) {
  return guard("psfm_known_rotation_translations", [&]() -> int {
    if (num_pairs < 0 || (num_pairs > 0 && (!pair_ptr || !qvec1 || !qvec2 || !tvec))) return PSFM_ERR_INVALID;
    int rc = require_device("psfm_known_rotation_translations");
    if (rc != PSFM_OK) return rc;
    if (num_pairs == 0) return PSFM_OK;
    const size_t m = (size_t)pair_ptr[num_pairs];
    if (pair_ptr[0] != 0 || (m > 0 && (!points1 || !points2))) return PSFM_ERR_INVALID;
    for (int i = 0; i < num_pairs; ++i)
      if (pair_ptr[i + 1] < pair_ptr[i]) return PSFM_ERR_INVALID;
    DBuf<double> d1, d2, dq1, dq2, dt;
    DBuf<int> dp, di;
    d1.alloc(2 * m); d2.alloc(2 * m); dq1.alloc(4 * (size_t)num_pairs); dq2.alloc(4 * (size_t)num_pairs);
    dt.alloc(3 * (size_t)num_pairs); dp.alloc((size_t)num_pairs + 1); di.alloc((size_t)num_pairs);
    d1.upload(points1, 2 * m, nullptr); d2.upload(points2, 2 * m, nullptr);
    dq1.upload(qvec1, dq1.n, nullptr); dq2.upload(qvec2, dq2.n, nullptr); dp.upload(pair_ptr, dp.n, nullptr);
    const PointArrays pts{reinterpret_cast<const double2*>(d1.p), reinterpret_cast<const double2*>(d2.p), dp.p};
    k_known_rotation<<<num_pairs, 128>>>(pts, dq1.p, dq2.p, dt.p, di.p);
    PSFM_LAUNCH_CHECK();
    PSFM_CUDA(cudaMemcpy(tvec, dt.p, sizeof(double) * dt.n, cudaMemcpyDeviceToHost));
    if (iterations) PSFM_CUDA(cudaMemcpy(iterations, di.p, sizeof(int) * di.n, cudaMemcpyDeviceToHost));
    return PSFM_OK;
  });
}

extern "C" int psfm_triangulate_tracks(const double* proj_matrices, const double* points, const int32_t* track_ptr,
                                       int32_t num_tracks, double* xyz) {
  return guard("psfm_triangulate_tracks", [&]() -> int {
    if (num_tracks < 0 || (num_tracks > 0 && (!track_ptr || !xyz))) return PSFM_ERR_INVALID;
    int rc = require_device("psfm_triangulate_tracks");
    if (rc != PSFM_OK) return rc;
    if (num_tracks == 0) return PSFM_OK;
    const size_t m = (size_t)track_ptr[num_tracks];
    if (track_ptr[0] != 0 || (m > 0 && (!proj_matrices || !points))) return PSFM_ERR_INVALID;
    for (int i = 0; i < num_tracks; ++i)
      if (track_ptr[i + 1] < track_ptr[i]) return PSFM_ERR_INVALID;
    DBuf<double> dP, dx, dX;
    DBuf<int> dp;
    dP.alloc(12 * m); dx.alloc(2 * m); dX.alloc(3 * (size_t)num_tracks); dp.alloc((size_t)num_tracks + 1);
    dP.upload(proj_matrices, 12 * m, nullptr); dx.upload(points, 2 * m, nullptr); dp.upload(track_ptr, dp.n, nullptr);
    k_triangulate_tracks<<<(num_tracks + 127) / 128, 128>>>(dP.p, reinterpret_cast<const double2*>(dx.p), dp.p, num_tracks, dX.p);
    PSFM_LAUNCH_CHECK();
    PSFM_CUDA(cudaMemcpy(xyz, dX.p, sizeof(double) * dX.n, cudaMemcpyDeviceToHost));
    return PSFM_OK;
  });
}

extern "C" int psfm_optimize_pairwise_translations(int32_t num_images, const int64_t* keypoint_ptr, const float* keypoints,
                                                   const int32_t* image_camera, const double* cameras, int32_t num_cameras,
                                                   int64_t num_pairs, const int32_t* pair_images, const int64_t* inlier_ptr,
                                                   const uint32_t* inlier_matches, const double* orientations,
                                                   const uint8_t* pair_used, double* tvec, int32_t* iterations) {
  const char* entry = "psfm_optimize_pairwise_translations";
  return guard(entry, [&]() -> int {
    int rc = check_sizes(entry, num_images, num_cameras, num_pairs);
    if (rc != PSFM_OK) return rc;
    if (num_pairs > 0 && (!keypoint_ptr || !image_camera || !cameras || !pair_images || !inlier_ptr || !orientations ||
                          !tvec || !iterations))
      return fail(entry, PSFM_ERR_INVALID, "null argument");
    const int R = (int)num_pairs;
    if (R > 0) {
      // no check_distinct_pairs: this stage accepts self pairs and repeated pairs
      if ((rc = check_keypoint_ptr(entry, num_images, keypoint_ptr)) != PSFM_OK) return rc;
      if ((rc = check_image_cameras(entry, num_images, image_camera, num_cameras)) != PSFM_OK) return rc;
      if ((rc = check_match_ptr(entry, "inlier_ptr", R, inlier_ptr)) != PSFM_OK) return rc;
      if ((rc = check_pair_images(entry, R, pair_images, num_images)) != PSFM_OK) return rc;
      for (int p = 0; p < R; ++p) {
        if (pair_used && !pair_used[p]) continue;
        for (int k = 0; k < 2; ++k) {
          const double* q = orientations + 4 * (size_t)pair_images[2 * p + k];
          const double n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
          if (!(std::isfinite(n2) && n2 > 0.0))
            return fail(entry, PSFM_ERR_INVALID, "a used pair's image has a zero or non-finite orientation");
        }
      }
      if (inlier_ptr[R] > 0 && (!inlier_matches || (keypoint_ptr[num_images] > 0 && !keypoints)))
        return fail(entry, PSFM_ERR_INVALID, "null argument");
      if ((rc = check_match_keypoints(entry, R, pair_images, keypoint_ptr, inlier_ptr, inlier_matches)) != PSFM_OK) return rc;
    }
    if ((rc = require_device(entry)) != PSFM_OK) return rc;
    if (R == 0) return PSFM_OK;
    const long long N = inlier_ptr[R], K = keypoint_ptr[num_images];
    // the kernel reads one quaternion pair per pair: gathered here from the image orientations
    std::vector<double> q1(4 * (size_t)R), q2(4 * (size_t)R);
    for (int p = 0; p < R; ++p)
      for (int k = 0; k < 4; ++k) {
        q1[4 * (size_t)p + k] = orientations[4 * (size_t)pair_images[2 * p] + k];
        q2[4 * (size_t)p + k] = orientations[4 * (size_t)pair_images[2 * p + 1] + k];
      }
    DBuf<double> d_q1, d_q2, d_t, d_cams;
    DBuf<int> d_it, d_pairs, d_cam;
    DBuf<long long> d_iptr, d_kp_ptr;
    DBuf<uint2> d_m;
    DBuf<float2> d_kps;
    DBuf<unsigned char> d_used;
    d_q1.alloc(4 * (size_t)R); d_q2.alloc(4 * (size_t)R); d_t.alloc(3 * (size_t)R); d_it.alloc(R);
    d_pairs.alloc(2 * (size_t)R); d_cam.alloc(num_images); d_cams.alloc(3 * (size_t)num_cameras);
    d_iptr.alloc((size_t)R + 1); d_kp_ptr.alloc((size_t)num_images + 1); d_m.alloc(N); d_kps.alloc(K);
    d_q1.upload(q1.data(), q1.size(), nullptr); d_q2.upload(q2.data(), q2.size(), nullptr);
    d_pairs.upload(pair_images, 2 * (size_t)R, nullptr); d_cam.upload(image_camera, num_images, nullptr);
    d_cams.upload(cameras, 3 * (size_t)num_cameras, nullptr);
    d_iptr.upload(reinterpret_cast<const long long*>(inlier_ptr), (size_t)R + 1, nullptr);
    d_kp_ptr.upload(reinterpret_cast<const long long*>(keypoint_ptr), (size_t)num_images + 1, nullptr);
    d_m.upload(reinterpret_cast<const uint2*>(inlier_matches), N, nullptr);
    d_kps.upload(reinterpret_cast<const float2*>(keypoints), K, nullptr);
    if (pair_used) { d_used.alloc(R); d_used.upload(pair_used, R, nullptr); }
    const MatchGather pts{d_iptr.p, d_m.p, d_pairs.p, d_kp_ptr.p, d_kps.p, d_cam.p, d_cams.p, pair_used ? d_used.p : nullptr};
    k_known_rotation<<<R, 128>>>(pts, d_q1.p, d_q2.p, d_t.p, d_it.p);
    PSFM_LAUNCH_CHECK();
    PSFM_CUDA(cudaMemcpy(tvec, d_t.p, sizeof(double) * 3 * (size_t)R, cudaMemcpyDeviceToHost));
    PSFM_CUDA(cudaMemcpy(iterations, d_it.p, sizeof(int) * (size_t)R, cudaMemcpyDeviceToHost));
    return PSFM_OK;
  });
}
