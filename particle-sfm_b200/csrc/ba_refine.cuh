// ba_refine.cuh — the between-round filters of the global refinement loop, on the device.
//
// IterativeGlobalRefinement (reference controllers/global_mapper.cc:245-271) alternates the
// global BA with point / observation filters; the observations never leave HBM here:
//   k_filter_negative_depth   Reconstruction::FilterObservationsWithNegativeDepth
//                             (base/reconstruction.cc:711-729 + DeleteObservation :300-320)
//   k_filter_points           Reconstruction::FilterAllPoints3D (:697-709) =
//                             FilterPoints3DWithLargeReprojectionError (:1383-1434) then
//                             FilterPoints3DWithSmallTriangulationAngle (:1321-1381)
//   k_proj_centres            Image::ProjectionCenter = -R' t
// They run on the point-sorted observation arrays of the tile structure (one thread per point:
// its observations are contiguous) and clear bits of the ALIVE mask over the caller's
// observations; the structure is then rebuilt from the surviving observations on the device
// (rebuild_structure in ba_solver.cu).  The reference's sequential DeleteObservation calls have
// order-independent per-point outcomes, written here in closed form (oracle/refine_oracle.py
// states and tests the same closed forms against hand-computed cases).
// COLMAP helpers not in the reference repository (base/projection.cc, base/triangulation.cc @bd84ad6)
// are restated: HasPointPositiveDepth (depth >= DBL_EPSILON), CalculateSquaredReprojectionError
// (DBL_MAX when depth < DBL_EPSILON), CalculateTriangulationAngle (law of cosines, min(a, pi - a)).
#pragma once
#include "ba_kernels.cuh"

namespace psfm {
namespace ba {

struct FilterCtx {
  const int* pt_ptr;        // [P + 1] observation range of each (internal) point
  const int* obs_img;       // [M]
  const double2* obs_xy;    // [M]
  const int* obs_orig;      // [M] sorted observation -> caller's observation index
  const int* pt_orig;       // [P] internal point -> caller's point index
  const int* img_cam;       // [F]
  const double* pose;       // [F][8] q (wxyz) t pad
  const double* X;          // [3P] internal order
  const double* K;          // [3C]
  int P;
  unsigned char* alive;     // [M0] over the caller's observations
  unsigned long long* count;   // [1] += filtered (the reference's num_filtered)
};

__device__ __forceinline__ void rot_from_q(const double* p, double* R) {
  const double q0 = p[0], q1 = p[1], q2 = p[2], q3 = p[3];
  R[0] = 1.0 - 2.0 * (q2 * q2 + q3 * q3); R[1] = 2.0 * (q1 * q2 - q0 * q3); R[2] = 2.0 * (q1 * q3 + q0 * q2);
  R[3] = 2.0 * (q1 * q2 + q0 * q3); R[4] = 1.0 - 2.0 * (q1 * q1 + q3 * q3); R[5] = 2.0 * (q2 * q3 - q0 * q1);
  R[6] = 2.0 * (q1 * q3 - q0 * q2); R[7] = 2.0 * (q2 * q3 + q0 * q1); R[8] = 1.0 - 2.0 * (q1 * q1 + q2 * q2);
}

__global__ void k_proj_centres(const double* pose, int F, double* centres) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= F) return;
  const double* p = pose + 8 * (size_t)i;
  double R[9];
  rot_from_q(p, R);
  for (int k = 0; k < 3; ++k) centres[3 * (size_t)i + k] = -(R[k] * p[4] + R[3 + k] * p[5] + R[6 + k] * p[6]);
}

// Per point with track length L and n observations of non-positive depth: the point goes when
// L - n < 2 (DeleteObservation deletes the whole point once Track().Length() <= 2); the
// reference counts one per DeleteObservation call it makes = min(n, max(L - 1, 1)).
__global__ void __launch_bounds__(128) k_filter_negative_depth(const FilterCtx c) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= c.P) return;
  const int b = c.pt_ptr[p], e = c.pt_ptr[p + 1], L = e - b;
  if (L == 0) return;
  const double X0 = c.X[3 * (size_t)p], X1 = c.X[3 * (size_t)p + 1], X2 = c.X[3 * (size_t)p + 2];
  int n = 0;
  for (int i = b; i < e; ++i) {
    const double* ps = c.pose + 8 * (size_t)c.obs_img[i];
    const double q0 = ps[0], q1 = ps[1], q2 = ps[2], q3 = ps[3];
    const double z = 2.0 * (q1 * q3 - q0 * q2) * X0 + 2.0 * (q2 * q3 + q0 * q1) * X1 + (1.0 - 2.0 * (q1 * q1 + q2 * q2)) * X2 + ps[6];
    n += !(z >= 2.220446049250313e-16);
  }
  if (n == 0) return;
  const bool del = L - n < 2;
  for (int i = b; i < e; ++i) {
    bool kill = del;
    if (!kill) {
      const double* ps = c.pose + 8 * (size_t)c.obs_img[i];
      const double q0 = ps[0], q1 = ps[1], q2 = ps[2], q3 = ps[3];
      const double z = 2.0 * (q1 * q3 - q0 * q2) * X0 + 2.0 * (q2 * q3 + q0 * q1) * X1 + (1.0 - 2.0 * (q1 * q1 + q2 * q2)) * X2 + ps[6];
      kill = !(z >= 2.220446049250313e-16);
    }
    if (kill) c.alive[c.obs_orig[i]] = 0;
  }
  atomicAdd(c.count, (unsigned long long)min(n, max(L - 1, 1)));
}

__device__ __forceinline__ double sq_reproj_error(const FilterCtx& c, int i, double X0, double X1, double X2) {
  const int img = c.obs_img[i];
  const double* ps = c.pose + 8 * (size_t)img;
  double R[9];
  rot_from_q(ps, R);
  const double p0 = R[0] * X0 + R[1] * X1 + R[2] * X2 + ps[4];
  const double p1 = R[3] * X0 + R[4] * X1 + R[5] * X2 + ps[5];
  const double p2 = R[6] * X0 + R[7] * X1 + R[8] * X2 + ps[6];
  if (p2 < 2.220446049250313e-16) return 1.7976931348623157e308;
  const double* K = c.K + 3 * (size_t)c.img_cam[img];
  const double2 xy = c.obs_xy[i];
  const double ex = K[0] * (p0 / p2) + K[1] - xy.x, ey = K[0] * (p1 / p2) + K[2] - xy.y;
  return ex * ex + ey * ey;
}

// Reprojection-error rule per point (L observations, d of them above the threshold): L < 2 or
// d >= L - 1 -> point deleted (L counted); else the d observations go (d counted) and the
// point's error is the mean of the kept ones.  Then, on what is left: the point stays iff some
// pair of its images sees it under >= min_tri_angle; a point deleted here counts ONE.
__global__ void __launch_bounds__(128) k_filter_points(const FilterCtx c, const double* centres, double max_sq_error,
                                                       double min_tri_angle_rad, double* point_error) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= c.P) return;
  const int b = c.pt_ptr[p], e = c.pt_ptr[p + 1], L = e - b;
  if (L == 0) return;
  const double X0 = c.X[3 * (size_t)p], X1 = c.X[3 * (size_t)p + 1], X2 = c.X[3 * (size_t)p + 2];
  int d = 0;
  double esum = 0.0;
  for (int i = b; i < e; ++i) {
    const double e2 = sq_reproj_error(c, i, X0, X1, X2);
    if (e2 > max_sq_error) ++d; else esum += sqrt(e2);
  }
  unsigned long long num = 0;
  bool del = (L < 2) || (d >= L - 1);
  if (del) {
    num = (unsigned long long)L;
  } else {
    num = (unsigned long long)d;
    point_error[c.pt_orig[p]] = esum / (double)(L - d);
    // triangulation angle over the kept observations
    bool keep = false;
    for (int i1 = b; i1 < e && !keep; ++i1) {
      if (d && sq_reproj_error(c, i1, X0, X1, X2) > max_sq_error) continue;
      const double* c1 = centres + 3 * (size_t)c.obs_img[i1];
      const double r1 = (X0 - c1[0]) * (X0 - c1[0]) + (X1 - c1[1]) * (X1 - c1[1]) + (X2 - c1[2]) * (X2 - c1[2]);
      for (int i2 = b; i2 < i1; ++i2) {
        if (d && sq_reproj_error(c, i2, X0, X1, X2) > max_sq_error) continue;
        const double* c2 = centres + 3 * (size_t)c.obs_img[i2];
        const double r2 = (X0 - c2[0]) * (X0 - c2[0]) + (X1 - c2[1]) * (X1 - c2[1]) + (X2 - c2[2]) * (X2 - c2[2]);
        const double bl = (c1[0] - c2[0]) * (c1[0] - c2[0]) + (c1[1] - c2[1]) * (c1[1] - c2[1]) + (c1[2] - c2[2]) * (c1[2] - c2[2]);
        const double den = 2.0 * sqrt(r1 * r2);
        double ang = 0.0;
        if (den != 0.0) {
          ang = fabs(acos((r1 + r2 - bl) / den));
          ang = fmin(ang, 3.141592653589793 - ang);
        }
        if (ang >= min_tri_angle_rad) { keep = true; break; }
      }
    }
    if (!keep) { del = true; num += 1; }
  }
  if (del || d) {
    for (int i = b; i < e; ++i)
      if (del || sq_reproj_error(c, i, X0, X1, X2) > max_sq_error) c.alive[c.obs_orig[i]] = 0;
  }
  if (num) atomicAdd(c.count, num);
}

// alive observations -> compact (image, point, xy) arrays + their caller's index (stream compaction
// done with a flagged select of the index; this kernel gathers)
__global__ void k_gather_alive(const int* sel, int n, const int* img, const int* pt, const double2* xy, int* oimg, int* opt,
                               double2* oxy) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int s = sel[i];
  oimg[i] = img[s]; opt[i] = pt[s]; oxy[i] = xy[s];
}

__global__ void k_compose_index(int* idx, const int* sel, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) idx[i] = sel[idx[i]];
}

// Reconstruction::Normalize applied to the points: X <- (X - t) s
__global__ void k_similarity_points(double* X, size_t n3, double t0, double t1, double t2, double s) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n3) return;
  const int k = (int)(i % 3);
  X[i] = (X[i] - (k == 0 ? t0 : (k == 1 ? t1 : t2))) * s;
}

}  // namespace ba
}  // namespace psfm
