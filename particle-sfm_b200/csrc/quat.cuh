// quat.cuh — COLMAP / Ceres quaternion helpers (w, x, y, z) shared by the global rotation averaging
// (rotation_averaging.cu) and the global position estimation (position_estimation.cu).
#pragma once
#include <cmath>

namespace psfm {
namespace quat {

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
__host__ __device__ inline Quat load_q(const double* q) { return {q[0], q[1], q[2], q[3]}; }

// QuaternionRotatePoint: the normalised quaternion applied to p as Eigen's Quaterniond * Vector3d does it
// (uv = 2 (q.vec x p), p + w uv + q.vec x uv)
__host__ __device__ inline void qrotate(const Quat& q0, const double* p, double* out) {
  const Quat q = qnormalize(q0);
  double uv0 = q.y * p[2] - q.z * p[1], uv1 = q.z * p[0] - q.x * p[2], uv2 = q.x * p[1] - q.y * p[0];
  uv0 += uv0; uv1 += uv1; uv2 += uv2;
  out[0] = p[0] + q.w * uv0 + (q.y * uv2 - q.z * uv1);
  out[1] = p[1] + q.w * uv1 + (q.z * uv0 - q.x * uv2);
  out[2] = p[2] + q.w * uv2 + (q.x * uv1 - q.y * uv0);
}

}  // namespace quat
}  // namespace psfm
