// triangulation.cu — GlobalMapper::TriangulateAllPoints: image poses and verified matches in, the 3D points and tracks
// the global bundle adjustment starts from out (DESIGN.md §4.7).
//
// Reference: GlobalMapper::TriangulateAllPoints (sfm/global_mapper.cc:232-247) runs IncrementalTriangulator::
// TriangulateImage (sfm/incremental_triangulator.cc:61-119) for every registered image in ascending id, every Point2D
// in index order: Find (:421-461), Continue (:550-590), Create (:463-548) with COLMAP's EstimateTriangulation
// (triangulation_recalled.cuh).  The restatement is oracle/triangulation_oracle.py.
//
// Processing an observation reads and writes state only inside its connected component of the correspondence graph
// restricted to registered, non-bogus images, so the sequential pass equals one sequential pass per component over
// its observations in keypoint order (keypoint index = (image, point2D) order), and point ids follow from sorting the
// created points by (creating keypoint, peel index).
// Device (K keypoints, N inlier matches of used pairs, A keypoints with an eligible correspondence, C components):
//   graph       k_entries (2 directed entries per match; an unused pair's sort last) -> stable radix sort by source
//               keypoint (push_back order: pair, then match) -> k_list_ptr -> k_neighbours (destination keypoint, flags
//               the pairs whose match list repeats an index) -> k_dedupe (one thread per flagged pair: the duplicate
//               rule in match order) -> k_drop -> k_degree (list sizes over the full graph, IsTwoViewObservation)
//   components  k_uf_hook (union-find, the smaller root wins: labels are the smallest keypoint, deterministic) ->
//               k_uf_label -> stable sort by label -> k_comp_heads -> scan -> k_comp_bounds -> sort by size, largest
//               first
//   replay      k_replay: one warp per component (handed out largest first); Find / Continue / Create as the reference
//               runs them.  EstimateTriangulation: lanes evaluate 32 consecutive pair samples (two-view DLT, depth and
//               angle tests, squared angular residuals in observation order, support), then a lane-ordered replay
//               applies the sequential rules (support comparison, local optimisation with the whole warp, the dynamic
//               trial bound); samples past the stopping trial are dropped.
//   assembly    stable sort of the points by creating keypoint -> k_point_ids -> k_elem_keys -> stable sort of the track
//               elements by point -> k_tracks -> k_kp_points
// The launch count is fixed per call; no floating-point atomics (integer counters only): two calls are bit-identical.
// Memory: the sort holds 24 bytes per directed entry (48 per match) with the matches (8) beside it; from the replay on,
// 8 bytes per match (the neighbour lists) and about 70 bytes per keypoint stay resident.  The handle keeps 20 bytes per
// keypoint (keypoint, image, point row) for psfm_ba_create_from_triangulation beside the points and tracks.
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <vector>

#include "dlt.cuh"
#include "pair_inputs.h"
#include "psfm_common.cuh"
#include "quat.cuh"
#include "radix_sort.cuh"
#include "triangulation_handle.cuh"
#include "triangulation_recalled.cuh"

namespace {

using namespace psfm;
using namespace psfm::tri;
typedef unsigned long long u64;

constexpr int kImg = 24;                 // doubles per image: P [12] row-major, centre [3], qvec [4], tvec [3], 2 unused
constexpr unsigned kNone = 0xffffffffu;  // sort key of an unused entry / slot

enum { kCntActive, kCntPoints, kCntElements, kCntContinued, kCntTrials, kCntLocal, kCntNext, kCntNum };

struct Ctx {
  const float2* kps;
  const int* img_of;
  const int* cam_of;
  const double* cams;
  const double* img;               // [F][kImg]
  const unsigned char* elig;
  const long long* list_ptr;
  const int* nbr;
  const int* deg;
  const int* first_nbr;
  const int* comp_kp;              // [A] keypoints by component
  const int* comp_off;             // [C + 1]
  const int* comp_order;           // [C] largest first
  int C;
  int* pt_of;                      // [K] slot of the keypoint's point, -1
  int* lst;                        // [A] per component: the current observation list
  int* tmp;                        // [A] per component: the inliers of the local optimisation
  double* pt_xyz;                  // [A][3] per component: its points
  unsigned* pt_creator;            // [A]
  int* el_slot;                    // [A] per component: the track elements in append order
  int* el_kp;
  u64* cnt;
  double thr;                      // create_max_angle_error^2 (radians)
  double cont_max;                 // continue_max_angle_error (radians)
  double min_tri;                  // min_angle (radians)
  int ignore_two_view;
  long long trial_cap;             // the RANSAC constructor's cap of max_num_trials
};


__device__ __forceinline__ int pair_of(const long long* iptr, int R, long long i) {
  int lo = 0, hi = R;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (iptr[mid] <= i) lo = mid;
    else hi = mid;
  }
  return lo;
}

// ---- graph ---------------------------------------------------------------------------------------------------------
__global__ void k_kp_image(int F, const long long* __restrict__ kp_ptr, int* __restrict__ img_of, int* __restrict__ pt_of,
                           int* __restrict__ parent, unsigned char* __restrict__ active) {
  const int f = blockIdx.x;
  if (f >= F) return;
  for (long long k = kp_ptr[f] + threadIdx.x; k < kp_ptr[f + 1]; k += blockDim.x) {
    img_of[k] = f; pt_of[k] = -1; parent[k] = (int)k; active[k] = 0;
  }
}

// one CTA per pair: entry 2 i (source in image 1) and 2 i + 1 (source in image 2) of match i
__global__ void k_entries(int R, const long long* __restrict__ iptr, const int2* __restrict__ pairs, const unsigned char* __restrict__ used,
                          const long long* __restrict__ kp_ptr, const uint2* __restrict__ m, unsigned* __restrict__ key,
                          u64* __restrict__ val, unsigned char* __restrict__ accepted, unsigned sentinel) {
  const int p = blockIdx.x;
  if (p >= R) return;
  const int2 ab = pairs[p];
  const bool u = !used || used[p];
  for (long long i = iptr[p] + threadIdx.x; i < iptr[p + 1]; i += blockDim.x) {
    const uint2 mm = m[i];
    key[2 * i] = u ? (unsigned)(kp_ptr[ab.x] + mm.x) : sentinel;
    key[2 * i + 1] = u ? (unsigned)(kp_ptr[ab.y] + mm.y) : sentinel;
    val[2 * i] = 2 * (u64)i;
    val[2 * i + 1] = 2 * (u64)i + 1;
    accepted[i] = 1;
  }
}

__global__ void k_list_ptr(long long K, long long E, const unsigned* __restrict__ key, long long* __restrict__ list_ptr) {
  const long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (k > K) return;
  long long lo = 0, hi = E;                  // first entry with key >= k
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (key[mid] < (unsigned)k) lo = mid + 1;
    else hi = mid;
  }
  list_ptr[k] = lo;
}

__device__ __forceinline__ int entry_dest(u64 e, const long long* iptr, int R, const int2* pairs, const long long* kp_ptr,
                                          const uint2* m, int* pair) {
  const long long i = (long long)(e >> 1);
  const int p = pair_of(iptr, R, i);
  const uint2 mm = m[i];
  *pair = p;
  return (e & 1) ? (int)(kp_ptr[pairs[p].x] + mm.x) : (int)(kp_ptr[pairs[p].y] + mm.y);
}

// destination keypoint of every used entry; a pair whose match list repeats an index has two adjacent entries with
// the same source and the same destination image
__global__ void k_neighbours(long long E, const unsigned* __restrict__ key, const u64* __restrict__ val, unsigned sentinel,
                             const long long* __restrict__ iptr, int R, const int2* __restrict__ pairs,
                             const long long* __restrict__ kp_ptr, const uint2* __restrict__ m, const int* __restrict__ img_of,
                             int* __restrict__ nbr, unsigned char* __restrict__ flag) {
  for (long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x; s < E; s += (long long)gridDim.x * blockDim.x) {
    if (key[s] == sentinel) { nbr[s] = -1; continue; }
    int p, q;
    const int d = entry_dest(val[s], iptr, R, pairs, kp_ptr, m, &p);
    nbr[s] = d;
    if (s > 0 && key[s - 1] == key[s]) {
      const int d0 = entry_dest(val[s - 1], iptr, R, pairs, kp_ptr, m, &q);
      if (img_of[d0] == img_of[d]) flag[p] = 1;
    }
  }
}

// AddCorrespondences' duplicate rule on a flagged pair, match by match: a match is dropped when an earlier accepted
// match of the pair shares its point in image 1 or in image 2
__global__ void k_dedupe(int R, const unsigned char* __restrict__ flag, const long long* __restrict__ iptr,
                         const int2* __restrict__ pairs, const long long* __restrict__ kp_ptr, const uint2* __restrict__ m,
                         const long long* __restrict__ list_ptr, const u64* __restrict__ val, unsigned char* accepted) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= R || !flag[p]) return;
  const long long i0 = iptr[p], i1 = iptr[p + 1];
  for (long long i = i0; i < i1; ++i) {
    const long long src[2] = {kp_ptr[pairs[p].x] + m[i].x, kp_ptr[pairs[p].y] + m[i].y};
    bool dup = false;
    for (int side = 0; side < 2 && !dup; ++side)
      for (long long s = list_ptr[src[side]]; s < list_ptr[src[side] + 1]; ++s) {
        const long long j = (long long)(val[s] >> 1);
        if (j >= i0 && j < i && accepted[j]) { dup = true; break; }
      }
    if (dup) accepted[i] = 0;
  }
}

__global__ void k_drop(long long E, const u64* __restrict__ val, const unsigned char* __restrict__ accepted, int* __restrict__ nbr) {
  for (long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x; s < E; s += (long long)gridDim.x * blockDim.x)
    if (nbr[s] >= 0 && !accepted[val[s] >> 1]) nbr[s] = -1;
}

__global__ void k_degree(long long K, const long long* __restrict__ list_ptr, const int* __restrict__ nbr, int* __restrict__ deg,
                         int* __restrict__ first_nbr) {
  const long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (k >= K) return;
  int n = 0, f = -1;
  for (long long s = list_ptr[k]; s < list_ptr[k + 1]; ++s)
    if (nbr[s] >= 0) {
      if (n == 0) f = nbr[s];
      ++n;
    }
  deg[k] = n;
  first_nbr[k] = f;
}

// ---- components ----------------------------------------------------------------------------------------------------
__device__ __forceinline__ int uf_find(const int* parent, int x) {
  int p = ((volatile const int*)parent)[x];
  while (p != x) { x = p; p = ((volatile const int*)parent)[x]; }
  return x;
}

__global__ void k_uf_hook(long long E, const unsigned* __restrict__ key, const int* __restrict__ nbr, const int* __restrict__ img_of,
                          const unsigned char* __restrict__ elig, int* parent, unsigned char* active) {
  for (long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x; s < E; s += (long long)gridDim.x * blockDim.x) {
    const int v = nbr[s];
    if (v < 0) continue;
    int u = (int)key[s];
    if (u > v || !elig[img_of[u]] || !elig[img_of[v]]) continue;
    active[u] = 1; active[v] = 1;
    int a = u, b = v;
    while (true) {
      a = uf_find(parent, a); b = uf_find(parent, b);
      if (a == b) break;
      if (a < b) { const int t = a; a = b; b = t; }
      if (atomicCAS(parent + a, a, b) == a) break;
    }
  }
}

__global__ void k_uf_label(long long K, const int* parent, const unsigned char* __restrict__ active, unsigned* __restrict__ key,
                           int* __restrict__ val, u64* cnt) {
  const long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (k >= K) return;
  const bool a = active[k];
  key[k] = a ? (unsigned)uf_find(parent, (int)k) : kNone;
  val[k] = (int)k;
  if (a) atomicAdd(cnt + kCntActive, 1ull);
}

__global__ void k_comp_heads(int A, const unsigned* __restrict__ key, int* __restrict__ head) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= A) return;
  head[s] = (s == 0 || key[s] != key[s - 1]) ? 1 : 0;
}

__global__ void k_comp_bounds(int A, const int* __restrict__ head, const int* __restrict__ cid, int* __restrict__ comp_off) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= A) return;
  if (head[s]) comp_off[cid[s] - 1] = s;
  if (s == A - 1) comp_off[cid[s]] = A;
}

__global__ void k_comp_sizes(int C, const int* __restrict__ comp_off, unsigned* __restrict__ key, int* __restrict__ val) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  key[c] = kNone - (unsigned)(comp_off[c + 1] - comp_off[c]);
  val[c] = c;
}

// ---- replay --------------------------------------------------------------------------------------------------------
// observation k: its normalised point (x, y) and its image's row of the per-image table
__device__ __forceinline__ const double* observation(const Ctx& c, int k, double& x, double& y) {
  const int f = c.img_of[k];
  const double* cam = c.cams + 3 * c.cam_of[f];
  const float2 u = c.kps[k];
  x = ((double)u.x - cam[1]) / cam[0];          // SIMPLE_PINHOLE ImageToWorld
  y = ((double)u.y - cam[2]) / cam[0];
  return c.img + (size_t)kImg * f;
}

__device__ __forceinline__ double ray_angle(double x, double y, const double* r) {
  const double c0 = y * r[2] - r[1], c1 = r[0] - x * r[2], c2 = x * r[1] - y * r[0];
  return atan2(sqrt(c0 * c0 + c1 * c1 + c2 * c2), x * r[0] + y * r[1] + r[2]);
}

// squared CalculateNormalizedAngularError, ProjectionMatrix form
__device__ __forceinline__ double sq_residual(const double* T, double x, double y, const double* X) {
  double r[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) r[i] = T[4 * i] * X[0] + T[4 * i + 1] * X[1] + T[4 * i + 2] * X[2] + T[4 * i + 3];
  const double a = ray_angle(x, y, r);
  return a * a;
}

__device__ __forceinline__ bool positive_depth(const double* T, const double* X) {
  return T[8] * X[0] + T[9] * X[1] + T[10] * X[2] + T[11] >= kDepthEpsilon;
}

__device__ __forceinline__ bool better(int n1, double s1, int n2, double s2) { return n1 > n2 || (n1 == n2 && s1 < s2); }

__device__ __forceinline__ double shfl(double v, int l) { return __shfl_sync(0xffffffffu, v, l); }

// the support of model X over the list (every lane gets it): inliers and their residual sum in lane-strided order
__device__ void warp_support(const Ctx& c, const int* lst, int m, const double* X, int& n, double& sum) {
  int cnt = 0;
  double s = 0.0;
  for (int j = threadIdx.x & 31; j < m; j += 32) {
    double x, y;
    const double* T = observation(c, lst[j], x, y);
    const double r = sq_residual(T, x, y, X);
    if (r <= c.thr) { ++cnt; s += r; }
  }
  n = __reduce_add_sync(0xffffffffu, cnt);
  sum = warp_sum(s);
}

// TriangulationEstimator::Estimate on the inliers of X (more than 2: the multi-view branch): the multi-view DLT, every
// inlier in front of its camera, some pair of inliers at min_angle or more.  Returns false without a model.
__device__ bool local_model(const Ctx& c, const int* lst, int* tmp, int m, const double* X, double* Xl) {
  const int lane = threadIdx.x & 31;
  double A[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) A[a][b] = 0.0;
  int ni = 0;
  for (int j0 = 0; j0 < m; j0 += 32) {
    const int j = j0 + lane;
    bool in = false;
    if (j < m) {
      double x, y;
      const double* T = observation(c, lst[j], x, y);
      in = sq_residual(T, x, y, X) <= c.thr;
      if (in) multi_view_accumulate(T, x, y, A);
    }
    const unsigned b = __ballot_sync(0xffffffffu, in);
    if (in) tmp[ni + __popc(b & ((1u << lane) - 1u))] = lst[j];
    ni += __popc(b);
  }
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) A[a][b] = warp_sum(A[a][b]);
  double v[4];
  smallest_eigenvector<4>(A, v);
  Xl[0] = v[0] / v[3]; Xl[1] = v[1] / v[3]; Xl[2] = v[2] / v[3];
  __syncwarp();
  bool ok = true;
  for (int j = lane; j < ni; j += 32) {
    double x, y;
    if (!positive_depth(observation(c, tmp[j], x, y), Xl)) ok = false;
  }
  if (!__all_sync(0xffffffffu, ok)) return false;
  // pairs (a, b < a) in linear order t = a (a - 1) / 2 + b
  const long long np = (long long)ni * (ni - 1) / 2;
  for (long long t0 = 0; t0 < np; t0 += 32) {
    const long long t = t0 + lane;
    bool hit = false;
    if (t < np) {
      long long a = (long long)((1.0 + sqrt(1.0 + 8.0 * (double)t)) * 0.5);
      while (a * (a - 1) / 2 > t) --a;
      while ((a + 1) * a / 2 <= t) ++a;
      const long long b = t - a * (a - 1) / 2;
      double x, y;
      const double* Ta = observation(c, tmp[a], x, y);
      const double* Tb = observation(c, tmp[b], x, y);
      hit = triangulation_angle(Ta + 12, Tb + 12, Xl) >= c.min_tri;
    }
    if (__any_sync(0xffffffffu, hit)) return true;
  }
  return false;
}

// EstimateTriangulation (LORANSAC, CombinationSampler, InlierSupportMeasurer); X receives the model.  Warp-uniform.
__device__ bool estimate_triangulation(const Ctx& c, const int* lst, int* tmp, int m, double* X, u64& trials, u64& locals) {
  const int lane = threadIdx.x & 31;
  const long long all = (long long)m * (m - 1) / 2;
  const long long max_trials = min(c.trial_cap, all);
  const long long min_trials = m <= kExhaustiveSamplingThreshold ? all : 0;
  long long dyn = max_trials;
  int best_n = 0;
  double best_s = 1.7976931348623157e308;
  bool done = false;
  for (long long base = 0; base < max_trials && !done; base += 32) {
    // this lane's sample: trial base + lane in CombinationSampler order
    const long long t = base + lane;
    bool valid = false;
    int n = 0;
    double s = 0.0, Xs[3] = {0.0, 0.0, 0.0};
    if (t < max_trials) {
      long long i = 0, r = t;
      while (r >= m - 1 - i) { r -= m - 1 - i; ++i; }
      const long long j = i + 1 + r;
      double x1, y1, x2, y2;
      const double* P1 = observation(c, lst[i], x1, y1);
      const double* P2 = observation(c, lst[j], x2, y2);
      double A[4][4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        A[0][k] = x1 * P1[8 + k] - P1[k];
        A[1][k] = y1 * P1[8 + k] - P1[4 + k];
        A[2][k] = x2 * P2[8 + k] - P2[k];
        A[3][k] = y2 * P2[8 + k] - P2[4 + k];
      }
      dlt_point_4x4(A, Xs);
      valid = positive_depth(P1, Xs) && positive_depth(P2, Xs) && triangulation_angle(P1 + 12, P2 + 12, Xs) >= c.min_tri;
      if (valid)
        for (int k = 0; k < m; ++k) {          // in observation order, as InlierSupportMeasurer::Evaluate sums
          double x, y;
          const double* T = observation(c, lst[k], x, y);
          const double rr = sq_residual(T, x, y, Xs);
          if (rr <= c.thr) { ++n; s += rr; }
        }
    }
    // lane-ordered replay of the sequential rules
    for (int l = 0; l < 32; ++l) {
      const long long tl = base + l;
      if (tl >= max_trials) break;
      ++trials;
      if (!__shfl_sync(0xffffffffu, (int)valid, l)) continue;
      const int nl = __shfl_sync(0xffffffffu, n, l);
      const double sl = shfl(s, l);
      if (better(nl, sl, best_n, best_s)) {
        best_n = nl; best_s = sl;
        X[0] = shfl(Xs[0], l); X[1] = shfl(Xs[1], l); X[2] = shfl(Xs[2], l);
        if (nl > kMinNumSamples) {
          for (int r = 0; r < kMaxNumLocalTrials; ++r) {
            const int prev = best_n;
            ++locals;
            double Xl[3];
            if (local_model(c, lst, tmp, m, X, Xl)) {
              int ln;
              double ls;
              warp_support(c, lst, m, Xl, ln, ls);
              if (better(ln, ls, best_n, best_s)) {
                best_n = ln; best_s = ls;
                X[0] = Xl[0]; X[1] = Xl[1]; X[2] = Xl[2];
              }
            }
            if (best_n <= prev) break;
          }
        }
        dyn = compute_num_trials(best_n, m);
      }
      if (tl >= dyn && tl >= min_trials) { done = true; break; }
    }
  }
  return best_n >= kMinNumSamples;
}

// one warp per component, components taken largest first
__global__ void __launch_bounds__(256) k_replay(Ctx c) {
  const int lane = threadIdx.x & 31;
  const unsigned below = (1u << lane) - 1u;
  while (true) {
    int w = 0;
    if (lane == 0) w = (int)atomicAdd(c.cnt + kCntNext, 1ull);
    w = __shfl_sync(0xffffffffu, w, 0);
    if (w >= c.C) return;
    const int comp = c.comp_order[w];
    const int o = c.comp_off[comp], nobs = c.comp_off[comp + 1] - o;
    int* lst = c.lst + o;
    int* tmp = c.tmp + o;
    int npts = 0, nel = 0;
    u64 trials = 0, locals = 0, conts = 0;
    for (int q = 0; q < nobs; ++q) {
      const int k = c.comp_kp[o + q];
      // Find: the correspondences in registered images of non-bogus cameras, in list order
      int L = 0, ntri = 0;
      for (long long e0 = c.list_ptr[k]; e0 < c.list_ptr[k + 1]; e0 += 32) {
        const long long e = e0 + lane;
        const int v = e < c.list_ptr[k + 1] ? c.nbr[e] : -1;
        const bool ok = v >= 0 && c.elig[c.img_of[v]];
        const unsigned b = __ballot_sync(0xffffffffu, ok);
        if (ok) lst[L + __popc(b & below)] = v;
        L += __popc(b);
        ntri += __popc(__ballot_sync(0xffffffffu, ok && c.pt_of[v] >= 0));
      }
      __syncwarp();
      if (L == 0) continue;
      if (ntri > 0 && c.pt_of[k] < 0) {
        // Continue: the existing point with the smallest angular error (the first of equal ones)
        double x, y;
        const double* T = observation(c, k, x, y);
        double best = 1.7976931348623157e308;
        int bi = 0x7fffffff;
        for (int j = lane; j < L; j += 32) {
          const int p = c.pt_of[lst[j]];
          if (p < 0) continue;
          const double* Xp = c.pt_xyz + 3 * (size_t)p;
          double r[3];
          quat::qrotate(quat::load_q(T + 15), Xp, r);       // CalculateAngularError: qvec / tvec form
          r[0] += T[19]; r[1] += T[20]; r[2] += T[21];
          const double err = ray_angle(x, y, r);
          if (err < best) { best = err; bi = j; }
        }
        for (int d = 16; d > 0; d >>= 1) {
          const double ob = shfl(best, lane ^ d);
          const int oi = __shfl_xor_sync(0xffffffffu, bi, d);
          if (ob < best || (ob == best && oi < bi)) { best = ob; bi = oi; }
        }
        if (bi != 0x7fffffff && best <= c.cont_max) {
          const int p = c.pt_of[lst[bi]];
          if (lane == 0) {
            c.pt_of[k] = p;
            c.el_slot[o + nel] = p;
            c.el_kp[o + nel] = k;
          }
          ++nel;
          ++conts;
        }
        __syncwarp();
      }
      // Create: the list with the reference observation last, without the observations that have a point
      if (lane == 0) lst[L] = k;
      __syncwarp();
      int cur = 0;
      for (int j0 = 0; j0 <= L; j0 += 32) {
        const int j = j0 + lane;
        const int v = j <= L ? lst[j] : -1;
        const bool keep = v >= 0 && c.pt_of[v] < 0;
        const unsigned b = __ballot_sync(0xffffffffu, keep);
        if (keep) lst[cur + __popc(b & below)] = v;
        cur += __popc(b);
      }
      __syncwarp();
      while (cur >= 2) {
        if (c.ignore_two_view && cur == 2) {      // IsTwoViewObservation of the first observation
          const int a = lst[0];
          if (c.deg[a] == 1 && c.deg[c.first_nbr[a]] == 1) break;
        }
        double X[3];
        if (!estimate_triangulation(c, lst, tmp, cur, X, trials, locals)) break;
        const int slot = o + npts;
        if (lane == 0) {
          c.pt_xyz[3 * (size_t)slot] = X[0]; c.pt_xyz[3 * (size_t)slot + 1] = X[1]; c.pt_xyz[3 * (size_t)slot + 2] = X[2];
          c.pt_creator[slot] = (unsigned)k;
        }
        // the inliers become the point's track in list order, the outliers the next list
        int nout = 0;
        for (int j0 = 0; j0 < cur; j0 += 32) {
          const int j = j0 + lane;
          bool in = false;
          int v = -1;
          if (j < cur) {
            v = lst[j];
            double x, y;
            const double* T = observation(c, v, x, y);
            in = sq_residual(T, x, y, X) <= c.thr;
          }
          const unsigned bi = __ballot_sync(0xffffffffu, in);
          const unsigned bo = __ballot_sync(0xffffffffu, j < cur && !in);
          if (in) {
            const int e = o + nel + __popc(bi & below);
            c.el_slot[e] = slot; c.el_kp[e] = v;
            c.pt_of[v] = slot;
          } else if (j < cur) {
            lst[nout + __popc(bo & below)] = v;
          }
          nel += __popc(bi);
          nout += __popc(bo);
        }
        __syncwarp();
        ++npts;
        cur = nout;
      }
    }
    if (lane == 0) {
      atomicAdd(c.cnt + kCntPoints, (u64)npts);
      atomicAdd(c.cnt + kCntElements, (u64)nel);
      atomicAdd(c.cnt + kCntContinued, conts);
      atomicAdd(c.cnt + kCntTrials, trials);
      atomicAdd(c.cnt + kCntLocal, locals);
    }
  }
}

// ---- assembly ------------------------------------------------------------------------------------------------------
__global__ void k_scratch_init(int A, unsigned* __restrict__ creator, int* __restrict__ slot, int* __restrict__ el_slot) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= A) return;
  creator[s] = kNone; slot[s] = s; el_slot[s] = -1;
}

__global__ void k_point_ids(int P, const int* __restrict__ sorted_slot, const double* __restrict__ pt_xyz, int* __restrict__ new_id,
                            double* __restrict__ xyz) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= P) return;
  const int s = sorted_slot[r];
  new_id[s] = r;
  for (int i = 0; i < 3; ++i) xyz[3 * (size_t)r + i] = pt_xyz[3 * (size_t)s + i];
}

__global__ void k_elem_keys(int A, const int* __restrict__ el_slot, const int* __restrict__ new_id, unsigned* __restrict__ key) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= A) return;
  key[s] = el_slot[s] >= 0 ? (unsigned)new_id[el_slot[s]] : kNone;
}

__global__ void k_tracks(int P, int E, const unsigned* __restrict__ key, const int* __restrict__ kp, const int* __restrict__ img_of,
                         const long long* __restrict__ kp_ptr, long long* __restrict__ track_ptr, int* __restrict__ track_image,
                         int* __restrict__ track_p2d) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i <= P) {
    int lo = 0, hi = E;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (key[mid] < (unsigned)i) lo = mid + 1;
      else hi = mid;
    }
    track_ptr[i] = lo;
  }
  if (i < E) {
    const int f = img_of[kp[i]];
    track_image[i] = f;
    track_p2d[i] = (int)(kp[i] - kp_ptr[f]);
  }
}

__global__ void k_kp_points(long long K, const int* __restrict__ pt_of, const int* __restrict__ new_id, long long* __restrict__ out) {
  const long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (k >= K) return;
  out[k] = pt_of[k] >= 0 ? new_id[pt_of[k]] : -1;
}

}  // namespace

// ---- hand-off to the bundle adjustment (psfm_ba_create_from_triangulation) ------------------------------------------
namespace {

// flag[k] = 1 when keypoint k lies in a registered image and has a point; flag[K] stays 0 for the scan's total
__global__ void k_obs_flag(long long K, const long long* __restrict__ kp_points, const int* __restrict__ img_of,
                           const int* __restrict__ rank, int* __restrict__ flag) {
  const long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (k >= K) return;
  flag[k] = (kp_points[k] >= 0 && rank[img_of[k]] >= 0) ? 1 : 0;
}

__global__ void k_obs_scatter(long long K, const int* __restrict__ flag, const int* __restrict__ pos,
                              const long long* __restrict__ kp_points, const int* __restrict__ img_of,
                              const int* __restrict__ rank, const float2* __restrict__ kps, int* __restrict__ obs_image,
                              int* __restrict__ obs_point, double2* __restrict__ obs_xy, int* __restrict__ obs_kp) {
  const long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (k >= K || !flag[k]) return;
  const int m = pos[k];
  const float2 x = kps[k];
  obs_image[m] = rank[img_of[k]];
  obs_point[m] = (int)kp_points[k];
  obs_xy[m] = make_double2((double)x.x, (double)x.y);
  obs_kp[m] = (int)k;
}

}  // namespace

long long psfm::triangulation_observations(const psfm_triangulation* h, const int* image_rank, cudaStream_t st,
                                           DBuf<int>& obs_image, DBuf<int>& obs_point, DBuf<double2>& obs_xy,
                                           DBuf<int>& obs_kp) {
  const long long K = h->K;
  DBuf<int> rank, flag, pos;
  rank.alloc(h->F, st); flag.alloc(K + 1, st); pos.alloc(K + 1, st);
  rank.upload(image_rank, h->F, st);
  flag.zero(st);
  if (K) { k_obs_flag<<<grid_of(K), 256, 0, st>>>(K, h->kp_points.p, h->img_of.p, rank.p, flag.p); PSFM_LAUNCH_CHECK(); }
  size_t bytes = 0;
  PSFM_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, flag.p, pos.p, K + 1, st));
  DBuf<unsigned char> tmp;
  tmp.alloc(bytes, st);
  PSFM_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, bytes, flag.p, pos.p, K + 1, st));
  PSFM_LAUNCH_CHECK();
  int M = 0;
  PSFM_CUDA(cudaMemcpyAsync(&M, pos.p + K, sizeof(int), cudaMemcpyDeviceToHost, st));
  PSFM_CUDA(cudaStreamSynchronize(st));
  obs_image.alloc(M, st); obs_point.alloc(M, st); obs_xy.alloc(M, st); obs_kp.alloc(M, st);
  if (K) {
    k_obs_scatter<<<grid_of(K), 256, 0, st>>>(K, flag.p, pos.p, h->kp_points.p, h->img_of.p, rank.p, h->kps.p, obs_image.p,
                                              obs_point.p, obs_xy.p, obs_kp.p);
    PSFM_LAUNCH_CHECK();
  }
  return M;
}

extern "C" void psfm_triangulator_default_options(psfm_triangulator_options* o) {
  if (!o) return;
  o->max_transitivity = 1;
  o->create_max_angle_error = 2.0;
  o->continue_max_angle_error = 2.0;
  o->min_angle = 1.5;
  o->ignore_two_view_tracks = 1;
  o->min_focal_length_ratio = 0.1;
  o->max_focal_length_ratio = 10.0;
  o->max_extra_param = 1.0;
}

extern "C" int psfm_triangulation_create(int32_t num_images, const int64_t* keypoint_ptr, const float* keypoints,
                                         const int32_t* image_camera, const double* cameras, int32_t num_cameras,
                                         const int32_t* camera_size, int64_t num_pairs, const int32_t* pair_images,
                                         const int64_t* inlier_ptr, const uint32_t* inlier_matches, const uint8_t* pair_used,
                                         const double* orientations, const double* image_tvec, const uint8_t* registered,
                                         const psfm_triangulator_options* opts, psfm_triangulation** out,
                                         int64_t* num_points3D, int64_t* num_track_elements) {
  return guard("psfm_triangulation_create", [&]() -> int {
    const auto t0 = std::chrono::steady_clock::now();
    const long long launches0 = g_launch_count.load();
    const char* entry = "psfm_triangulation_create";
    if (!out) return fail(entry, PSFM_ERR_INVALID, "null argument");
    *out = nullptr;
    int rc = check_sizes(entry, num_images, num_cameras, num_pairs);
    if (rc != PSFM_OK) return rc;
    if (!keypoint_ptr || (num_images > 0 && (!image_camera || !orientations || !image_tvec || !registered)) ||
        (num_cameras > 0 && (!cameras || !camera_size)) || (num_pairs > 0 && (!pair_images || !inlier_ptr)))
      return fail(entry, PSFM_ERR_INVALID, "null argument");
    psfm_triangulator_options o;
    psfm_triangulator_default_options(&o);
    if (opts) o = *opts;
    if (!(o.max_transitivity >= 0 && o.create_max_angle_error > 0 && o.continue_max_angle_error > 0 && o.min_angle > 0 &&
          o.min_focal_length_ratio > 0 && o.max_focal_length_ratio > 0 && o.max_extra_param >= 0 &&
          std::isfinite(o.create_max_angle_error) && std::isfinite(o.continue_max_angle_error) && std::isfinite(o.min_angle) &&
          std::isfinite(o.min_focal_length_ratio) && std::isfinite(o.max_focal_length_ratio) && std::isfinite(o.max_extra_param)))
      return fail(entry, PSFM_ERR_INVALID, "options fail the IncrementalTriangulator::Options Check()");
    if (o.max_transitivity != 1) return fail(entry, PSFM_ERR_UNSUPPORTED, "max_transitivity != 1 is not supported");
    const int F = num_images, R = (int)num_pairs;
    if ((rc = check_keypoint_ptr(entry, F, keypoint_ptr)) != PSFM_OK) return rc;
    const long long K = keypoint_ptr[F];
    if (K >= 0x7fffffffLL) return fail(entry, PSFM_ERR_UNSUPPORTED, "2^31 - 1 keypoints or more");
    if (K > 0 && !keypoints) return fail(entry, PSFM_ERR_INVALID, "null argument");
    if ((rc = check_image_cameras(entry, F, image_camera, num_cameras)) != PSFM_OK) return rc;
    if ((rc = check_camera_sizes(entry, num_cameras, camera_size)) != PSFM_OK) return rc;
    if (R > 0) {
      if ((rc = check_match_ptr(entry, "inlier_ptr", R, inlier_ptr)) != PSFM_OK) return rc;
      if ((rc = check_pair_images(entry, R, pair_images, F)) != PSFM_OK) return rc;
      if ((rc = check_distinct_pairs(entry, R, pair_images)) != PSFM_OK) return rc;
      if (inlier_ptr[R] > 0 && !inlier_matches) return fail(entry, PSFM_ERR_INVALID, "null argument");
      if ((rc = check_match_keypoints(entry, R, pair_images, keypoint_ptr, inlier_ptr, inlier_matches)) != PSFM_OK) return rc;
    }
    // per image: P = [R | t], the projection centre -R' t, qvec, tvec; eligible = registered with a non-bogus camera
    // (Camera::HasBogusParams, SIMPLE_PINHOLE: principal point in [0, w] x [0, h], f / max(w, h) in the ratio range)
    std::vector<double> img((size_t)kImg * F, 0.0);
    std::vector<unsigned char> elig(F, 0);
    for (int f = 0; f < F; ++f) {
      if (!registered[f]) continue;
      const double* q = orientations + 4 * (size_t)f;
      const double* t = image_tvec + 3 * (size_t)f;
      for (int i = 0; i < 4; ++i)
        if (!std::isfinite(q[i])) return fail(entry, PSFM_ERR_INVALID, "a registered image with a non-finite pose");
      for (int i = 0; i < 3; ++i)
        if (!std::isfinite(t[i])) return fail(entry, PSFM_ERR_INVALID, "a registered image with a non-finite pose");
      const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
      if (!(n > 0.0)) return fail(entry, PSFM_ERR_INVALID, "a registered image with a non-finite pose");
      const double w = q[0] / n, x = q[1] / n, y = q[2] / n, z = q[3] / n;
      const double Rm[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                            2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                            2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)};
      double* T = img.data() + (size_t)kImg * f;
      for (int r = 0; r < 3; ++r) {
        for (int cc = 0; cc < 3; ++cc) T[4 * r + cc] = Rm[3 * r + cc];
        T[4 * r + 3] = t[r];
      }
      for (int cc = 0; cc < 3; ++cc) T[12 + cc] = -(Rm[cc] * t[0] + Rm[3 + cc] * t[1] + Rm[6 + cc] * t[2]);
      for (int i = 0; i < 4; ++i) T[15 + i] = q[i];
      for (int i = 0; i < 3; ++i) T[19 + i] = t[i];
      const int cam = image_camera[f];
      const double fl = cameras[3 * cam], cx = cameras[3 * cam + 1], cy = cameras[3 * cam + 2];
      const double wd = camera_size[2 * cam], ht = camera_size[2 * cam + 1];
      const bool bogus_pp = cx < 0 || cx > wd || cy < 0 || cy > ht;
      const double ratio = fl / std::max(wd, ht);
      elig[f] = !(bogus_pp || ratio < o.min_focal_length_ratio || ratio > o.max_focal_length_ratio);
    }
    if ((rc = require_device(entry)) != PSFM_OK) return rc;
    const long long N = R > 0 ? inlier_ptr[R] : 0, E = 2 * N;
    psfm_triangulation_summary sm;
    memset(&sm, 0, sizeof(sm));
    sm.host_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    std::unique_ptr<psfm_triangulation> h(new psfm_triangulation());
    Event ev[5];
    // the keypoints, their images and keypoint_ptr stay with the handle for psfm_ba_create_from_triangulation
    DBuf<long long>& d_kp_ptr = h->kp_ptr;
    DBuf<float2>& d_kps = h->kps;
    DBuf<int>& d_img_of = h->img_of;
    h->F = F; h->C = num_cameras;
    h->h_kp_ptr.assign(keypoint_ptr, keypoint_ptr + F + 1);
    h->image_camera.assign(image_camera, image_camera + F);
    h->registered.assign(registered, registered + F);
    DBuf<long long> d_iptr, d_list_ptr;
    DBuf<int> d_cam_of, d_pt_of, d_parent, d_deg, d_first, d_nbr;
    DBuf<int2> d_pairs;
    DBuf<uint2> d_m;
    DBuf<double> d_cams, d_img;
    DBuf<unsigned char> d_elig, d_used, d_acc, d_flag, d_active;
    DBuf<unsigned> d_key0, d_key1;
    DBuf<u64> d_val0, d_val1, d_cnt;
    d_kp_ptr.alloc(F + 1); d_kps.alloc(K); d_cam_of.alloc(F); d_img_of.alloc(K); d_pt_of.alloc(K); d_parent.alloc(K);
    d_deg.alloc(K); d_first.alloc(K); d_active.alloc(K); d_list_ptr.alloc(K + 1);
    d_cams.alloc(3 * (size_t)num_cameras); d_img.alloc((size_t)kImg * F); d_elig.alloc(F);
    d_iptr.alloc(R + 1); d_pairs.alloc(R); d_flag.alloc(R); d_m.alloc(N); d_acc.alloc(N);
    d_key0.alloc(E); d_key1.alloc(E); d_val0.alloc(E); d_val1.alloc(E); d_cnt.alloc(kCntNum);
    d_kp_ptr.upload(reinterpret_cast<const long long*>(keypoint_ptr), F + 1, nullptr);
    d_kps.upload(reinterpret_cast<const float2*>(keypoints), K, nullptr);
    d_cam_of.upload(image_camera, F, nullptr);
    d_cams.upload(cameras, 3 * (size_t)num_cameras, nullptr);
    d_img.upload(img.data(), img.size(), nullptr);
    d_elig.upload(elig.data(), F, nullptr);
    if (R > 0) {
      d_iptr.upload(reinterpret_cast<const long long*>(inlier_ptr), R + 1, nullptr);
      d_pairs.upload(reinterpret_cast<const int2*>(pair_images), R, nullptr);
      d_m.upload(reinterpret_cast<const uint2*>(inlier_matches), N, nullptr);
      if (pair_used) { d_used.alloc(R); d_used.upload(pair_used, R, nullptr); }
    }
    d_flag.zero(nullptr); d_cnt.zero(nullptr);
    const unsigned sentinel = (unsigned)K;
    PSFM_CUDA(cudaEventRecord(ev[0], nullptr));
    // ---- graph
    k_kp_image<<<std::max(F, 1), 256>>>(F, d_kp_ptr.p, d_img_of.p, d_pt_of.p, d_parent.p, d_active.p);
    PSFM_LAUNCH_CHECK();
    k_entries<<<std::max(R, 1), 256>>>(R, d_iptr.p, d_pairs.p, pair_used ? d_used.p : nullptr, d_kp_ptr.p, d_m.p, d_key0.p,
                                       d_val0.p, d_acc.p, sentinel);
    PSFM_LAUNCH_CHECK();
    cub::DoubleBuffer<unsigned> keys(d_key0.p, d_key1.p);
    cub::DoubleBuffer<u64> vals(d_val0.p, d_val1.p);
    sort_pairs(keys, vals, E, key_bits((unsigned long long)K));
    const unsigned* skey = keys.Current();
    const u64* sval = vals.Current();
    d_nbr.alloc(E);
    k_list_ptr<<<grid_of(K + 1), 256>>>(K, E, skey, d_list_ptr.p);
    PSFM_LAUNCH_CHECK();
    k_neighbours<<<grid_stride_of(E), 256>>>(E, skey, sval, sentinel, d_iptr.p, R, d_pairs.p, d_kp_ptr.p, d_m.p, d_img_of.p,
                                             d_nbr.p, d_flag.p);
    PSFM_LAUNCH_CHECK();
    k_dedupe<<<grid_of(R), 256>>>(R, d_flag.p, d_iptr.p, d_pairs.p, d_kp_ptr.p, d_m.p, d_list_ptr.p, sval, d_acc.p);
    PSFM_LAUNCH_CHECK();
    k_drop<<<grid_stride_of(E), 256>>>(E, sval, d_acc.p, d_nbr.p);
    PSFM_LAUNCH_CHECK();
    k_degree<<<grid_of(K), 256>>>(K, d_list_ptr.p, d_nbr.p, d_deg.p, d_first.p);
    PSFM_LAUNCH_CHECK();
    PSFM_CUDA(cudaEventRecord(ev[1], nullptr));
    // ---- components
    k_uf_hook<<<grid_stride_of(E), 256>>>(E, skey, d_nbr.p, d_img_of.p, d_elig.p, d_parent.p, d_active.p);
    PSFM_LAUNCH_CHECK();
    // only the neighbour lists stay: 8 bytes per match
    d_m.release(); d_acc.release(); d_val0.release(); d_val1.release(); d_key0.release(); d_key1.release();
    DBuf<unsigned> c_key0, c_key1;
    DBuf<int> c_val0, c_val1;
    c_key0.alloc(K); c_key1.alloc(K); c_val0.alloc(K); c_val1.alloc(K);
    k_uf_label<<<grid_of(K), 256>>>(K, d_parent.p, d_active.p, c_key0.p, c_val0.p, d_cnt.p);
    PSFM_LAUNCH_CHECK();
    cub::DoubleBuffer<unsigned> ckeys(c_key0.p, c_key1.p);
    cub::DoubleBuffer<int> cvals(c_val0.p, c_val1.p);
    sort_pairs(ckeys, cvals, K, 32);
    u64 cnt_h[kCntNum];
    PSFM_CUDA(cudaMemcpy(cnt_h, d_cnt.p, sizeof(cnt_h), cudaMemcpyDeviceToHost));
    const int A = (int)cnt_h[kCntActive];
    DBuf<int> d_head, d_cid, d_comp_off;
    d_head.alloc(A); d_cid.alloc(A); d_comp_off.alloc(A + 1);
    k_comp_heads<<<grid_of(A), 256>>>(A, ckeys.Current(), d_head.p);
    PSFM_LAUNCH_CHECK();
    {
      size_t bytes = 0;
      PSFM_CUDA(cub::DeviceScan::InclusiveSum(nullptr, bytes, d_head.p, d_cid.p, A, nullptr));
      DBuf<unsigned char> tmp;
      tmp.alloc(bytes);
      PSFM_CUDA(cub::DeviceScan::InclusiveSum(tmp.p, bytes, d_head.p, d_cid.p, A, nullptr));
      PSFM_LAUNCH_CHECK();
    }
    k_comp_bounds<<<grid_of(A), 256>>>(A, d_head.p, d_cid.p, d_comp_off.p);
    PSFM_LAUNCH_CHECK();
    int C = 0;
    if (A > 0) PSFM_CUDA(cudaMemcpy(&C, d_cid.p + (A - 1), sizeof(int), cudaMemcpyDeviceToHost));
    DBuf<unsigned> o_key0, o_key1;
    DBuf<int> o_val0, o_val1;
    o_key0.alloc(C); o_key1.alloc(C); o_val0.alloc(C); o_val1.alloc(C);
    k_comp_sizes<<<grid_of(C), 256>>>(C, d_comp_off.p, o_key0.p, o_val0.p);
    PSFM_LAUNCH_CHECK();
    cub::DoubleBuffer<unsigned> okeys(o_key0.p, o_key1.p);
    cub::DoubleBuffer<int> ovals(o_val0.p, o_val1.p);
    sort_pairs(okeys, ovals, C, 32);
    PSFM_CUDA(cudaEventRecord(ev[2], nullptr));
    // ---- replay
    DBuf<int> d_lst, d_tmp, d_slot0, d_slot1, d_el_slot, d_el_kp, d_new_id;
    DBuf<double> d_pt_xyz;
    DBuf<unsigned> d_creator0, d_creator1;
    d_lst.alloc(A); d_tmp.alloc(A); d_slot0.alloc(A); d_slot1.alloc(A); d_el_slot.alloc(A); d_el_kp.alloc(A);
    d_new_id.alloc(A); d_pt_xyz.alloc(3 * (size_t)A); d_creator0.alloc(A); d_creator1.alloc(A);
    k_scratch_init<<<grid_of(A), 256>>>(A, d_creator0.p, d_slot0.p, d_el_slot.p);
    PSFM_LAUNCH_CHECK();
    Ctx c;
    c.kps = d_kps.p; c.img_of = d_img_of.p; c.cam_of = d_cam_of.p; c.cams = d_cams.p;
    c.img = d_img.p; c.elig = d_elig.p; c.list_ptr = d_list_ptr.p; c.nbr = d_nbr.p; c.deg = d_deg.p;
    c.first_nbr = d_first.p; c.comp_kp = cvals.Current(); c.comp_off = d_comp_off.p; c.comp_order = ovals.Current();
    c.C = C; c.pt_of = d_pt_of.p; c.lst = d_lst.p; c.tmp = d_tmp.p; c.pt_xyz = d_pt_xyz.p; c.pt_creator = d_creator0.p;
    c.el_slot = d_el_slot.p; c.el_kp = d_el_kp.p; c.cnt = d_cnt.p;
    const double deg2rad = M_PI / 180.0;
    c.thr = (o.create_max_angle_error * deg2rad) * (o.create_max_angle_error * deg2rad);
    c.cont_max = o.continue_max_angle_error * deg2rad;
    c.min_tri = o.min_angle * deg2rad;
    c.ignore_two_view = o.ignore_two_view_tracks != 0;
    c.trial_cap = std::min(kMaxNumTrials, compute_num_trials((long long)(kMinInlierRatio * kCapNumSamples), kCapNumSamples));
    k_replay<<<(unsigned)std::max(1, std::min((C + 7) / 8, 132 * 8)), 256>>>(c);
    PSFM_LAUNCH_CHECK();
    PSFM_CUDA(cudaEventRecord(ev[3], nullptr));
    PSFM_CUDA(cudaMemcpy(cnt_h, d_cnt.p, sizeof(cnt_h), cudaMemcpyDeviceToHost));
    const int P = (int)cnt_h[kCntPoints], NE = (int)cnt_h[kCntElements];
    // ---- assembly
    cub::DoubleBuffer<unsigned> pkeys(d_creator0.p, d_creator1.p);
    cub::DoubleBuffer<int> pvals(d_slot0.p, d_slot1.p);
    sort_pairs(pkeys, pvals, A, 32);
    h->xyz.alloc(3 * (size_t)P); h->track_ptr.alloc(P + 1); h->track_image.alloc(NE); h->track_p2d.alloc(NE);
    h->kp_points.alloc(K);
    k_point_ids<<<grid_of(P), 256>>>(P, pvals.Current(), d_pt_xyz.p, d_new_id.p, h->xyz.p);
    PSFM_LAUNCH_CHECK();
    DBuf<unsigned> e_key0, e_key1;
    DBuf<int> e_val1;
    e_key0.alloc(A); e_key1.alloc(A); e_val1.alloc(A);
    k_elem_keys<<<grid_of(A), 256>>>(A, d_el_slot.p, d_new_id.p, e_key0.p);
    PSFM_LAUNCH_CHECK();
    cub::DoubleBuffer<unsigned> ekeys(e_key0.p, e_key1.p);
    cub::DoubleBuffer<int> evals(d_el_kp.p, e_val1.p);
    sort_pairs(ekeys, evals, A, 32);
    k_tracks<<<grid_of(std::max(P + 1, NE)), 256>>>(P, NE, ekeys.Current(), evals.Current(), d_img_of.p, d_kp_ptr.p,
                                                     h->track_ptr.p, h->track_image.p, h->track_p2d.p);
    PSFM_LAUNCH_CHECK();
    k_kp_points<<<grid_of(K), 256>>>(K, d_pt_of.p, d_new_id.p, h->kp_points.p);
    PSFM_LAUNCH_CHECK();
    PSFM_CUDA(cudaEventRecord(ev[4], nullptr));
    PSFM_CUDA(cudaEventSynchronize(ev[4]));
    float ms[4];
    for (int i = 0; i < 4; ++i) PSFM_CUDA(cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]));
    sm.graph_ms = ms[0]; sm.components_ms = ms[1]; sm.replay_ms = ms[2]; sm.assembly_ms = ms[3];
    sm.num_components = C;
    if (C > 0) {
      unsigned k0 = 0;
      PSFM_CUDA(cudaMemcpy(&k0, okeys.Current(), sizeof(unsigned), cudaMemcpyDeviceToHost));
      sm.largest_component = kNone - k0;
    }
    sm.num_points3D = P;
    sm.num_continued = (long long)cnt_h[kCntContinued];
    sm.num_ransac_trials = (long long)cnt_h[kCntTrials];
    sm.num_local_estimates = (long long)cnt_h[kCntLocal];
    h->P = P; h->E = NE; h->K = K;
    sm.num_launches = g_launch_count.load() - launches0;
    h->summary = sm;
    if (num_points3D) *num_points3D = h->P;
    if (num_track_elements) *num_track_elements = h->E;
    *out = h.release();
    return PSFM_OK;
  });
}

extern "C" int psfm_triangulation_result(const psfm_triangulation* h, double* xyz, int64_t* track_ptr, int32_t* track_image,
                                         int32_t* track_point2D, int64_t* point3D_of_keypoint,
                                         psfm_triangulation_summary* summary) {
  return guard("psfm_triangulation_result", [&]() -> int {
    if (!h) {
      set_error("psfm_triangulation_result: null handle");
      return PSFM_ERR_INVALID;
    }
    if (xyz && h->P) PSFM_CUDA(cudaMemcpy(xyz, h->xyz.p, sizeof(double) * 3 * (size_t)h->P, cudaMemcpyDeviceToHost));
    if (track_ptr) PSFM_CUDA(cudaMemcpy(track_ptr, h->track_ptr.p, sizeof(int64_t) * (size_t)(h->P + 1), cudaMemcpyDeviceToHost));
    if (track_image && h->E) PSFM_CUDA(cudaMemcpy(track_image, h->track_image.p, sizeof(int32_t) * (size_t)h->E, cudaMemcpyDeviceToHost));
    if (track_point2D && h->E) PSFM_CUDA(cudaMemcpy(track_point2D, h->track_p2d.p, sizeof(int32_t) * (size_t)h->E, cudaMemcpyDeviceToHost));
    if (point3D_of_keypoint && h->K)
      PSFM_CUDA(cudaMemcpy(point3D_of_keypoint, h->kp_points.p, sizeof(int64_t) * (size_t)h->K, cudaMemcpyDeviceToHost));
    if (summary) *summary = h->summary;
    return PSFM_OK;
  });
}

extern "C" void psfm_triangulation_destroy(psfm_triangulation* h) { delete h; }
