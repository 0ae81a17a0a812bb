// motion_seg.cu — the trajectory labeller's device steps (DESIGN.md §4.17).
//
// Reference: motion_seg/load_cut_seq.py (windows, depth maps, coordinates), core/network/traj_oa_depth.py
// (augment_traj and the transformer encoder) and main_motion_segmentation.py (merge) with core/utils/utils.py
// (draw_traj_cls).  The OANet decoder stays torch calls (particlesfm_b200/motion_seg.py).
//
//   psfm_seg_hits          per window and trajectory, the number of the window's frames the trajectory is seen in.
//   psfm_seg_shuffle       (host) the permutation of 0 .. K-1 that TrajectorySet::sample_inside_window applies to an
//                          over-full window: std::shuffle with std::mt19937(5489).
//   psfm_seg_windows       the padded window arrays of the sampled rows: float64 locations [R][L][2], 0 where the
//                          trajectory is not seen, and the valid mask [R][L].
//   psfm_seg_depth_resize  cv2.imread(png, -1) / 65535.0 resized by cv2.resize(INTER_LINEAR) to 240 x 424 in float64,
//                          then cast to float32.
//   psfm_seg_encode        the fused encoder: coordinates, the 10 input channels, both 1x1 projections, the whole
//                          nn.Transformer (2 + 2 post-norm layers, d = 16, 4 heads, FFN 64) and the max over time,
//                          one warp per window row, the weights in shared memory.
//   psfm_seg_merge         per observation, the label of the first window that sampled its trajectory and holds its
//                          frame (-1: dropped); per trajectory, the first row that sampled it.
//   psfm_seg_draw          draw_traj_cls's four image rows of a window from pixel stamps of cv2.circle.
//
// The depth resize restates cv2's unfused float64 arithmetic with explicit rounding intrinsics, so that the rest of
// the unit (the encoder's dot products) keeps fused multiply-adds.
#include <float.h>
#include <math.h>

#include <algorithm>
#include <numeric>
#include <random>
#include <vector>

#include "psfm_common.cuh"

namespace {

using namespace psfm;

constexpr int kH = 240, kW = 424;      // the network's resolution (example_test.yaml)
constexpr int kD = 16, kF = 64;        // d_model, dim_feedforward

// packed encoder weights (particlesfm_b200/motion_seg.py:pack_encoder): every matrix transposed to [in][out]
constexpr int OFF_P1W = 0, OFF_P1B = 160, OFF_P2W = 176, OFF_P2B = 432, OFF_ENC = 448;
constexpr int ENC_INW = 0, ENC_INB = 768, ENC_OUTW = 816, ENC_OUTB = 1072, ENC_L1W = 1088, ENC_L1B = 2112,
              ENC_L2W = 2176, ENC_L2B = 3200, ENC_N1 = 3216, ENC_N2 = 3248, ENC_SIZE = 3280;
constexpr int OFF_ENC_NORM = OFF_ENC + 2 * ENC_SIZE, OFF_DEC = OFF_ENC_NORM + 32;
constexpr int DEC_SA = 0, DEC_CA = 1088, DEC_L1W = 2176, DEC_L1B = 3200, DEC_L2W = 3264, DEC_L2B = 4288,
              DEC_N1 = 4304, DEC_N2 = 4336, DEC_N3 = 4368, DEC_SIZE = 4400;
constexpr int OFF_DEC_NORM = OFF_DEC + 2 * DEC_SIZE, OFF_KINV = OFF_DEC_NORM + 32;
constexpr int kWeights = OFF_KINV + 9;                 // 15881 floats
constexpr int kWeightsPadded = (kWeights + 3) & ~3;
constexpr int kWarpFloats = 6 * kD;                    // per token: P/Y (16), X/memory (16), scratch (64)
constexpr int kSmemMax = 227 * 1024;

// ----------------------------------------------------------------------------- windows

__global__ void k_hits(const int64_t* __restrict__ ptr, const int32_t* __restrict__ frames, int T,
                       const int32_t* __restrict__ win_start, int num_windows, int L, int32_t* __restrict__ hits) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)T * num_windows) return;
  const int t = (int)(i % T), w = (int)(i / T);
  const int a = win_start[w], b = a + L;
  long long lo = ptr[t], hi = ptr[t + 1];
  long long s = lo, e = hi;                            // first frame >= a
  while (s < e) {
    const long long m = (s + e) >> 1;
    if (frames[m] < a) s = m + 1; else e = m;
  }
  long long u = s;                                      // first frame >= b
  e = hi;
  while (u < e) {
    const long long m = (u + e) >> 1;
    if (frames[m] < b) u = m + 1; else e = m;
  }
  hits[i] = (int32_t)(u - s);
}

__global__ void k_windows(const int64_t* __restrict__ ptr, const int32_t* __restrict__ frames,
                          const double* __restrict__ xy, const int32_t* __restrict__ rows,
                          const int32_t* __restrict__ row_window, int R, const int32_t* __restrict__ win_start, int L,
                          double* __restrict__ loc, uint8_t* __restrict__ valid) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)R * L) return;
  const int r = (int)(i / L), j = (int)(i % L);
  const int t = rows[r];
  const int f = win_start[row_window[r]] + j;
  long long s = ptr[t], e = ptr[t + 1];
  while (s < e) {
    const long long m = (s + e) >> 1;
    if (frames[m] < f) s = m + 1; else e = m;
  }
  const bool hit = s < ptr[t + 1] && frames[s] == f;
  loc[2 * i] = hit ? xy[2 * s] : 0.0;
  loc[2 * i + 1] = hit ? xy[2 * s + 1] : 0.0;
  valid[i] = hit ? 1 : 0;
}

// ----------------------------------------------------------------------------- depth

// the bilinear resize of a float64 image as cv2 computes it to within float64 rounding: the source coordinate
// (d + 0.5) / (dst / src) - 0.5 and the weights 1 - a and a in float64; a coordinate left of the first or right of the
// last source sample takes that sample.  Cast to float32, this equals cv2.resize(INTER_LINEAR) of the float64 map.
__device__ __forceinline__ void cv_linear(int d, double scale, int n, int& s0, int& s1, double& a) {
  double f = __dsub_rn(__dmul_rn(d + 0.5, scale), 0.5);
  int s = (int)floor(f);
  f = __dsub_rn(f, (double)s);
  if (s < 0) { s = 0; f = 0.0; }
  if (s >= n - 1) { s = n - 1; f = 0.0; }
  s0 = s;
  s1 = min(s + 1, n - 1);
  a = f;
}

__global__ void k_depth_resize(const uint16_t* __restrict__ px, int h, int w, double scale_x, double scale_y,
                               float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= kH * kW) return;
  const int frame = blockIdx.y;
  const int X = i % kW, Y = i / kW;
  int x0, x1, y0, y1;
  double ax, ay;
  cv_linear(X, scale_x, w, x0, x1, ax);
  cv_linear(Y, scale_y, h, y0, y1, ay);
  const uint16_t* img = px + (long long)frame * h * w;
  const double bx0 = __dsub_rn(1.0, ax), bx1 = ax;
  auto row = [&](int y) {
    const double v0 = (double)img[(long long)y * w + x0] / 65535.0, v1 = (double)img[(long long)y * w + x1] / 65535.0;
    return __dadd_rn(__dmul_rn(v0, bx0), __dmul_rn(v1, bx1));
  };
  const double r0 = row(y0), r1 = row(y1);
  out[(long long)frame * kH * kW + i] = (float)__dadd_rn(__dmul_rn(r0, __dsub_rn(1.0, ay)), __dmul_rn(r1, ay));
}

// ----------------------------------------------------------------------------- encoder

// out[t][o] = b[o] + sum_k in[t][k] W[k][o] for t < L, o < NOUT; W has row stride ws.  Lanes run over (t, o).
template <int NIN, int NOUT, bool RELU>
__device__ __forceinline__ void linear(const float* in, int is, const float* W, int ws, const float* b, float* out,
                                       int os, int L, int lane) {
  for (int idx = lane; idx < L * NOUT; idx += 32) {
    const int t = idx / NOUT, o = idx - t * NOUT;
    const float* x = in + t * is;
    float acc = b[o];
#pragma unroll
    for (int k = 0; k < NIN; ++k) acc += x[k] * W[k * ws + o];
    out[t * os + o] = RELU ? fmaxf(acc, 0.f) : acc;
  }
}

__device__ __forceinline__ float sum16(float v) {
#pragma unroll
  for (int m = 8; m >= 1; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
  return v;
}

// LayerNorm(16, eps 1e-5) of one token's value v held by 16 consecutive lanes
__device__ __forceinline__ float layer_norm(float v, const float* g, const float* beta, int o) {
  const float mean = sum16(v) * (1.f / kD);
  const float d = v - mean;
  const float var = sum16(d * d) * (1.f / kD);
  return d * rsqrtf(var + 1e-5f) * g[o] + beta[o];
}

// X[t] = LayerNorm(X[t] + in[t] W + b) for the [L][16] state X; 16 lanes per token, every lane takes part in the
// shuffles
template <int NIN>
__device__ __forceinline__ void linear_residual_norm(const float* in, int is, const float* W, const float* b,
                                                     const float* g, const float* beta, float* X, int L, int lane) {
  for (int base = 0; base < L * kD; base += 32) {
    const int idx = base + lane, t = idx >> 4, o = idx & 15;
    const bool live = t < L;
    float v = 0.f;
    if (live) {
      const float* x = in + t * is;
      float acc = b[o];
#pragma unroll
      for (int k = 0; k < NIN; ++k) acc += x[k] * W[k * kD + o];
      v = X[idx] + acc;
    }
    const float y = layer_norm(v, g, beta, o);
    if (live) X[idx] = y;
  }
}

__device__ __forceinline__ void norm_only(const float* g, const float* beta, float* X, int L, int lane) {
  for (int base = 0; base < L * kD; base += 32) {
    const int idx = base + lane, o = idx & 15;
    const bool live = (idx >> 4) < L;
    const float y = layer_norm(live ? X[idx] : 0.f, g, beta, o);
    if (live) X[idx] = y;
  }
}

// multi-head attention of 4 heads of width 4: A[t] = softmax(q_t k_s / 2 over keys s) v_s, keys with valid[s] = 0
// left out when valid is given.  Q, K, V rows have stride qs; A has stride 16.  Lanes run over (t, head).
__device__ __forceinline__ void attention(const float* Q, const float* K, const float* V, int qs,
                                          const uint8_t* valid, float* A, int L, int lane) {
  for (int idx = lane; idx < L * 4; idx += 32) {
    const int t = idx >> 2, h = (idx & 3) * 4;
    const float q0 = Q[t * qs + h] * 0.5f, q1 = Q[t * qs + h + 1] * 0.5f, q2 = Q[t * qs + h + 2] * 0.5f,
                q3 = Q[t * qs + h + 3] * 0.5f;
    float mx = -INFINITY;
    for (int s = 0; s < L; ++s) {
      if (valid && !valid[s]) continue;
      const float* k = K + s * qs + h;
      mx = fmaxf(mx, q0 * k[0] + q1 * k[1] + q2 * k[2] + q3 * k[3]);
    }
    float sum = 0.f, a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    for (int s = 0; s < L; ++s) {
      if (valid && !valid[s]) continue;
      const float* k = K + s * qs + h;
      const float* v = V + s * qs + h;
      const float p = expf(q0 * k[0] + q1 * k[1] + q2 * k[2] + q3 * k[3] - mx);
      sum += p;
      a0 += p * v[0];
      a1 += p * v[1];
      a2 += p * v[2];
      a3 += p * v[3];
    }
    const float r = 1.f / sum;
    A[t * kD + h] = a0 * r;
    A[t * kD + h + 1] = a1 * r;
    A[t * kD + h + 2] = a2 * r;
    A[t * kD + h + 3] = a3 * r;
  }
}

// one layer's self-attention block on the state S: S = norm(S + out_proj(attention(S W_in)))
__device__ __forceinline__ void self_attention(const float* w, int n_off, const uint8_t* valid, float* S, float* Z,
                                               int L, int lane) {
  float* A = Z + 48 * L;
  linear<kD, 48, false>(S, kD, w + ENC_INW, 48, w + ENC_INB, Z, 48, L, lane);
  __syncwarp();
  attention(Z, Z + 16, Z + 32, 48, valid, A, L, lane);
  __syncwarp();
  linear_residual_norm<kD>(A, kD, w + ENC_OUTW, w + ENC_OUTB, w + n_off, w + n_off + 16, S, L, lane);
  __syncwarp();
}

// S = norm(S + linear2(relu(linear1(S)))), the hidden [L][64] in the scratch Z
__device__ __forceinline__ void feed_forward(const float* l1w, const float* l1b, const float* l2w, const float* l2b,
                                             const float* g, float* S, float* Z, int L, int lane) {
  linear<kD, kF, true>(S, kD, l1w, kF, l1b, Z, kF, L, lane);
  __syncwarp();
  linear_residual_norm<kF>(Z, kF, l2w, l2b, g, g + 16, S, L, lane);
  __syncwarp();
}

__global__ void __launch_bounds__(256) k_encode(const double* __restrict__ loc, const uint8_t* __restrict__ valid,
                                                const int32_t* __restrict__ row_window,
                                                const int32_t* __restrict__ win_start, int R, int L,
                                                const float* __restrict__ depth, int num_frames, double ratio_w,
                                                double ratio_h, const float* __restrict__ weights,
                                                float* __restrict__ feat) {
  extern __shared__ __align__(16) float smem[];
  float* w = smem;
  for (int i = threadIdx.x; i < kWeights; i += blockDim.x) w[i] = weights[i];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, warps = blockDim.x >> 5;
  float* P = smem + kWeightsPadded + warp * kWarpFloats * L;   // projected input, then the decoder state
  float* X = P + kD * L;                                        // encoder state, then the memory
  float* Z = X + kD * L;                                        // scratch [L][64]
  const float* kinv = w + OFF_KINV;
  for (int r = blockIdx.x * warps + warp; r < R; r += gridDim.x * warps) {
    const uint8_t* vr = valid + (long long)r * L;
    const int f0 = win_start[row_window[r]];
    // augment_traj: xy, motion_2d, xyz, motion_3d in Z[t][0..9]; xy in Z[t][10..11], xyz in Z[t][12..14] for t + 1
    for (int t = lane; t < L; t += 32) {
      const double* p = loc + ((long long)r * L + t) * 2;
      const float x = (float)fmin(fmax(p[0] / ratio_w / (double)kW, 0.0), 1.0);
      const float y = (float)fmin(fmax(p[1] / ratio_h / (double)kH, 0.0), 1.0);
      int g = (int)(y * (float)kH) * kW + (int)(x * (float)kW);
      g = min(max(g, 0), kH * kW - 1);
      const float u = (float)(g % kW), v = (float)(g / kW);
      const int frame = min(f0 + t, num_frames - 1);
      const float d = depth[(long long)frame * kH * kW + g];
      float* z = Z + t * kF;
      z[0] = x;
      z[1] = y;
      z[4] = d * ((kinv[0] * u + kinv[1] * v) + kinv[2]);
      z[5] = d * ((kinv[3] * u + kinv[4] * v) + kinv[5]);
      z[6] = d * ((kinv[6] * u + kinv[7] * v) + kinv[8]);
    }
    __syncwarp();
    for (int t = lane; t < L; t += 32) {
      float* z = Z + t * kF;
      if (t + 1 < L) {
        const float m = vr[t + 1] ? 1.f : 0.f;
        const float* n = Z + (t + 1) * kF;
        z[2] = (n[0] - z[0]) * m;
        z[3] = (n[1] - z[1]) * m;
        z[7] = (n[4] - z[4]) * m;
        z[8] = (n[5] - z[5]) * m;
        z[9] = (n[6] - z[6]) * m;
      } else {
        z[2] = z[3] = z[7] = z[8] = z[9] = 0.f;
      }
    }
    __syncwarp();
    linear<10, kD, true>(Z, kF, w + OFF_P1W, kD, w + OFF_P1B, Z + 16, kF, L, lane);
    __syncwarp();
    linear<kD, kD, true>(Z + 16, kF, w + OFF_P2W, kD, w + OFF_P2B, P, kD, L, lane);
    __syncwarp();
    for (int i = lane; i < L * kD; i += 32) X[i] = P[i];
    __syncwarp();
    // encoder: two post-norm layers with the key padding mask, then the final norm
    for (int l = 0; l < 2; ++l) {
      const float* e = w + OFF_ENC + l * ENC_SIZE;
      self_attention(e, ENC_N1, vr, X, Z, L, lane);
      feed_forward(e + ENC_L1W, e + ENC_L1B, e + ENC_L2W, e + ENC_L2B, e + ENC_N2, X, Z, L, lane);
    }
    norm_only(w + OFF_ENC_NORM, w + OFF_ENC_NORM + 16, X, L, lane);
    __syncwarp();
    // decoder: masked self-attention, cross-attention over every memory row, feed-forward; then the final norm
    for (int l = 0; l < 2; ++l) {
      const float* dl = w + OFF_DEC + l * DEC_SIZE;
      self_attention(dl + DEC_SA, DEC_N1, vr, P, Z, L, lane);
      const float* ca = dl + DEC_CA;
      float* A = Z + 48 * L;
      linear<kD, kD, false>(P, kD, ca + ENC_INW, 48, ca + ENC_INB, Z, 48, L, lane);
      linear<kD, 32, false>(X, kD, ca + ENC_INW + 16, 48, ca + ENC_INB + 16, Z + 16, 48, L, lane);
      __syncwarp();
      attention(Z, Z + 16, Z + 32, 48, nullptr, A, L, lane);
      __syncwarp();
      linear_residual_norm<kD>(A, kD, ca + ENC_OUTW, ca + ENC_OUTB, dl + DEC_N2, dl + DEC_N2 + 16, P, L, lane);
      __syncwarp();
      feed_forward(dl + DEC_L1W, dl + DEC_L1B, dl + DEC_L2W, dl + DEC_L2B, dl + DEC_N3, P, Z, L, lane);
    }
    norm_only(w + OFF_DEC_NORM, w + OFF_DEC_NORM + 16, P, L, lane);
    __syncwarp();
    if (lane < kD) {
      float m = -INFINITY;
      for (int t = 0; t < L; ++t) m = fmaxf(m, P[t * kD + lane]);
      feat[(long long)r * kD + lane] = m;
    }
    __syncwarp();
  }
}

// ----------------------------------------------------------------------------- merge

__global__ void k_merge(const int64_t* __restrict__ ptr, const int32_t* __restrict__ frames, int T,
                        const int32_t* __restrict__ win_start, int num_windows, int L,
                        const int32_t* __restrict__ row_of, const uint8_t* __restrict__ pred,
                        int8_t* __restrict__ labels, int32_t* __restrict__ first_row) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  int first = -1;
  for (int w = 0; w < num_windows; ++w) {
    const int r = row_of[(long long)w * T + t];
    if (r >= 0) { first = r; break; }
  }
  first_row[t] = first;
  for (long long j = ptr[t]; j < ptr[t + 1]; ++j) {
    const int f = frames[j];
    int8_t lab = -1;
    for (int w = 0; w < num_windows; ++w) {
      const int r = row_of[(long long)w * T + t];
      if (r >= 0 && f >= win_start[w] && f < win_start[w] + L) { lab = pred[r] ? 1 : 0; break; }
    }
    labels[j] = lab;
  }
}

// ----------------------------------------------------------------------------- drawing

__constant__ uint8_t kColors[6][3] = {{255, 0, 0}, {0, 255, 0}, {0, 0, 255}, {255, 255, 0}, {255, 0, 255}, {0, 255, 255}};

// the circle centre draw_traj_cls uses: int(normalised coordinate * resolution), the coordinate in float64
__device__ __forceinline__ void centre(const double* p, double ratio_w, double ratio_h, int& cx, int& cy) {
  cx = (int)(fmin(fmax(p[0] / ratio_w / (double)kW, 0.0), 1.0) * (double)kW);
  cy = (int)(fmin(fmax(p[1] / ratio_h / (double)kH, 0.0), 1.0) * (double)kH);
}

__device__ __forceinline__ void stamp(int32_t* img, int cx, int cy, const int16_t* st, int n, int32_t order) {
  for (int k = 0; k < n; ++k) {
    const int x = cx + st[2 * k], y = cy + st[2 * k + 1];
    if (x >= 0 && x < kW && y >= 0 && y < kH) atomicMax(img + y * kW + x, order);
  }
}

// order [L][3][H][W]: rows 0 and 1 take trajectory i + 1 of every valid observation (stamps a and b), row 2 takes
// draw k + 1 of the random trajectories (stamp c)
__global__ void k_draw_stamp(const double* __restrict__ loc, const uint8_t* __restrict__ valid, int K, int L,
                             double ratio_w, double ratio_h, const int32_t* __restrict__ draws, int num_draws,
                             const int16_t* __restrict__ stamps, int na, int nb, int nc, int32_t* __restrict__ order) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long n1 = (long long)K * L;
  int cx, cy;
  if (i < n1) {
    if (!valid[i]) return;
    const int k = (int)(i / L), j = (int)(i % L);
    centre(loc + 2 * i, ratio_w, ratio_h, cx, cy);
    int32_t* img = order + (long long)j * 3 * kH * kW;
    stamp(img, cx, cy, stamps, na, k + 1);
    stamp(img + kH * kW, cx, cy, stamps + 2 * na, nb, k + 1);
  } else if (i < n1 + (long long)num_draws * L) {
    const int d = (int)((i - n1) / L), j = (int)((i - n1) % L);
    const long long e = (long long)draws[d] * L + j;
    if (!valid[e]) return;
    centre(loc + 2 * e, ratio_w, ratio_h, cx, cy);
    stamp(order + ((long long)j * 3 + 2) * kH * kW, cx, cy, stamps + 2 * (na + nb), nc, d + 1);
  }
}

// out [L][4H][W][3] BGR: the frame, the labels, the sampled points, the random trajectories
__global__ void k_draw_colour(const uint8_t* __restrict__ frames, int L, const int32_t* __restrict__ order,
                              const uint8_t* __restrict__ pred, const int32_t* __restrict__ draws,
                              uint8_t* __restrict__ out) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)L * 4 * kH * kW) return;
  const int x = (int)(i % kW);
  const int Y = (int)((i / kW) % (4 * kH));
  const int j = (int)(i / ((long long)4 * kH * kW));
  const int row = Y / kH, y = Y % kH;
  const uint8_t* src = frames + (((long long)j * kH + y) * kW + x) * 3;
  uint8_t* dst = out + i * 3;
  int32_t o = 0;
  if (row > 0) o = order[(((long long)j * 3 + row - 1) * kH + y) * kW + x];
  if (o == 0) {
    dst[0] = src[0];
    dst[1] = src[1];
    dst[2] = src[2];
    return;
  }
  const int c = row == 1 ? (pred[o - 1] ? 1 : 0) : row == 2 ? 0 : draws[o - 1] % 6;
  dst[0] = kColors[c][0];
  dst[1] = kColors[c][1];
  dst[2] = kColors[c][2];
}

int check_window(const char* entry, int num_windows, int L) {
  if (num_windows < 1) return fail(entry, PSFM_ERR_INVALID, "num_windows must be positive");
  if (L < 1) return fail(entry, PSFM_ERR_INVALID, "window length must be positive");
  return PSFM_OK;
}

int encode_warps(int L) {
  const long long per = (long long)kWarpFloats * L * 4;
  return (int)std::min<long long>(8, (kSmemMax - kWeightsPadded * 4) / per);
}

}  // namespace

extern "C" int psfm_seg_max_window(void) {
  return (int)((kSmemMax - kWeightsPadded * 4) / ((long long)kWarpFloats * 4));
}

extern "C" int psfm_seg_hits(const int64_t* d_ptr, const int32_t* d_frames, int32_t num_trajs,
                             const int32_t* d_win_start, int32_t num_windows, int32_t L, int32_t* d_hits,
                             void* stream) {
  const char* entry = "psfm_seg_hits";
  return guard(entry, [&]() -> int {
    if (!d_ptr || !d_frames || !d_win_start || !d_hits) return fail(entry, PSFM_ERR_INVALID, "null argument");
    if (num_trajs < 1) return fail(entry, PSFM_ERR_INVALID, "num_trajs must be positive");
    int rc = check_window(entry, num_windows, L);
    if (rc != PSFM_OK) return rc;
    rc = require_device(entry);
    if (rc != PSFM_OK) return rc;
    const long long n = (long long)num_trajs * num_windows;
    k_hits<<<grid_of(n), 256, 0, (cudaStream_t)stream>>>(d_ptr, d_frames, num_trajs, d_win_start, num_windows, L,
                                                          d_hits);
    PSFM_LAUNCH_CHECK();
    return PSFM_OK;
  });
}

extern "C" int psfm_seg_shuffle(int32_t K, int32_t* perm) {
  const char* entry = "psfm_seg_shuffle";
  return guard(entry, [&]() -> int {
    if (!perm) return fail(entry, PSFM_ERR_INVALID, "null argument");
    if (K < 0) return fail(entry, PSFM_ERR_INVALID, "K must not be negative");
    std::vector<int32_t> p((size_t)K);
    std::iota(p.begin(), p.end(), 0);
    std::mt19937 rng(5489u);
    std::shuffle(p.begin(), p.end(), rng);
    std::copy(p.begin(), p.end(), perm);
    return PSFM_OK;
  });
}

extern "C" int psfm_seg_windows(const int64_t* d_ptr, const int32_t* d_frames, const double* d_xy,
                                const int32_t* d_rows, const int32_t* d_row_window, int32_t num_rows,
                                const int32_t* d_win_start, int32_t L, double* d_loc, uint8_t* d_valid,
                                void* stream) {
  const char* entry = "psfm_seg_windows";
  return guard(entry, [&]() -> int {
    if (!d_ptr || !d_frames || !d_xy || !d_rows || !d_row_window || !d_win_start || !d_loc || !d_valid)
      return fail(entry, PSFM_ERR_INVALID, "null argument");
    if (num_rows < 1) return fail(entry, PSFM_ERR_INVALID, "num_rows must be positive");
    int rc = check_window(entry, 1, L);
    if (rc != PSFM_OK) return rc;
    rc = require_device(entry);
    if (rc != PSFM_OK) return rc;
    const long long n = (long long)num_rows * L;
    k_windows<<<grid_of(n), 256, 0, (cudaStream_t)stream>>>(d_ptr, d_frames, d_xy, d_rows, d_row_window, num_rows,
                                                             d_win_start, L, d_loc, d_valid);
    PSFM_LAUNCH_CHECK();
    return PSFM_OK;
  });
}

extern "C" int psfm_seg_depth_resize(const uint16_t* d_pixels, int32_t num_frames, int32_t h, int32_t w, float* d_out,
                                     void* stream) {
  const char* entry = "psfm_seg_depth_resize";
  return guard(entry, [&]() -> int {
    if (!d_pixels || !d_out) return fail(entry, PSFM_ERR_INVALID, "null argument");
    if (num_frames < 1 || num_frames > 65535) return fail(entry, PSFM_ERR_INVALID, "num_frames must be 1 .. 65535");
    if (h < 1 || w < 1 || (long long)h * w > (1ll << 28)) return fail(entry, PSFM_ERR_INVALID, "bad frame size");
    int rc = require_device(entry);
    if (rc != PSFM_OK) return rc;
    // cv::resize: inv_scale = dsize / ssize, and resizeGeneric_ takes scale = 1 / inv_scale
    const double scale_x = 1.0 / ((double)kW / w), scale_y = 1.0 / ((double)kH / h);
    const dim3 grid(grid_of((long long)kH * kW), num_frames);
    k_depth_resize<<<grid, 256, 0, (cudaStream_t)stream>>>(d_pixels, h, w, scale_x, scale_y, d_out);
    PSFM_LAUNCH_CHECK();
    return PSFM_OK;
  });
}

extern "C" int psfm_seg_encode(const double* d_loc, const uint8_t* d_valid, const int32_t* d_row_window,
                               const int32_t* d_win_start, int32_t num_windows, int32_t num_rows, int32_t L,
                               const float* d_depth, int32_t num_frames, int32_t raw_h, int32_t raw_w,
                               const float* d_weights, float* d_feat, void* stream) {
  const char* entry = "psfm_seg_encode";
  return guard(entry, [&]() -> int {
    if (!d_loc || !d_valid || !d_row_window || !d_win_start || !d_depth || !d_weights || !d_feat)
      return fail(entry, PSFM_ERR_INVALID, "null argument");
    if (num_rows < 1) return fail(entry, PSFM_ERR_INVALID, "num_rows must be positive");
    int rc = check_window(entry, num_windows, L);
    if (rc != PSFM_OK) return rc;
    if (L > psfm_seg_max_window())
      return fail(entry, PSFM_ERR_INVALID, "window length " + std::to_string(L) + " exceeds the fused encoder's " +
                                               std::to_string(psfm_seg_max_window()));
    if (num_frames < 1) return fail(entry, PSFM_ERR_INVALID, "num_frames must be positive");
    if (raw_h < 1 || raw_w < 1) return fail(entry, PSFM_ERR_INVALID, "bad frame size");
    rc = require_device(entry);
    if (rc != PSFM_OK) return rc;
    const int warps = encode_warps(L);
    const size_t smem = (size_t)(kWeightsPadded + (long long)warps * kWarpFloats * L) * 4;
    PSFM_CUDA(cudaFuncSetAttribute(k_encode, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int dev = 0, sms = 0, per_sm = 0;
    PSFM_CUDA(cudaGetDevice(&dev));
    PSFM_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    PSFM_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_encode, warps * 32, smem));
    const long long blocks = std::min<long long>((num_rows + warps - 1) / warps, (long long)sms * std::max(per_sm, 1));
    k_encode<<<(unsigned)blocks, warps * 32, smem, (cudaStream_t)stream>>>(
        d_loc, d_valid, d_row_window, d_win_start, num_rows, L, d_depth, num_frames, (double)raw_w / (double)kW,
        (double)raw_h / (double)kH, d_weights, d_feat);
    PSFM_LAUNCH_CHECK();
    return PSFM_OK;
  });
}

extern "C" int psfm_seg_merge(const int64_t* d_ptr, const int32_t* d_frames, int32_t num_trajs,
                              const int32_t* d_win_start, int32_t num_windows, int32_t L, const int32_t* d_row_of,
                              const uint8_t* d_pred, int8_t* d_labels, int32_t* d_first_row, void* stream) {
  const char* entry = "psfm_seg_merge";
  return guard(entry, [&]() -> int {
    if (!d_ptr || !d_frames || !d_win_start || !d_row_of || !d_pred || !d_labels || !d_first_row)
      return fail(entry, PSFM_ERR_INVALID, "null argument");
    if (num_trajs < 1) return fail(entry, PSFM_ERR_INVALID, "num_trajs must be positive");
    int rc = check_window(entry, num_windows, L);
    if (rc != PSFM_OK) return rc;
    rc = require_device(entry);
    if (rc != PSFM_OK) return rc;
    k_merge<<<grid_of(num_trajs), 256, 0, (cudaStream_t)stream>>>(d_ptr, d_frames, num_trajs, d_win_start,
                                                                   num_windows, L, d_row_of, d_pred, d_labels,
                                                                   d_first_row);
    PSFM_LAUNCH_CHECK();
    return PSFM_OK;
  });
}

extern "C" int psfm_seg_draw(const uint8_t* d_frames, const double* d_loc, const uint8_t* d_valid,
                             const uint8_t* d_pred, int32_t K, int32_t L, int32_t raw_h, int32_t raw_w,
                             const int32_t* d_draws, int32_t num_draws, const int16_t* d_stamps, int32_t na,
                             int32_t nb, int32_t nc, int32_t* d_order, uint8_t* d_out, void* stream) {
  const char* entry = "psfm_seg_draw";
  return guard(entry, [&]() -> int {
    if (!d_frames || !d_order || !d_out || !d_stamps) return fail(entry, PSFM_ERR_INVALID, "null argument");
    if (K > 0 && (!d_loc || !d_valid || !d_pred)) return fail(entry, PSFM_ERR_INVALID, "null argument");
    if (num_draws > 0 && !d_draws) return fail(entry, PSFM_ERR_INVALID, "null argument");
    if (K < 0 || num_draws < 0 || (num_draws > 0 && K == 0))
      return fail(entry, PSFM_ERR_INVALID, "bad trajectory or draw count");
    if (na < 1 || nb < 1 || nc < 1) return fail(entry, PSFM_ERR_INVALID, "empty stamp");
    int rc = check_window(entry, 1, L);
    if (rc != PSFM_OK) return rc;
    if (raw_h < 1 || raw_w < 1) return fail(entry, PSFM_ERR_INVALID, "bad frame size");
    rc = require_device(entry);
    if (rc != PSFM_OK) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    PSFM_CUDA(cudaMemsetAsync(d_order, 0, (size_t)L * 3 * kH * kW * sizeof(int32_t), st));
    const long long n = ((long long)K + num_draws) * L;
    if (n > 0) {
      k_draw_stamp<<<grid_of(n), 256, 0, st>>>(d_loc, d_valid, K, L, (double)raw_w / (double)kW,
                                                (double)raw_h / (double)kH, d_draws, num_draws, d_stamps, na, nb, nc,
                                                d_order);
      PSFM_LAUNCH_CHECK();
    }
    k_draw_colour<<<grid_of((long long)L * 4 * kH * kW), 256, 0, st>>>(d_frames, L, d_order, d_pred, d_draws, d_out);
    PSFM_LAUNCH_CHECK();
    return PSFM_OK;
  });
}
