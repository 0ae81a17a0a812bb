// optical_flow.cu — the non-convolution parts of RAFT's inference on the device (DESIGN.md §4.14).
//
// Reference: third_party/RAFT core/corr.py (CorrBlock), core/raft.py:upsample_flow, core/utils/utils.py
// (bilinear_sampler, InputPadder) and core/utils/flow_viz.py (flow_to_image).  The convolutions stay cuDNN calls
// through torch (particlesfm_b200/optical_flow.py).
//
//   psfm_corr_pyramids   both directions' 4-level pyramids of one pair from one product fmap1^T fmap2: the product
//                        is scaled by 1/16 in place (the forward level 0) and transposed into the backward level 0
//                        (k_corr_level0, 32 x 32 tiles through shared memory), then both are avg-pooled 2 x 2 level by
//                        level (k_pool), as F.avg_pool2d does: ((a00 + a01) + a10) + a11, then / 4.
//   psfm_corr_lookup     the radius-4 lookup of every level (k_lookup): one thread per (pixel, level, problem), 81
//                        bilinear taps in the 10 x 10 patch around the centre, written to the [P][324][h][w] tensor
//                        convc1 reads.  Channel l * 81 + a * 9 + b holds the tap at (x / 2^l + a - 4, y / 2^l + b - 4):
//                        torch.meshgrid(dy, dx) stacked on the last axis adds the first window index to x.  Each tap
//                        goes through bilinear_sampler's normalisation 2 x / (W - 1) - 1 and grid_sample's
//                        align_corners unnormalisation, so its corners and weights are the reference's.
//   psfm_flow_upsample   the convex upsampling of the last iteration (k_upsample): softmax over 0.25 * the mask's 9
//                        logits, the weighted sum of 8 * flow over the 3 x 3 neighbourhood (zero outside), the padding
//                        removed, written as [P][H][W][2] float32 (the .flo and tracker layout).
//   psfm_flow_to_image   flow_to_image(flow, convert_to_bgr=True): the image-wide maximum radius (k_rad_max, a block
//                        reduction and an integer atomicMax on the non-negative float's bits), then one thread per
//                        pixel for the colour wheel (k_colour), in numpy's float32 / float64 promotions.
//
// Compiled with -fmad=false: the colour image restates numpy's unfused float32 and float64 arithmetic, so its bytes
// equal the restatement's (oracle/raft_oracle.py:flow_to_image).  The angle is the correctly rounded float32 atan2
// (atan2 in double, rounded once); numpy's own float32 arctan2 differs by CPU (SVML on AVX-512, libm elsewhere).
#include <math.h>

#include "psfm_common.cuh"

namespace {

using namespace psfm;

constexpr int kLevels = 4;
constexpr int kRadius = 4;
constexpr int kWin = 2 * kRadius + 1;              // 9
constexpr int kCorrChannels = kLevels * kWin * kWin;   // 324

// floats of one direction's pyramid of an h x w grid: h w images of every level's size
long long pyramid_floats(int h, int w) {
  long long per = 0;
  int hl = h, wl = w;
  for (int l = 0; l < kLevels; ++l) {
    per += (long long)hl * wl;
    hl /= 2;
    wl /= 2;
  }
  return (long long)h * w * per;
}

__global__ void k_corr_level0(float* __restrict__ fwd, float* __restrict__ bwd, int n) {
  __shared__ float tile[32][33];
  const int q0 = blockIdx.x * 32, p0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int p = p0 + j, q = q0 + threadIdx.x;
    if (p < n && q < n) {
      const size_t i = (size_t)p * n + q;
      const float v = fwd[i] * 0.0625f;     // / sqrt(256): a power of two, exact
      fwd[i] = v;
      tile[j][threadIdx.x] = v;
    }
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int q = q0 + j, p = p0 + threadIdx.x;
    if (p < n && q < n) bwd[(size_t)q * n + p] = tile[threadIdx.x][j];
  }
}

// one level of both directions: in [N][hi][wi] -> out [N][hi/2][wi/2]; blockIdx.y picks the direction
__global__ void k_pool(const float* __restrict__ in0, float* __restrict__ out0, const float* __restrict__ in1,
                       float* __restrict__ out1, long long N, int hi, int wi) {
  const float* in = blockIdx.y ? in1 : in0;
  float* out = blockIdx.y ? out1 : out0;
  const int ho = hi / 2, wo = wi / 2;
  const long long total = N * ho * wo;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(i % wo);
    const long long r = i / wo;
    const int y = (int)(r % ho);
    const long long n = r / ho;
    const float* s = in + (n * hi + 2 * y) * wi + 2 * x;
    float v = s[0];
    v = v + s[1];
    v = v + s[wi];
    v = v + s[wi + 1];
    out[i] = v / 4.0f;
  }
}

// bilinear_sampler's normalisation followed by grid_sample's align_corners unnormalisation, in float32
__device__ __forceinline__ float round_trip(float x, int size) {
  const float s = (float)(size - 1);
  const float g = (2.0f * x) / s - 1.0f;
  return ((g + 1.0f) / 2.0f) * s;
}

__global__ void k_lookup(const float* __restrict__ pyr, long long problem_stride, int h, int w,
                         const float* __restrict__ coords, float* __restrict__ out) {
  const int hw = h * w;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= hw) return;
  const int l = blockIdx.y, prob = blockIdx.z;
  long long off = 0;
  int hl = h, wl = w;
  for (int k = 0; k < l; ++k) {
    off += (long long)hw * hl * wl;
    hl /= 2;
    wl /= 2;
  }
  const float* img = pyr + prob * problem_stride + off + (long long)pix * hl * wl;
  const float scale = 1.0f / (float)(1 << l);
  const float cx = coords[((long long)prob * 2 + 0) * hw + pix] * scale;
  const float cy = coords[((long long)prob * 2 + 1) * hw + pix] * scale;
  float* o = out + ((long long)prob * kCorrChannels + l * kWin * kWin) * hw + pix;
  for (int a = 0; a < kWin; ++a) {
    const float ix = round_trip(cx + (float)(a - kRadius), wl);
    const float x0 = floorf(ix), x1 = x0 + 1.0f;
    const bool okx0 = x0 >= 0.0f && x0 <= (float)(wl - 1), okx1 = x1 >= 0.0f && x1 <= (float)(wl - 1);
    const int xi0 = okx0 ? (int)x0 : 0, xi1 = okx1 ? (int)x1 : 0;
    for (int b = 0; b < kWin; ++b) {
      const float iy = round_trip(cy + (float)(b - kRadius), hl);
      const float y0 = floorf(iy), y1 = y0 + 1.0f;
      const bool oky0 = y0 >= 0.0f && y0 <= (float)(hl - 1), oky1 = y1 >= 0.0f && y1 <= (float)(hl - 1);
      const int yi0 = oky0 ? (int)y0 : 0, yi1 = oky1 ? (int)y1 : 0;
      // grid_sampler_2d's bilinear weights and accumulation order (nw, ne, sw, se)
      const float nw = (x1 - ix) * (y1 - iy), ne = (ix - x0) * (y1 - iy);
      const float sw = (x1 - ix) * (iy - y0), se = (ix - x0) * (iy - y0);
      float v = 0.0f;
      if (okx0 && oky0) v = v + __ldg(img + yi0 * wl + xi0) * nw;
      if (okx1 && oky0) v = v + __ldg(img + yi0 * wl + xi1) * ne;
      if (okx0 && oky1) v = v + __ldg(img + yi1 * wl + xi0) * sw;
      if (okx1 && oky1) v = v + __ldg(img + yi1 * wl + xi1) * se;
      o[(long long)(a * kWin + b) * hw] = v;
    }
  }
}

__global__ void k_upsample(const float* __restrict__ flow, const float* __restrict__ mask, int h, int w, int out_h,
                           int out_w, int pad_top, int pad_left, float* __restrict__ out) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const int prob = blockIdx.y;
  if (i >= (long long)out_h * out_w) return;
  const int X = (int)(i % out_w) + pad_left, Y = (int)(i / out_w) + pad_top;
  const int x = X >> 3, y = Y >> 3, si = Y & 7, sj = X & 7;
  const long long hw = (long long)h * w;
  const float* m = mask + (long long)prob * 576 * hw + (si * 8 + sj) * hw + (long long)y * w + x;
  float logit[9], mx = -INFINITY;
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    logit[k] = 0.25f * m[k * 64 * hw];
    mx = fmaxf(mx, logit[k]);
  }
  float sum = 0.0f;
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    logit[k] = expf(logit[k] - mx);
    sum += logit[k];
  }
  const float* fu = flow + (long long)prob * 2 * hw;
  float u = 0.0f, v = 0.0f;
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    const int yy = y + k / 3 - 1, xx = x + k % 3 - 1;
    if (yy < 0 || yy >= h || xx < 0 || xx >= w) continue;       // unfold's zero padding
    const float wk = logit[k] / sum;
    u += wk * (8.0f * fu[(long long)yy * w + xx]);
    v += wk * (8.0f * fu[hw + (long long)yy * w + xx]);
  }
  float* o = out + ((long long)prob * out_h * out_w + i) * 2;
  o[0] = u;
  o[1] = v;
}

__device__ __forceinline__ float radius(float u, float v) { return sqrtf(u * u + v * v); }

__global__ void k_rad_max(const float* __restrict__ flow, long long hw, unsigned* __restrict__ rad_max) {
  __shared__ unsigned s[32];
  const float* f = flow + (long long)blockIdx.y * hw * 2;
  unsigned m = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < hw; i += (long long)gridDim.x * blockDim.x)
    m = max(m, __float_as_uint(radius(f[2 * i], f[2 * i + 1])));    // rad >= 0: its bits order as the values
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x < 32) {
    m = threadIdx.x < (blockDim.x >> 5) ? s[threadIdx.x] : 0u;
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (threadIdx.x == 0) atomicMax(rad_max + blockIdx.y, m);
  }
}

// make_colorwheel(): 55 x 3 float64 entries, floor(255 * i / n) as numpy evaluates (255 * i) / n
__device__ double wheel(int k, int c) {
  const int RY = 15, YG = 6, GC = 4, CB = 11, BM = 13, MR = 6;
  auto ramp = [](int i, int n) { return floor((double)(255 * i) / (double)n); };
  if (k < RY) return c == 0 ? 255.0 : c == 1 ? ramp(k, RY) : 0.0;
  k -= RY;
  if (k < YG) return c == 0 ? 255.0 - ramp(k, YG) : c == 1 ? 255.0 : 0.0;
  k -= YG;
  if (k < GC) return c == 0 ? 0.0 : c == 1 ? 255.0 : ramp(k, GC);
  k -= GC;
  if (k < CB) return c == 0 ? 0.0 : c == 1 ? 255.0 - ramp(k, CB) : 255.0;
  k -= CB;
  if (k < BM) return c == 0 ? ramp(k, BM) : c == 1 ? 0.0 : 255.0;
  k -= BM;
  return c == 0 ? 255.0 : c == 1 ? 0.0 : 255.0 - ramp(k, MR);
}

__global__ void k_colour(const float* __restrict__ flow, long long hw, const unsigned* __restrict__ rad_max,
                         uint8_t* __restrict__ bgr) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= hw) return;
  const int map = blockIdx.y;
  const float* f = flow + ((long long)map * hw + i) * 2;
  const float d = __uint_as_float(rad_max[map]) + 1e-5f;     // float32 + a Python float: float32 under NEP 50
  const float u = f[0] / d, v = f[1] / d;
  const float rad = radius(u, v);
  const float a = (float)atan2(-(double)v, -(double)u) / 3.14159265358979323846f;
  const float fk = (a + 1.0f) / 2.0f * 54.0f;
  const int k0 = (int)floorf(fk);
  const int k1 = k0 + 1 == 55 ? 0 : k0 + 1;
  const double fr = (double)fk - (double)k0;      // float32 - int32 promotes to float64
  uint8_t* o = bgr + ((long long)map * hw + i) * 3;
  for (int c = 0; c < 3; ++c) {
    const double col0 = wheel(k0, c) / 255.0, col1 = wheel(k1, c) / 255.0;
    double col = (1.0 - fr) * col0 + fr * col1;
    if (rad <= 1.0f) col = 1.0 - (double)rad * (1.0 - col);
    else col = col * 0.75;
    o[2 - c] = (uint8_t)floor(255.0 * col);
  }
}

}  // namespace

extern "C" int psfm_corr_pyramids(float* d_fwd, float* d_bwd, int32_t h, int32_t w, void* stream) {
  const char* entry = "psfm_corr_pyramids";
  if (!d_fwd || !d_bwd) return fail(entry, PSFM_ERR_INVALID, "null argument");
  if (h < 8 || w < 8) return fail(entry, PSFM_ERR_INVALID, "bad sizes: every level needs at least one pixel (h, w >= 8)");
  if ((long long)h * w > (1 << 20)) return fail(entry, PSFM_ERR_INVALID, "bad sizes: more than 2^20 pixels at 1/8");
  int rc = require_device(entry);
  if (rc != PSFM_OK) return rc;
  try {
    cudaStream_t st = (cudaStream_t)stream;
    const int n = h * w;
    k_corr_level0<<<dim3((n + 31) / 32, (n + 31) / 32), dim3(32, 8), 0, st>>>(d_fwd, d_bwd, n);
    PSFM_LAUNCH_CHECK();
    long long off = 0;
    int hl = h, wl = w;
    for (int l = 1; l < kLevels; ++l) {
      const long long next = off + (long long)n * hl * wl;
      const long long outs = (long long)n * (hl / 2) * (wl / 2);
      k_pool<<<dim3(grid_stride_of(outs), 2), 256, 0, st>>>(d_fwd + off, d_fwd + next, d_bwd + off, d_bwd + next, n, hl, wl);
      PSFM_LAUNCH_CHECK();
      off = next;
      hl /= 2;
      wl /= 2;
    }
    return PSFM_OK;
  } catch (const CudaFail& f) { return f.code; }
}

extern "C" int64_t psfm_corr_pyramid_floats(int32_t h, int32_t w) {
  if (h < 8 || w < 8 || (long long)h * w > (1 << 20)) return fail("psfm_corr_pyramid_floats", PSFM_ERR_INVALID, "bad sizes");
  return pyramid_floats(h, w);
}

extern "C" int psfm_corr_lookup(const float* d_pyramids, int32_t num_problems, int32_t h, int32_t w, const float* d_coords,
                                float* d_out, void* stream) {
  const char* entry = "psfm_corr_lookup";
  if (!d_pyramids || !d_coords || !d_out) return fail(entry, PSFM_ERR_INVALID, "null argument");
  if (h < 8 || w < 8 || (long long)h * w > (1 << 20)) return fail(entry, PSFM_ERR_INVALID, "bad sizes");
  if (num_problems < 1 || num_problems > 65535) return fail(entry, PSFM_ERR_INVALID, "num_problems must be 1 .. 65535");
  int rc = require_device(entry);
  if (rc != PSFM_OK) return rc;
  try {
    const int hw = h * w;
    k_lookup<<<dim3((hw + 127) / 128, kLevels, num_problems), 128, 0, (cudaStream_t)stream>>>(
        d_pyramids, pyramid_floats(h, w), h, w, d_coords, d_out);
    PSFM_LAUNCH_CHECK();
    return PSFM_OK;
  } catch (const CudaFail& f) { return f.code; }
}

extern "C" int psfm_flow_upsample(const float* d_flow, const float* d_mask, int32_t num_problems, int32_t h, int32_t w,
                                  const int32_t* pad, float* d_out, void* stream) {
  const char* entry = "psfm_flow_upsample";
  if (!d_flow || !d_mask || !pad || !d_out) return fail(entry, PSFM_ERR_INVALID, "null argument");
  if (h < 1 || w < 1 || (long long)h * w > (1 << 20)) return fail(entry, PSFM_ERR_INVALID, "bad sizes");
  if (num_problems < 1 || num_problems > 65535) return fail(entry, PSFM_ERR_INVALID, "num_problems must be 1 .. 65535");
  for (int k = 0; k < 4; ++k)
    if (pad[k] < 0 || pad[k] > 7) return fail(entry, PSFM_ERR_INVALID, "padding must be 0 .. 7");
  const int out_w = 8 * w - pad[0] - pad[1], out_h = 8 * h - pad[2] - pad[3];
  if (out_w < 1 || out_h < 1) return fail(entry, PSFM_ERR_INVALID, "padding leaves no pixel");
  int rc = require_device(entry);
  if (rc != PSFM_OK) return rc;
  try {
    const long long n = (long long)out_h * out_w;
    k_upsample<<<dim3(grid_of(n), num_problems), 256, 0, (cudaStream_t)stream>>>(d_flow, d_mask, h, w, out_h, out_w,
                                                                                   pad[2], pad[0], d_out);
    PSFM_LAUNCH_CHECK();
    return PSFM_OK;
  } catch (const CudaFail& f) { return f.code; }
}

extern "C" int psfm_flow_to_image(const float* d_flow, int32_t num_maps, int32_t h, int32_t w, uint8_t* d_bgr, void* stream) {
  const char* entry = "psfm_flow_to_image";
  if (!d_flow || !d_bgr) return fail(entry, PSFM_ERR_INVALID, "null argument");
  if (h < 1 || w < 1) return fail(entry, PSFM_ERR_INVALID, "bad sizes");
  if (num_maps < 1 || num_maps > 65535) return fail(entry, PSFM_ERR_INVALID, "num_maps must be 1 .. 65535");
  int rc = require_device(entry);
  if (rc != PSFM_OK) return rc;
  try {
    cudaStream_t st = (cudaStream_t)stream;
    const long long hw = (long long)h * w;
    DBuf<unsigned> rmax;
    rmax.alloc(num_maps, st);
    rmax.zero(st);
    k_rad_max<<<dim3((unsigned)std::min<long long>((hw + 255) / 256, 264), num_maps), 256, 0, st>>>(d_flow, hw, rmax.p);
    PSFM_LAUNCH_CHECK();
    k_colour<<<dim3(grid_of(hw), num_maps), 256, 0, st>>>(d_flow, hw, rmax.p, d_bgr);
    PSFM_LAUNCH_CHECK();
    return PSFM_OK;
  } catch (const CudaFail& f) { return f.code; }
}
