// midas.cu — the host-side steps around MiDaS's network on the device (DESIGN.md §4.16).
//
// Reference: third_party/MiDaS run.py:run_midas with model midas_v21, midas/transforms.py (Resize, NormalizeImage,
// PrepareForNet) and midas_utils.py (read_image, write_depth).  The network itself stays cuDNN calls through torch
// (particlesfm_b200/midas.py).
//
//   psfm_depth_prepare    uint8 RGB frames [n][h][w][3] -> the network input [n][3][H][W] with channels_last strides
//                         (memory [n][H][W][3]), fp32 or fp16: read_image's / 255, Resize's cv2.resize(INTER_CUBIC)
//                         of the float64 image and NormalizeImage, all in float64 as the reference computes them on
//                         the host, rounded once to float32 (then to fp16, as sample.half() rounds the float32 input).
//                         cv2's bicubic: source x = (float)((X + 0.5) * scale - 0.5), float coefficients with
//                         A = -0.75, replicated border, the horizontal pass of each source row then the vertical one,
//                         each a left-to-right sum of four float64 products.
//   psfm_depth_upsample   F.interpolate(prediction, (h, w), mode="bicubic", align_corners=False) as torch's CUDA
//                         kernel computes it (float accumulation, one rounding to the prediction's dtype), written as
//                         float32 with the rows flipped (write_pfm's np.flipud: the PFM payload), and each frame's
//                         minimum and maximum.
//   psfm_depth_quantize   write_depth(bits=2) on the float32 map: 65535 * (d - min) / (max - min), each operation
//                         rounded to float32 in that order, truncated to uint16; a frame whose max - min is not above
//                         float64 eps gets zeros.  Pixels in frame orientation from the flipped maps.
//
// Compiled with -fmad=false: the input transform and the quantisation restate unfused float64 / float32 arithmetic.
// Where torch's kernel is compiled with contraction (the bicubic upsampling), the fused products are written out.
#include <cuda_fp16.h>
#include <float.h>
#include <math.h>

#include "psfm_common.cuh"

namespace {

using namespace psfm;

// ImageNet statistics of NormalizeImage, as the Python floats (float64) the reference subtracts and divides by
__constant__ double kMean[3] = {0.485, 0.456, 0.406};
__constant__ double kStd[3] = {0.229, 0.224, 0.225};

// cv2's interpolateCubic (imgproc/src/resize.cpp), in float
__device__ __forceinline__ void cv_cubic_coeffs(float x, float c[4]) {
  const float A = -0.75f;
  c[0] = ((A * (x + 1) - 5 * A) * (x + 1) + 8 * A) * (x + 1) - 4 * A;
  c[1] = ((A + 2) * x - (A + 3)) * x * x + 1;
  c[2] = ((A + 2) * (1 - x) - (A + 3)) * (1 - x) * (1 - x) + 1;
  c[3] = 1.f - c[0] - c[1] - c[2];
}

// one destination coordinate of cv2's resizeGeneric_: the first of the four source indices and the coefficients
__device__ __forceinline__ int cv_source(int d, double scale, float c[4]) {
  float f = (float)((d + 0.5) * scale - 0.5);
  const int s = (int)floorf(f);
  f -= (float)s;
  cv_cubic_coeffs(f, c);
  return s - 1;
}

template <typename T>
__global__ void k_prepare(const uint8_t* __restrict__ rgb, int h, int w, int H, int W, double scale_x, double scale_y,
                          T* __restrict__ out) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)H * W) return;
  const int frame = blockIdx.y;
  const int X = (int)(i % W), Y = (int)(i / W);
  float ax[4], ay[4];
  const int x0 = cv_source(X, scale_x, ax), y0 = cv_source(Y, scale_y, ay);
  int xs[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) xs[j] = min(max(x0 + j, 0), w - 1);
  const uint8_t* img = rgb + (long long)frame * h * w * 3;
  T* o = out + ((long long)frame * H * W + i) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    double v = 0.0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint8_t* row = img + (long long)min(max(y0 + k, 0), h - 1) * w * 3 + c;
      double r = 0.0;
#pragma unroll
      for (int j = 0; j < 4; ++j) r = r + ((double)row[xs[j] * 3] / 255.0) * (double)ax[j];
      v = v + r * (double)ay[k];
    }
    const float f = (float)((v - kMean[c]) / kStd[c]);
    if constexpr (sizeof(T) == 2) o[c] = __float2half_rn(f);
    else o[c] = f;
  }
}

// torch's upsample_bicubic2d: get_cubic_upsample_coefficients and cubic_interp1d in float, with the fused products
// of its CUDA build
__device__ __forceinline__ float conv1(float x) {          // ((A + 2) x - (A + 3)) x x + 1
  const float A = -0.75f;
  return __fmaf_rn(__fmaf_rn(A + 2.0f, x, -(A + 3.0f)) * x, x, 1.0f);
}
__device__ __forceinline__ float conv2(float x) {          // ((A x - 5 A) x + 8 A) x - 4 A
  const float A = -0.75f;
  return __fmaf_rn(__fmaf_rn(__fmaf_rn(A, x, -5.0f * A), x, 8.0f * A), x, -4.0f * A);
}
__device__ __forceinline__ float interp1d(float x0, float x1, float x2, float x3, float t) {
  const float c0 = conv2(t + 1.0f), c1 = conv1(t), c2 = conv1(1.0f - t), c3 = conv2((1.0f - t) + 1.0f);
  return __fmaf_rn(x3, c3, __fmaf_rn(x2, c2, __fmaf_rn(x1, c1, x0 * c0)));
}

template <typename T>
__device__ __forceinline__ float load(const T* p) {
  if constexpr (sizeof(T) == 2) return __half2float(*p);
  else return *p;
}

template <typename T>
__device__ __forceinline__ float round_to(float v) {
  if constexpr (sizeof(T) == 2) return __half2float(__float2half_rn(v));
  else return v;
}

// ordered encoding of a float for unsigned atomics: a < b  <=>  enc(a) < enc(b)
__device__ __forceinline__ unsigned enc(float v) {
  const unsigned u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float dec(unsigned e) {
  return __uint_as_float((e & 0x80000000u) ? (e & 0x7fffffffu) : ~e);
}

__global__ void k_minmax_init(unsigned* __restrict__ mm, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    mm[2 * i] = 0xffffffffu;
    mm[2 * i + 1] = 0u;
  }
}

template <typename T>
__global__ void k_upsample(const T* __restrict__ pred, int ih, int iw, int h, int w, float* __restrict__ out,
                           unsigned* __restrict__ mm) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const int frame = blockIdx.y;
  const bool live = i < (long long)h * w;
  unsigned lo = 0xffffffffu, hi = 0u;
  if (live) {
    const int x = (int)(i % w), y = (int)(i / w);
    const T* in = pred + (long long)frame * ih * iw;
    float v;
    if (ih == h && iw == w) {
      v = load(in + i);
    } else {
      const float sy = (float)ih / (float)h, sx = (float)iw / (float)w;
      const float ry = __fmaf_rn(sy, (float)y + 0.5f, -0.5f), rx = __fmaf_rn(sx, (float)x + 0.5f, -0.5f);
      const int y0 = (int)floorf(ry), x0 = (int)floorf(rx);
      const float ty = ry - (float)y0, tx = rx - (float)x0;
      int xs[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) xs[j] = min(max(x0 - 1 + j, 0), iw - 1);
      float r[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const T* row = in + (long long)min(max(y0 - 1 + k, 0), ih - 1) * iw;
        r[k] = interp1d(load(row + xs[0]), load(row + xs[1]), load(row + xs[2]), load(row + xs[3]), tx);
      }
      v = round_to<T>(interp1d(r[0], r[1], r[2], r[3], ty));
    }
    out[((long long)frame * h + (h - 1 - y)) * w + x] = v;
    if (v == v) lo = hi = enc(v);
  }
  for (int o = 16; o > 0; o >>= 1) {
    lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  if ((threadIdx.x & 31) == 0 && hi >= lo) {
    atomicMin(mm + 2 * frame, lo);
    atomicMax(mm + 2 * frame + 1, hi);
  }
}

__global__ void k_minmax_decode(const unsigned* __restrict__ mm, int n, float* __restrict__ minmax) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 2 * n) minmax[i] = mm[i / 2 * 2 + 1] >= mm[i / 2 * 2] ? dec(mm[i]) : NAN;
}

__global__ void k_quantize(const float* __restrict__ maps, int h, int w, const float* __restrict__ minmax,
                           uint16_t* __restrict__ out) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)h * w) return;
  const int frame = blockIdx.y;
  const int x = (int)(i % w), y = (int)(i / w);
  const float lo = minmax[2 * frame], hi = minmax[2 * frame + 1];
  const float range = hi - lo;
  uint16_t q = 0;
  if ((double)range > DBL_EPSILON) {
    const float d = maps[((long long)frame * h + (h - 1 - y)) * w + x];
    const float t = (65535.0f * (d - lo)) / range;
    q = (uint16_t)__float2uint_rz(t);
  }
  out[(long long)frame * h * w + i] = q;
}

int check_sizes(const char* entry, int32_t n, int32_t h, int32_t w) {
  if (n < 1 || n > 65535) return fail(entry, PSFM_ERR_INVALID, "num_frames must be 1 .. 65535");
  if (h < 1 || w < 1 || (long long)h * w > (1ll << 28)) return fail(entry, PSFM_ERR_INVALID, "bad frame size");
  return PSFM_OK;
}

}  // namespace

extern "C" int psfm_depth_prepare(const uint8_t* d_rgb, int32_t num_frames, int32_t h, int32_t w, int32_t net_h,
                                  int32_t net_w, int32_t half, void* d_out, void* stream) {
  const char* entry = "psfm_depth_prepare";
  return guard(entry, [&]() -> int {
    if (!d_rgb || !d_out) return fail(entry, PSFM_ERR_INVALID, "null argument");
    int rc = check_sizes(entry, num_frames, h, w);
    if (rc != PSFM_OK) return rc;
    if (net_h < 1 || net_w < 1 || (long long)net_h * net_w > (1ll << 28))
      return fail(entry, PSFM_ERR_INVALID, "bad network input size");
    if (half != 0 && half != 1) return fail(entry, PSFM_ERR_INVALID, "half must be 0 or 1");
    rc = require_device(entry);
    if (rc != PSFM_OK) return rc;
    // cv::resize: inv_scale = dsize / ssize, and resizeGeneric_ takes scale = 1 / inv_scale
    const double scale_x = 1.0 / ((double)net_w / w), scale_y = 1.0 / ((double)net_h / h);
    const dim3 grid(grid_of((long long)net_h * net_w), num_frames);
    cudaStream_t st = (cudaStream_t)stream;
    if (half) k_prepare<__half><<<grid, 256, 0, st>>>(d_rgb, h, w, net_h, net_w, scale_x, scale_y, (__half*)d_out);
    else k_prepare<float><<<grid, 256, 0, st>>>(d_rgb, h, w, net_h, net_w, scale_x, scale_y, (float*)d_out);
    PSFM_LAUNCH_CHECK();
    return PSFM_OK;
  });
}

extern "C" int psfm_depth_upsample(const void* d_pred, int32_t num_frames, int32_t net_h, int32_t net_w, int32_t half,
                                   int32_t h, int32_t w, float* d_flipped, float* d_minmax, void* stream) {
  const char* entry = "psfm_depth_upsample";
  return guard(entry, [&]() -> int {
    if (!d_pred || !d_flipped || !d_minmax) return fail(entry, PSFM_ERR_INVALID, "null argument");
    int rc = check_sizes(entry, num_frames, h, w);
    if (rc != PSFM_OK) return rc;
    if (net_h < 1 || net_w < 1 || (long long)net_h * net_w > (1ll << 28))
      return fail(entry, PSFM_ERR_INVALID, "bad network output size");
    if (half != 0 && half != 1) return fail(entry, PSFM_ERR_INVALID, "half must be 0 or 1");
    rc = require_device(entry);
    if (rc != PSFM_OK) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    DBuf<unsigned> mm;
    mm.alloc(2 * (size_t)num_frames, st);
    k_minmax_init<<<grid_of(num_frames), 256, 0, st>>>(mm.p, num_frames);
    PSFM_LAUNCH_CHECK();
    const dim3 grid(grid_of((long long)h * w), num_frames);
    if (half) k_upsample<__half><<<grid, 256, 0, st>>>((const __half*)d_pred, net_h, net_w, h, w, d_flipped, mm.p);
    else k_upsample<float><<<grid, 256, 0, st>>>((const float*)d_pred, net_h, net_w, h, w, d_flipped, mm.p);
    PSFM_LAUNCH_CHECK();
    k_minmax_decode<<<grid_of(2 * (long long)num_frames), 256, 0, st>>>(mm.p, num_frames, d_minmax);
    PSFM_LAUNCH_CHECK();
    return PSFM_OK;
  });
}

extern "C" int psfm_depth_quantize(const float* d_flipped, int32_t num_frames, int32_t h, int32_t w,
                                   const float* d_minmax, uint16_t* d_pixels, void* stream) {
  const char* entry = "psfm_depth_quantize";
  return guard(entry, [&]() -> int {
    if (!d_flipped || !d_minmax || !d_pixels) return fail(entry, PSFM_ERR_INVALID, "null argument");
    int rc = check_sizes(entry, num_frames, h, w);
    if (rc != PSFM_OK) return rc;
    rc = require_device(entry);
    if (rc != PSFM_OK) return rc;
    k_quantize<<<dim3(grid_of((long long)h * w), num_frames), 256, 0, (cudaStream_t)stream>>>(d_flipped, h, w, d_minmax,
                                                                                            d_pixels);
    PSFM_LAUNCH_CHECK();
    return PSFM_OK;
  });
}
