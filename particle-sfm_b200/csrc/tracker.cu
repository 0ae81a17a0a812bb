// tracker.cu — the tracker stage AROUND HP1 on the device (SURVEY.md §8f row f-1).
//
// Reference (Python, per frame and per particle):
//   grid_sample                point_trajectory/trajectory.py:25-37   torch grid_sample, bilinear, zeros
//                              padding, align_corners=True, after the normalisation x /= (W-1)/2; x -= 1
//   step_forward               trajectory.py:45-62      flow / occlusion sampling, survival flags
//   optimize_buffer            trajectory.py:161-194    flow01 / flow02 / occ02 sampling -> ref1, ref2, scale
//   extend_all                 trajectory.py:129-152    occupancy at (int(y), int(x)), re-seeding where the
//                              Euclidean distance transform exceeds sample_ratio on the strided grid
//   flow_check / get_occ_mask  point_trajectory/utils.py:58-105   forward/backward consistency
//
// The integer track connectivity is thresholded from these float32 results, so they are reproduced
// BIT FOR BIT: torch's CPU kernel (ATen GridSamplerKernel, vectorised build) evaluates
//     ix = (g + 1) * ((W - 1) / 2),  w = ix - floor(ix),  e = 1 - w   (same for y: n, s)
//     out = fma(v_se, w n, fma(v_sw, e n, fma(v_ne, w s, v_nw * (e s))))
// in float32 — established by comparing a numpy emulation with torch on 10^5 random samples (0 bit
// differences; the plain sum and the other fma orders differ in ~70 % of the samples), and re-checked
// against torch itself on the GPU by tests/test_gpu_tracker.py.  Every float32 operation below is
// an explicit round-to-nearest intrinsic, immune to -fmad.  torch.norm over the 2 flow channels is
// sqrt(a*a + b*b) without fma.  The distance transform is only ever compared with the integer
// sample_ratio: dist > r  <=>  no occupied pixel within squared distance r^2 — exact in integers.
#include <vector>

#include "psfm_common.cuh"

namespace {

using namespace psfm;

struct Coord {
  float ix, iy;
};

// the reference's normalisation followed by ATen's unnormalisation (align_corners = true)
__device__ __forceinline__ Coord gs_coord(float x, float y, int H, int W) {
  const float hx = (float)((double)(W - 1) / 2.0), hy = (float)((double)(H - 1) / 2.0);   // python float -> float32 tensor divide
  const float gx = __fsub_rn(__fdiv_rn(x, hx), 1.0f), gy = __fsub_rn(__fdiv_rn(y, hy), 1.0f);
  const float sx = __fdiv_rn((float)(W - 1), 2.0f), sy = __fdiv_rn((float)(H - 1), 2.0f);
  Coord c;
  c.ix = __fmul_rn(__fadd_rn(gx, 1.0f), sx);
  c.iy = __fmul_rn(__fadd_rn(gy, 1.0f), sy);
  return c;
}

// bilinear sample of channel-interleaved map [H][W][C] (C <= 2) or of a byte map (C == 1, as float 0/1)
template <typename T>
__device__ __forceinline__ void gs_sample(const T* __restrict__ map, int H, int W, int C, Coord c, float* out) {
  const float x0 = floorf(c.ix), y0 = floorf(c.iy);
  const float w = __fsub_rn(c.ix, x0), e = __fsub_rn(1.0f, w), n = __fsub_rn(c.iy, y0), s = __fsub_rn(1.0f, n);
  const float nw = __fmul_rn(e, s), ne = __fmul_rn(w, s), sw = __fmul_rn(e, n), se = __fmul_rn(w, n);
  const float x1 = x0 + 1.0f, y1 = y0 + 1.0f;
  const bool okx0 = x0 >= 0.0f && x0 <= (float)(W - 1), okx1 = x1 >= 0.0f && x1 <= (float)(W - 1);
  const bool oky0 = y0 >= 0.0f && y0 <= (float)(H - 1), oky1 = y1 >= 0.0f && y1 <= (float)(H - 1);
  const int xi0 = okx0 ? (int)x0 : 0, xi1 = okx1 ? (int)x1 : 0, yi0 = oky0 ? (int)y0 : 0, yi1 = oky1 ? (int)y1 : 0;
  for (int ch = 0; ch < C; ++ch) {
    const float vnw = (okx0 && oky0) ? (float)map[((size_t)yi0 * W + xi0) * C + ch] : 0.0f;
    const float vne = (okx1 && oky0) ? (float)map[((size_t)yi0 * W + xi1) * C + ch] : 0.0f;
    const float vsw = (okx0 && oky1) ? (float)map[((size_t)yi1 * W + xi0) * C + ch] : 0.0f;
    const float vse = (okx1 && oky1) ? (float)map[((size_t)yi1 * W + xi1) * C + ch] : 0.0f;
    float r = __fmul_rn(vnw, nw);
    r = __fmaf_rn(vne, ne, r);
    r = __fmaf_rn(vsw, sw, r);
    r = __fmaf_rn(vse, se, r);
    out[ch] = r;
  }
}

__global__ void k_grid_sample(const float* map, int H, int W, int C, const double* xy, int n, float* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float r[2] = {0.f, 0.f};
  gs_sample(map, H, W, C, gs_coord((float)xy[2 * (size_t)i], (float)xy[2 * (size_t)i + 1], H, W), r);
  for (int ch = 0; ch < C; ++ch) out[(size_t)i * C + ch] = r[ch];
}

// utils.py:58-105: grid = coord + flow_f; warp = grid_sample(flow_b, grid); err = |warp + flow_f|;
// occ = err > thres or grid outside [0, W-1] x [0, H-1]
__global__ void k_flow_check(const float* ff, const float* fb, int H, int W, float thres, float* err, unsigned char* occ) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= H * W) return;
  const int y = idx / W, x = idx % W;
  const float f0 = ff[2 * (size_t)idx], f1 = ff[2 * (size_t)idx + 1];
  const float gx = __fadd_rn((float)x, f0), gy = __fadd_rn((float)y, f1);
  const bool oob = gx < 0.0f || gx > (float)(W - 1) || gy < 0.0f || gy > (float)(H - 1);
  float r[2];
  gs_sample(fb, H, W, 2, gs_coord(gx, gy, H, W), r);
  const float s0 = __fadd_rn(r[0], f0), s1 = __fadd_rn(r[1], f1);
  const float e = __fsqrt_rn(__fadd_rn(__fmul_rn(s0, s0), __fmul_rn(s1, s1)));
  if (err) err[idx] = e;
  occ[idx] = (e > thres || oob) ? 1 : 0;
}

// step_forward (trajectory.py:45-62) for every live particle: next = cur + flow(cur) (float64 + float32),
// flag = inside the open image rectangle and sampled occlusion <= 0.1
__global__ void k_tracker_step(const float* flow, const unsigned char* occ, int H, int W, const double* cur, int n, double* next,
                               unsigned char* flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double cx = cur[2 * (size_t)i], cy = cur[2 * (size_t)i + 1];
  const Coord c = gs_coord((float)cx, (float)cy, H, W);
  float f[2], o[1];
  gs_sample(flow, H, W, 2, c, f);
  gs_sample(occ, H, W, 1, c, o);
  const double nx = cx + (double)f[0], ny = cy + (double)f[1];
  next[2 * (size_t)i] = nx; next[2 * (size_t)i + 1] = ny;
  const bool valid = nx > 0.0 && nx < (double)(W - 1) && ny > 0.0 && ny < (double)(H - 1);
  flags[i] = (valid && !(o[0] > 0.1f)) ? 1 : 0;
}

// optimize_buffer (trajectory.py:171-183): ref1 = x0 + flow01(x0), ref2 = x0 + flow02(x0),
// scale = (1 - occ02(x0)) * (|flow02(x0)| < upper_flow), all sampled in float32
__global__ void k_buffer_inputs(const float* f01, const float* f02, const unsigned char* occ02, int H, int W, const double* x0, int n,
                                double upper_flow, double* ref1, double* ref2, double* scale) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double px = x0[2 * (size_t)i], py = x0[2 * (size_t)i + 1];
  const Coord c = gs_coord((float)px, (float)py, H, W);
  float a[2], b[2], o[1];
  gs_sample(f01, H, W, 2, c, a);
  gs_sample(f02, H, W, 2, c, b);
  gs_sample(occ02, H, W, 1, c, o);
  ref1[2 * (size_t)i] = px + (double)a[0]; ref1[2 * (size_t)i + 1] = py + (double)a[1];
  ref2[2 * (size_t)i] = px + (double)b[0]; ref2[2 * (size_t)i + 1] = py + (double)b[1];
  const float nrm = __fsqrt_rn(__fadd_rn(__fmul_rn(b[0], b[0]), __fmul_rn(b[1], b[1])));    // np.linalg.norm of a float32 pair
  const float keep = ((double)nrm < upper_flow) ? 1.0f : 0.0f;
  scale[i] = (double)__fmul_rn(__fsub_rn(1.0f, o[0]), keep);
}

__global__ void k_occupancy(const double* xy, int n, int H, int W, unsigned char* occ) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long x = (long long)xy[2 * (size_t)i], y = (long long)xy[2 * (size_t)i + 1];      // astype(int64): truncation
  if (x >= 0 && x < W && y >= 0 && y < H) occ[(size_t)y * W + x] = 1;
}

// (distance_transform_edt(1 - occupied) > ratio)[::ratio, ::ratio]: a strided grid point is a new seed iff no
// occupied pixel lies within squared distance ratio^2
__global__ void k_reseed_mask(const unsigned char* occ, int H, int W, int ratio, int GH, int GW, unsigned char* mask) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= GH * GW) return;
  const int y = (g / GW) * ratio, x = (g % GW) * ratio;
  const int r2 = ratio * ratio;
  bool hit = false;
  for (int dy = -ratio; dy <= ratio && !hit; ++dy) {
    const int yy = y + dy;
    if (yy < 0 || yy >= H) continue;
    for (int dx = -ratio; dx <= ratio; ++dx) {
      const int xx = x + dx;
      if (xx < 0 || xx >= W || dy * dy + dx * dx > r2) continue;
      if (occ[(size_t)yy * W + xx]) { hit = true; break; }
    }
  }
  mask[g] = hit ? 0 : 1;
}

int device_ok() {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
    cudaGetLastError();
    set_error("no CUDA device available (this library has no CPU path)");
    return PSFM_ERR_NO_DEVICE;
  }
  return PSFM_OK;
}

inline unsigned grid_of(size_t n) { return (unsigned)((n + 255) / 256); }

}  // namespace

extern "C" int psfm_grid_sample(const float* map, int32_t h, int32_t w, int32_t channels, const double* xy, int32_t n, float* out) {
  if (!map || !xy || !out || h < 2 || w < 2 || channels < 1 || channels > 2 || n < 0) return PSFM_ERR_INVALID;
  int rc = device_ok();
  if (rc != PSFM_OK) return rc;
  if (n == 0) return PSFM_OK;
  try {
    DBuf<float> dm, dout; DBuf<double> dxy;
    dm.alloc((size_t)h * w * channels); dxy.alloc(2 * (size_t)n); dout.alloc((size_t)n * channels);
    dm.upload(map, dm.n, nullptr); dxy.upload(xy, dxy.n, nullptr);
    k_grid_sample<<<grid_of(n), 256>>>(dm.p, h, w, channels, dxy.p, n, dout.p);
    PSFM_LAUNCH_CHECK();
    PSFM_CUDA(cudaMemcpy(out, dout.p, sizeof(float) * dout.n, cudaMemcpyDeviceToHost));
    return PSFM_OK;
  } catch (const CudaFail& f) { return f.code; }
}

extern "C" int psfm_flow_check(const float* flow_f, const float* flow_b, int32_t h, int32_t w, float thres, float* err, uint8_t* occ) {
  if (!flow_f || !flow_b || !occ || h < 2 || w < 2) return PSFM_ERR_INVALID;
  int rc = device_ok();
  if (rc != PSFM_OK) return rc;
  try {
    const size_t hw = (size_t)h * w;
    DBuf<float> df, db, de; DBuf<unsigned char> dof;
    df.alloc(2 * hw); db.alloc(2 * hw); de.alloc(hw); dof.alloc(hw);
    df.upload(flow_f, 2 * hw, nullptr); db.upload(flow_b, 2 * hw, nullptr);
    k_flow_check<<<grid_of(hw), 256>>>(df.p, db.p, h, w, thres, de.p, dof.p);
    PSFM_LAUNCH_CHECK();
    if (err) PSFM_CUDA(cudaMemcpy(err, de.p, sizeof(float) * hw, cudaMemcpyDeviceToHost));
    PSFM_CUDA(cudaMemcpy(occ, dof.p, hw, cudaMemcpyDeviceToHost));
    return PSFM_OK;
  } catch (const CudaFail& f) { return f.code; }
}

extern "C" int psfm_tracker_step(const float* flow, const uint8_t* occ, int32_t h, int32_t w, const double* cur_xy, int32_t n,
                                 int32_t sample_ratio, double* next_xy, uint8_t* flags, uint8_t* reseed_mask) {
  if (!flow || !occ || !cur_xy || !next_xy || !flags || h < 2 || w < 2 || n < 0 || sample_ratio < 1) return PSFM_ERR_INVALID;
  int rc = device_ok();
  if (rc != PSFM_OK) return rc;
  try {
    const size_t hw = (size_t)h * w;
    const int gh = (h + sample_ratio - 1) / sample_ratio, gw = (w + sample_ratio - 1) / sample_ratio;
    DBuf<float> df; DBuf<unsigned char> dof, dfl, docc, dmask; DBuf<double> dcur, dnext, dkept;
    df.alloc(2 * hw); dof.alloc(hw); dcur.alloc(2 * (size_t)n); dnext.alloc(2 * (size_t)n); dfl.alloc(n);
    df.upload(flow, 2 * hw, nullptr); dof.upload(occ, hw, nullptr); dcur.upload(cur_xy, 2 * (size_t)n, nullptr);
    if (n) { k_tracker_step<<<grid_of(n), 256>>>(df.p, dof.p, h, w, dcur.p, n, dnext.p, dfl.p); PSFM_LAUNCH_CHECK(); }
    if (n) PSFM_CUDA(cudaMemcpy(next_xy, dnext.p, sizeof(double) * 2 * (size_t)n, cudaMemcpyDeviceToHost));
    if (n) PSFM_CUDA(cudaMemcpy(flags, dfl.p, (size_t)n, cudaMemcpyDeviceToHost));
    if (reseed_mask) {
      // occupancy of the SURVIVORS' next positions (extend_all), then the thresholded distance transform
      std::vector<double> kept;
      kept.reserve(2 * (size_t)n);
      for (int i = 0; i < n; ++i)
        if (flags[i]) { kept.push_back(next_xy[2 * (size_t)i]); kept.push_back(next_xy[2 * (size_t)i + 1]); }
      const int nk = (int)(kept.size() / 2);
      docc.alloc(hw); dmask.alloc((size_t)gh * gw); dkept.alloc(kept.size());
      PSFM_CUDA(cudaMemset(docc.p, 0, hw));
      dkept.upload(kept.data(), kept.size(), nullptr);
      if (nk) { k_occupancy<<<grid_of(nk), 256>>>(dkept.p, nk, h, w, docc.p); PSFM_LAUNCH_CHECK(); }
      k_reseed_mask<<<grid_of((size_t)gh * gw), 256>>>(docc.p, h, w, sample_ratio, gh, gw, dmask.p);
      PSFM_LAUNCH_CHECK();
      PSFM_CUDA(cudaMemcpy(reseed_mask, dmask.p, (size_t)gh * gw, cudaMemcpyDeviceToHost));
    }
    return PSFM_OK;
  } catch (const CudaFail& f) { return f.code; }
}

extern "C" int psfm_tracker_buffer_inputs(const float* flow01, const float* flow02, const uint8_t* occ02, int32_t h, int32_t w,
                                          const double* x0, int32_t n, double upper_flow, double* ref1, double* ref2, double* scale) {
  if (!flow01 || !flow02 || !occ02 || !x0 || !ref1 || !ref2 || !scale || h < 2 || w < 2 || n < 0) return PSFM_ERR_INVALID;
  int rc = device_ok();
  if (rc != PSFM_OK) return rc;
  if (n == 0) return PSFM_OK;
  try {
    const size_t hw = (size_t)h * w;
    DBuf<float> d1, d2; DBuf<unsigned char> dof; DBuf<double> dx, r1, r2, sc;
    d1.alloc(2 * hw); d2.alloc(2 * hw); dof.alloc(hw); dx.alloc(2 * (size_t)n); r1.alloc(2 * (size_t)n); r2.alloc(2 * (size_t)n); sc.alloc(n);
    d1.upload(flow01, 2 * hw, nullptr); d2.upload(flow02, 2 * hw, nullptr); dof.upload(occ02, hw, nullptr); dx.upload(x0, 2 * (size_t)n, nullptr);
    k_buffer_inputs<<<grid_of(n), 256>>>(d1.p, d2.p, dof.p, h, w, dx.p, n, upper_flow, r1.p, r2.p, sc.p);
    PSFM_LAUNCH_CHECK();
    PSFM_CUDA(cudaMemcpy(ref1, r1.p, sizeof(double) * 2 * (size_t)n, cudaMemcpyDeviceToHost));
    PSFM_CUDA(cudaMemcpy(ref2, r2.p, sizeof(double) * 2 * (size_t)n, cudaMemcpyDeviceToHost));
    PSFM_CUDA(cudaMemcpy(scale, sc.p, sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost));
    return PSFM_OK;
  } catch (const CudaFail& f) { return f.code; }
}
