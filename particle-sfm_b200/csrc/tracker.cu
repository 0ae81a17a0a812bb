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
#include <thrust/iterator/transform_iterator.h>

#include <algorithm>
#include <cub/device/device_scan.cuh>
#include <vector>

#include "match_table.cuh"
#include "psfm_common.cuh"
#include "track_npy.cuh"
#include "traj_solver.cuh"

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

__device__ __forceinline__ void mark_occupied(const double* xy, int H, int W, unsigned char* occ) {
  const long long x = (long long)xy[0], y = (long long)xy[1];      // astype(int64): truncation
  if (x >= 0 && x < W && y >= 0 && y < H) occ[(size_t)y * W + x] = 1;
}

__global__ void k_occupancy(const double* xy, int n, int H, int W, unsigned char* occ) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  mark_occupied(xy + 2 * (size_t)i, H, W, occ);
}

// (distance_transform_edt(1 - occupied) > ratio)[::ratio, ::ratio]: a strided grid point is a new seed iff no
// occupied pixel lies within squared distance ratio^2
__device__ __forceinline__ bool occupied_near(const unsigned char* occ, int H, int W, int ratio, int y, int x) {
  const int r2 = ratio * ratio;
  for (int dy = -ratio; dy <= ratio; ++dy) {
    const int yy = y + dy;
    if (yy < 0 || yy >= H) continue;
    for (int dx = -ratio; dx <= ratio; ++dx) {
      const int xx = x + dx;
      if (xx < 0 || xx >= W || dy * dy + dx * dx > r2) continue;
      if (occ[(size_t)yy * W + xx]) return true;
    }
  }
  return false;
}

__global__ void k_reseed_mask(const unsigned char* occ, int H, int W, int ratio, int GH, int GW, unsigned char* mask) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= GH * GW) return;
  mask[g] = occupied_near(occ, H, W, ratio, (g / GW) * ratio, (g % GW) * ratio) ? 0 : 1;
}

// ------------------------------------------------------------------ resident stage (psfm_tracker_*)
//
// The active list mirrors the reference's active_trajs: entry i is the particle in slot i of history[t]
// (survivors first, then this frame's seeds), with its id, length and its slots one and two steps back.
// Every compaction is an exclusive scan of 0/1 flags followed by a scatter, so it keeps the active order.

// new_traj_all (trajectory.py:117-120): the grid points whose mask is set (all of them when mask == NULL),
// in row-major order, appended after the `base` survivors of history[t] and of the active list
__global__ void k_seed(const unsigned char* mask, const int* pos, int G, int GW, int ratio, int next_id, int base,
                       int* hid, double* hxy, int* act_id, int* act_len, int* act_m1, int* act_m2) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G || (mask && !mask[g])) return;
  const int k = mask ? pos[g] : g;
  const size_t i = (size_t)base + k;
  hid[i] = next_id + k;
  hxy[2 * i] = (double)((g % GW) * ratio);
  hxy[2 * i + 1] = (double)((g / GW) * ratio);
  act_id[i] = next_id + k; act_len[i] = 1; act_m1[i] = -1; act_m2[i] = -1;
}

// extend_all (trajectory.py:129-152): survivors move to the new active list and to history[t + 1] in active
// order; the others retire, ranked in active order after the `retired` already retired ones
__global__ void k_extend(int n, const unsigned char* flags, const int* pos, const double* next, const int* act_id,
                         const int* act_len, const int* act_m1, int t, int retired, int* nid, int* nlen, int* nm1, int* nm2,
                         int* hid_next, double* hxy_next, int* rank, int* rlen, int* rstart) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int p = pos[i], id = act_id[i], len = act_len[i];
  if (flags[i]) {
    nid[p] = id; nlen[p] = len + 1; nm1[p] = i; nm2[p] = act_m1[i];
    hid_next[p] = id;
    hxy_next[2 * (size_t)p] = next[2 * (size_t)i];
    hxy_next[2 * (size_t)p + 1] = next[2 * (size_t)i + 1];
  } else {
    const int r = retired + (i - p);
    rank[id] = r; rlen[r] = len; rstart[r] = t - len + 1;
  }
}

// number of set flags, from the exclusive scan of them
__global__ void k_total(const unsigned char* flags, const int* pos, int n, int* out) {
  *out = n ? pos[n - 1] + (flags[n - 1] ? 1 : 0) : 0;
}

__global__ void k_occupancy_kept(const double* next, const unsigned char* flags, int n, int H, int W, unsigned char* occ) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !flags[i]) return;
  mark_occupied(next + 2 * (size_t)i, H, W, occ);
}

// the re-seed mask of extend_all.  Without a survivor, the occupancy map scipy's distance_transform_edt
// receives ([H, W, 1], 1 - occupied) has no zero; scipy 1.x then returns sqrt((y + 1)^2 + x^2) at (y, x, 0).
__global__ void k_reseed_stage(const unsigned char* occ, int H, int W, int ratio, int GH, int GW, const int* num_survivors,
                               unsigned char* mask) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= GH * GW) return;
  const int y = (g / GW) * ratio, x = (g % GW) * ratio;
  if (*num_survivors == 0) {
    const long long d2 = (long long)(y + 1) * (y + 1) + (long long)x * x;
    mask[g] = d2 > (long long)ratio * ratio ? 1 : 0;
  } else {
    mask[g] = occupied_near(occ, H, W, ratio, y, x) ? 0 : 1;
  }
}

// optimize_buffer's selection (trajectory.py:165): the survivors with three observations, in active order
__global__ void k_buffer_flags(const int* len, const int* num_survivors, int n, unsigned char* flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  flags[i] = (i < *num_survivors && len[i] >= 3) ? 1 : 0;
}

// x0 = history[t-1], uv12 = (history[t], history[t+1]) of the selected particles, and their active slot
__global__ void k_buffer_gather(int n, const unsigned char* flags, const int* pos, const int* m1, const int* m2,
                                const double* hxy_prev, const double* hxy_cur, const double* hxy_next, double* x0,
                                double* uv12, int* slot) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !flags[i]) return;
  const size_t b = pos[i], a = m2[i], c = m1[i];
  x0[2 * b] = hxy_prev[2 * a]; x0[2 * b + 1] = hxy_prev[2 * a + 1];
  uv12[4 * b] = hxy_cur[2 * c]; uv12[4 * b + 1] = hxy_cur[2 * c + 1];
  uv12[4 * b + 2] = hxy_next[2 * (size_t)i]; uv12[4 * b + 3] = hxy_next[2 * (size_t)i + 1];
  slot[b] = i;
}

// optimize_buffer's write-back (trajectory.py:190-194): optimised x1 into history[t], x2 into history[t+1]
__global__ void k_writeback(int n, const double* out, const int* slot, const int* m1, double* hxy_cur, double* hxy_next) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n) return;
  const size_t j = slot[b], c = m1[j];
  hxy_cur[2 * c] = out[4 * (size_t)b]; hxy_cur[2 * c + 1] = out[4 * (size_t)b + 1];
  hxy_next[2 * j] = out[4 * (size_t)b + 2]; hxy_next[2 * j + 1] = out[4 * (size_t)b + 3];
}

// clear_active (trajectory.py:154-159): the particles still alive at time t retire in active order
__global__ void k_clear_active(int n, const int* act_id, const int* act_len, int t, int retired, int* rank, int* rlen, int* rstart) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int r = retired + i, len = act_len[i];
  rank[act_id[i]] = r; rlen[r] = len; rstart[r] = t - len + 1;
}

// main_connect_point_trajectories.py:57-60: keep the trajectories of at least min_len observations
__global__ void k_keep(int T, const int* rlen, int min_len, unsigned char* keep, long long* klen) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= T) return;
  const bool k = rlen[r] >= min_len;
  keep[r] = k ? 1 : 0;
  klen[r] = k ? rlen[r] : 0;
}

__global__ void k_emit_ids(int T, const unsigned char* keep, const int* kpos, const long long* off, const long long* klen,
                           long long* ids, long long* ptr, long long* totals) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= T) return;
  if (keep[r]) { ids[kpos[r]] = r; ptr[kpos[r]] = off[r]; }
  if (r == T - 1) {
    const long long nt = kpos[r] + (keep[r] ? 1 : 0), m = off[r] + klen[r];
    ptr[nt] = m;
    totals[0] = nt; totals[1] = m;
  }
}

// every observation of time t goes to offset[rank] + (t - start[rank]): the track set in full_trajs order
__global__ void k_emit_obs(int n, int t, const int* hid, const double* hxy, const int* rank, const unsigned char* keep,
                           const long long* off, const int* rstart, int* frame_ids, double* xy) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int r = rank[hid[i]];
  if (!keep[r]) return;
  const size_t o = (size_t)(off[r] + (t - rstart[r]));
  frame_ids[o] = t;
  xy[2 * o] = hxy[2 * (size_t)i]; xy[2 * o + 1] = hxy[2 * (size_t)i + 1];
}

struct FlagToInt {
  __host__ __device__ int operator()(unsigned char f) const { return f ? 1 : 0; }
};

}  // namespace

extern "C" int psfm_grid_sample(const float* map, int32_t h, int32_t w, int32_t channels, const double* xy, int32_t n, float* out) {
  return guard("psfm_grid_sample", [&]() -> int {
    if (!map || !xy || !out || h < 2 || w < 2 || channels < 1 || channels > 2 || n < 0) return PSFM_ERR_INVALID;
    int rc = require_device("psfm_grid_sample");
    if (rc != PSFM_OK) return rc;
    if (n == 0) return PSFM_OK;
    DBuf<float> dm, dout; DBuf<double> dxy;
    dm.alloc((size_t)h * w * channels); dxy.alloc(2 * (size_t)n); dout.alloc((size_t)n * channels);
    dm.upload(map, dm.n, nullptr); dxy.upload(xy, dxy.n, nullptr);
    k_grid_sample<<<grid_of(n), 256>>>(dm.p, h, w, channels, dxy.p, n, dout.p);
    PSFM_LAUNCH_CHECK();
    PSFM_CUDA(cudaMemcpy(out, dout.p, sizeof(float) * dout.n, cudaMemcpyDeviceToHost));
    return PSFM_OK;
  });
}

extern "C" int psfm_flow_check(const float* flow_f, const float* flow_b, int32_t h, int32_t w, float thres, float* err, uint8_t* occ) {
  return guard("psfm_flow_check", [&]() -> int {
    if (!flow_f || !flow_b || !occ || h < 2 || w < 2) return PSFM_ERR_INVALID;
    int rc = require_device("psfm_flow_check");
    if (rc != PSFM_OK) return rc;
    const size_t hw = (size_t)h * w;
    DBuf<float> df, db, de; DBuf<unsigned char> dof;
    df.alloc(2 * hw); db.alloc(2 * hw); de.alloc(hw); dof.alloc(hw);
    df.upload(flow_f, 2 * hw, nullptr); db.upload(flow_b, 2 * hw, nullptr);
    k_flow_check<<<grid_of(hw), 256>>>(df.p, db.p, h, w, thres, de.p, dof.p);
    PSFM_LAUNCH_CHECK();
    if (err) PSFM_CUDA(cudaMemcpy(err, de.p, sizeof(float) * hw, cudaMemcpyDeviceToHost));
    PSFM_CUDA(cudaMemcpy(occ, dof.p, hw, cudaMemcpyDeviceToHost));
    return PSFM_OK;
  });
}

extern "C" int psfm_tracker_step(const float* flow, const uint8_t* occ, int32_t h, int32_t w, const double* cur_xy, int32_t n,
                                 int32_t sample_ratio, double* next_xy, uint8_t* flags, uint8_t* reseed_mask) {
  return guard("psfm_tracker_step", [&]() -> int {
    if (!flow || !occ || !cur_xy || !next_xy || !flags || h < 2 || w < 2 || n < 0 || sample_ratio < 1) return PSFM_ERR_INVALID;
    int rc = require_device("psfm_tracker_step");
    if (rc != PSFM_OK) return rc;
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
  });
}

extern "C" int psfm_tracker_buffer_inputs(const float* flow01, const float* flow02, const uint8_t* occ02, int32_t h, int32_t w,
                                          const double* x0, int32_t n, double upper_flow, double* ref1, double* ref2, double* scale) {
  return guard("psfm_tracker_buffer_inputs", [&]() -> int {
    if (!flow01 || !flow02 || !occ02 || !x0 || !ref1 || !ref2 || !scale || h < 2 || w < 2 || n < 0) return PSFM_ERR_INVALID;
    int rc = require_device("psfm_tracker_buffer_inputs");
    if (rc != PSFM_OK) return rc;
    if (n == 0) return PSFM_OK;
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
  });
}

// ------------------------------------------------------------------ resident stage: host side

namespace {

template <typename T>
void swap_buf(DBuf<T>& a, DBuf<T>& b) {
  std::swap(a.p, b.p); std::swap(a.n, b.n); std::swap(a.st, b.st); std::swap(a.async, b.async);
}

// capacity >= need, the first `keep` elements preserved; grows geometrically
template <typename T>
void grow(DBuf<T>& b, size_t need, size_t keep, cudaStream_t st) {
  if (b.p && b.n >= need) return;
  DBuf<T> nb;
  nb.alloc(std::max(need, 2 * b.n), st);
  if (keep) PSFM_CUDA(cudaMemcpyAsync(nb.p, b.p, keep * sizeof(T), cudaMemcpyDeviceToDevice, st));
  swap_buf(b, nb);
}

}  // namespace

struct psfm_tracker {
  int h = 0, w = 0, ratio = 1, gh = 0, gw = 0, num_frames = 0;
  bool path_consistency = true;   // false: track.py:24-50, no buffer and no HP1
  cudaStream_t st = nullptr;
  int t = 0;                      // frames advanced; the active particles live at time t
  int n_active = 0;               // = history[t]'s survivors until the next seeding
  int seeds = 0;                  // seeds of the next frame (set bits of `mask`)
  int next_id = 0, retired = 0;
  int n_buf = 0, buf_frame = -1;  // buffered set of frame buf_frame waiting for HP1 (n_buf > 0)
  const float* flow12 = nullptr;  // flows[buf_frame] (the caller's map)
  bool finished = false;
  bool failed = false;            // a CUDA failure left the device state unknown: every later call is refused
  long long res_trajs = 0, res_obs = 0;
  std::vector<long long> hoff;    // history[s] starts at hoff[s]
  std::vector<int> hcnt;          // particles alive at time s
  DBuf<int> hid; DBuf<double> hxy;
  DBuf<int> act_id[2], act_len[2], act_m1[2], act_m2[2];
  int cur = 0;
  DBuf<double> next; DBuf<unsigned char> flags, bflags; DBuf<int> pos, bpos;
  DBuf<unsigned char> occ, mask; DBuf<int> mpos;
  DBuf<int> rank, rlen, rstart;
  DBuf<double> bx0, buv, bref1, bref2, bscale, bout; DBuf<int> bslot;
  DBuf<unsigned char> keep; DBuf<int> kpos; DBuf<long long> klen, off, ids, ptr, totals;
  DBuf<int> res_frames; DBuf<double> res_xy;
  DBuf<unsigned char> tmp;        // CUB scratch
  DBuf<int> d_counts;
  int* h_counts = nullptr;        // pinned [3]
  long long* h_totals = nullptr;  // pinned [2]

  template <typename In, typename Out>
  void scan(In in, Out out, int n) {
    if (n == 0) return;
    size_t bytes = 0;
    PSFM_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, n, st));
    grow(tmp, bytes, 0, st);
    PSFM_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, bytes, in, out, n, st));
    PSFM_LAUNCH_CHECK();
  }
  void scan_flags(const unsigned char* f, int* out, int n) { scan(thrust::make_transform_iterator(f, FlagToInt()), out, n); }
  void sync() { PSFM_CUDA(cudaStreamSynchronize(st)); }
};

namespace {

// argument check shared by the calls on a handle: PSFM_OK or the error to return
int tracker_usable(const psfm_tracker* T, bool args_ok, const char* fn) {
  if (!T || !args_ok) return fail(fn, PSFM_ERR_INVALID, "null argument");
  if (T->failed) return fail(fn, PSFM_ERR_INVALID, "an earlier call on this tracker failed; destroy it");
  return PSFM_OK;
}

// a failure left the device state unknown (T is NULL when the argument check itself threw)
int tracker_broken(psfm_tracker* T, int code) {
  if (T) T->failed = true;
  return code;
}

}  // namespace

extern "C" int psfm_flow_check_device(const float* d_flow_f, const float* d_flow_b, int32_t h, int32_t w, float thres, float* d_err,
                                      uint8_t* d_occ, void* stream) {
  return guard("psfm_flow_check_device", [&]() -> int {
    if (!d_flow_f || !d_flow_b || !d_occ) return fail("psfm_flow_check_device", PSFM_ERR_INVALID, "null argument");
    if (h < 2 || w < 2) return fail("psfm_flow_check_device", PSFM_ERR_INVALID, "bad sizes");
    int rc = require_device("psfm_flow_check_device");
    if (rc != PSFM_OK) return rc;
    const size_t hw = (size_t)h * w;
    k_flow_check<<<grid_of(hw), 256, 0, (cudaStream_t)stream>>>(d_flow_f, d_flow_b, h, w, thres, d_err, d_occ);
    PSFM_LAUNCH_CHECK();
    return PSFM_OK;
  });
}

namespace {

int tracker_create(const char* entry, int32_t h, int32_t w, int32_t sample_ratio, int32_t num_frames, int32_t path_consistency,
                   void* stream, psfm_tracker** out) {
  if (!out) return fail(entry, PSFM_ERR_INVALID, "null argument");
  *out = nullptr;
  if (h < 2 || w < 2 || sample_ratio < 1 || num_frames < 1) return fail(entry, PSFM_ERR_INVALID, "bad sizes");
  if (path_consistency != 0 && path_consistency != 1) return fail(entry, PSFM_ERR_INVALID, "path_consistency must be 0 or 1");
  int rc = require_device(entry);
  if (rc != PSFM_OK) return rc;
  std::unique_ptr<psfm_tracker, decltype(&psfm_tracker_destroy)> T(new psfm_tracker, psfm_tracker_destroy);
  T->h = h; T->w = w; T->ratio = sample_ratio; T->num_frames = num_frames;
  T->path_consistency = path_consistency != 0;
  T->gh = (h + sample_ratio - 1) / sample_ratio; T->gw = (w + sample_ratio - 1) / sample_ratio;
  T->st = (cudaStream_t)stream;
  T->hoff.assign(1, 0);
  T->hcnt.assign(1, 0);
  const size_t G = (size_t)T->gh * T->gw;
  T->occ.alloc((size_t)h * w, T->st);
  T->mask.alloc(G, T->st);
  T->mpos.alloc(G, T->st);
  T->d_counts.alloc(3, T->st);
  T->totals.alloc(2, T->st);
  PSFM_CUDA(cudaMallocHost((void**)&T->h_counts, 3 * sizeof(int)));
  PSFM_CUDA(cudaMallocHost((void**)&T->h_totals, 2 * sizeof(long long)));
  *out = T.release();
  return PSFM_OK;
}

}  // namespace

extern "C" int psfm_tracker_create(int32_t h, int32_t w, int32_t sample_ratio, int32_t num_frames, void* stream, psfm_tracker** out) {
  const char* entry = "psfm_tracker_create";
  return guard(entry, [&] { return tracker_create(entry, h, w, sample_ratio, num_frames, 1, stream, out); });
}

extern "C" int psfm_tracker_create_mode(int32_t h, int32_t w, int32_t sample_ratio, int32_t num_frames, int32_t path_consistency,
                                        void* stream, psfm_tracker** out) {
  const char* entry = "psfm_tracker_create_mode";
  return guard(entry, [&] { return tracker_create(entry, h, w, sample_ratio, num_frames, path_consistency, stream, out); });
}

extern "C" int psfm_tracker_advance(psfm_tracker* T, const float* d_flow, const uint8_t* d_occ, const float* d_flow_prev,
                                    const float* d_flow2_prev, const uint8_t* d_occ2_prev, int32_t* counts) {
  const char* entry = "psfm_tracker_advance";
  return guard(entry, [&]() -> int {
    int rc = tracker_usable(T, d_flow && d_occ, entry);
    if (rc != PSFM_OK) return rc;
    if (T->finished) return fail(entry, PSFM_ERR_INVALID, "the track set was already assembled");
    if (T->n_buf > 0) return fail(entry, PSFM_ERR_INVALID, "the buffered set of the previous frame was not optimised");
    if (T->t + 1 >= T->num_frames) return fail(entry, PSFM_ERR_INVALID, "more frames than the tracker was created for");
    if (T->path_consistency && T->t >= 1 && (!d_flow_prev || !d_flow2_prev || !d_occ2_prev))
      return fail(entry, PSFM_ERR_INVALID, "from frame 1 on, flows[t-1], flows_f2[t-1] and occ_maps_s2[t-1] are needed");
    cudaStream_t st = T->st;
    const int t = T->t, G = T->gh * T->gw, H = T->h, W = T->w;
    const int seeds = t == 0 ? G : T->seeds, base = T->n_active, n = base + seeds;
    const long long h0 = T->hoff[t], h1 = h0 + n;
    // capacities: history[t + 1] gets at most n entries; ids, ranks and the per-frame scratch grow with them
    grow(T->hid, (size_t)(h1 + n), (size_t)(h0 + base), st);
    grow(T->hxy, 2 * (size_t)(h1 + n), 2 * (size_t)(h0 + base), st);
    const int c = T->cur, d = 1 - c;
    grow(T->act_id[c], n, base, st); grow(T->act_len[c], n, base, st);
    grow(T->act_m1[c], n, base, st); grow(T->act_m2[c], n, base, st);
    grow(T->act_id[d], n, 0, st); grow(T->act_len[d], n, 0, st); grow(T->act_m1[d], n, 0, st); grow(T->act_m2[d], n, 0, st);
    const size_t ids_now = (size_t)T->next_id + seeds;
    grow(T->rank, ids_now, T->next_id, st); grow(T->rlen, ids_now, T->next_id, st); grow(T->rstart, ids_now, T->next_id, st);
    grow(T->next, 2 * (size_t)n, 0, st); grow(T->flags, n, 0, st); grow(T->pos, n, 0, st);
    if (T->path_consistency) {
      grow(T->bflags, n, 0, st); grow(T->bpos, n, 0, st);
      grow(T->bx0, 2 * (size_t)n, 0, st); grow(T->buv, 4 * (size_t)n, 0, st); grow(T->bslot, n, 0, st);
      grow(T->bref1, 2 * (size_t)n, 0, st); grow(T->bref2, 2 * (size_t)n, 0, st); grow(T->bscale, n, 0, st);
      grow(T->bout, 4 * (size_t)n, 0, st);
    }
    int* hid_t = T->hid.p + h0;
    double* hxy_t = T->hxy.p + 2 * h0;
    // 1. seed (new_traj_all)
    if (seeds) {
      k_seed<<<grid_of(G), 256, 0, st>>>(t == 0 ? nullptr : T->mask.p, T->mpos.p, G, T->gw, T->ratio, T->next_id, base, hid_t, hxy_t,
                                         T->act_id[c].p, T->act_len[c].p, T->act_m1[c].p, T->act_m2[c].p);
      PSFM_LAUNCH_CHECK();
    }
    // 2. step (step_forward) from history[t], which is in active order
    if (n) {
      k_tracker_step<<<grid_of(n), 256, 0, st>>>(d_flow, d_occ, H, W, hxy_t, n, T->next.p, T->flags.p);
      PSFM_LAUNCH_CHECK();
    }
    // 3. extend (extend_all): stable compaction, retire ranks, then the re-seed mask of the survivors' next positions
    T->scan_flags(T->flags.p, T->pos.p, n);
    if (n) {
      k_extend<<<grid_of(n), 256, 0, st>>>(n, T->flags.p, T->pos.p, T->next.p, T->act_id[c].p, T->act_len[c].p, T->act_m1[c].p, t,
                                           T->retired, T->act_id[d].p, T->act_len[d].p, T->act_m1[d].p, T->act_m2[d].p,
                                           T->hid.p + h1, T->hxy.p + 2 * h1, T->rank.p, T->rlen.p, T->rstart.p);
      PSFM_LAUNCH_CHECK();
    }
    k_total<<<1, 1, 0, st>>>(T->flags.p, T->pos.p, n, T->d_counts.p);
    PSFM_LAUNCH_CHECK();
    PSFM_CUDA(cudaMemsetAsync(T->occ.p, 0, (size_t)H * W, st));
    if (n) {
      k_occupancy_kept<<<grid_of(n), 256, 0, st>>>(T->next.p, T->flags.p, n, H, W, T->occ.p);
      PSFM_LAUNCH_CHECK();
    }
    k_reseed_stage<<<grid_of(G), 256, 0, st>>>(T->occ.p, H, W, T->ratio, T->gh, T->gw, T->d_counts.p, T->mask.p);
    PSFM_LAUNCH_CHECK();
    T->scan_flags(T->mask.p, T->mpos.p, G);
    k_total<<<1, 1, 0, st>>>(T->mask.p, T->mpos.p, G, T->d_counts.p + 1);
    PSFM_LAUNCH_CHECK();
    // 4. buffer (optimize_buffer's selection and gather), from frame 1 on, with path consistency only
    if (T->path_consistency && t >= 1 && n) {
      k_buffer_flags<<<grid_of(n), 256, 0, st>>>(T->act_len[d].p, T->d_counts.p, n, T->bflags.p);
      PSFM_LAUNCH_CHECK();
      T->scan_flags(T->bflags.p, T->bpos.p, n);
      k_total<<<1, 1, 0, st>>>(T->bflags.p, T->bpos.p, n, T->d_counts.p + 2);
      PSFM_LAUNCH_CHECK();
      k_buffer_gather<<<grid_of(n), 256, 0, st>>>(n, T->bflags.p, T->bpos.p, T->act_m1[d].p, T->act_m2[d].p,
                                                  T->hxy.p + 2 * T->hoff[t - 1], hxy_t, T->hxy.p + 2 * h1, T->bx0.p, T->buv.p,
                                                  T->bslot.p);
      PSFM_LAUNCH_CHECK();
    } else {
      PSFM_CUDA(cudaMemsetAsync(T->d_counts.p + 2, 0, sizeof(int), st));
    }
    PSFM_CUDA(cudaMemcpyAsync(T->h_counts, T->d_counts.p, 3 * sizeof(int), cudaMemcpyDeviceToHost, st));
    T->sync();
    // the host-side state moves on only once the frame's device work has completed
    const int survivors = T->h_counts[0];
    T->hcnt[t] = n;
    T->hoff.push_back(h1);
    T->next_id += seeds;
    T->retired += n - survivors;
    T->n_active = survivors;
    T->seeds = T->h_counts[1];
    T->cur = d;
    T->t = t + 1;
    T->hcnt.push_back(survivors);
    T->n_buf = T->h_counts[2];
    T->buf_frame = t;
    T->flow12 = d_flow;
    if (T->n_buf > 0) {
      k_buffer_inputs<<<grid_of(T->n_buf), 256, 0, st>>>(d_flow_prev, d_flow2_prev, d_occ2_prev, H, W, T->bx0.p, T->n_buf, 20.0,
                                                          T->bref1.p, T->bref2.p, T->bscale.p);
      PSFM_LAUNCH_CHECK();
    }
    if (counts) { counts[0] = survivors; counts[1] = T->seeds; counts[2] = T->n_buf; }
    return PSFM_OK;
  }, [&](int code) { return tracker_broken(T, code); });
}

namespace {

int tracker_writeback(psfm_tracker* T) {
  const int t = T->buf_frame;
  k_writeback<<<grid_of(T->n_buf), 256, 0, T->st>>>(T->n_buf, T->bout.p, T->bslot.p, T->act_m1[T->cur].p, T->hxy.p + 2 * T->hoff[t],
                                                     T->hxy.p + 2 * T->hoff[t + 1]);
  PSFM_LAUNCH_CHECK();
  T->n_buf = 0;
  return PSFM_OK;
}

}  // namespace

extern "C" int psfm_tracker_optimize(psfm_tracker* T, const psfm_traj_options* opts, psfm_traj_summary* summary) {
  return guard("psfm_tracker_optimize", [&]() -> int {
    if (summary) memset(summary, 0, sizeof(*summary));
    int rc = tracker_usable(T, true, "psfm_tracker_optimize");
    if (rc != PSFM_OK) return rc;
    if (T->n_buf <= 0) return fail("psfm_tracker_optimize", PSFM_ERR_INVALID, "no buffered trajectory");
    // HP1 runs on the tracker's stream, after k_buffer_inputs.  NULL (the legacy default stream) is passed as
    // cudaStreamLegacy: a NULL stream would make solve_device use the HP1 workspace's non-blocking stream, which
    // is not ordered after the legacy stream's work.
    rc = traj::solve_device(T->buv.p, T->bref1.p, T->bref2.p, T->bscale.p, T->flow12, T->n_buf, T->w, T->h, opts, T->bout.p,
                            summary, T->st ? T->st : cudaStreamLegacy);
    if (rc != PSFM_OK) return tracker_broken(T, rc);
    return tracker_writeback(T);
  }, [&](int code) { return tracker_broken(T, code); });
}

extern "C" int psfm_tracker_get_buffer(psfm_tracker* T, double* uv12, double* ref1, double* ref2, double* scale) {
  return guard("psfm_tracker_get_buffer", [&]() -> int {
    int rc = tracker_usable(T, uv12 && ref1 && ref2 && scale, "psfm_tracker_get_buffer");
    if (rc != PSFM_OK) return rc;
    if (T->n_buf <= 0) return fail("psfm_tracker_get_buffer", PSFM_ERR_INVALID, "no buffered trajectory");
    const size_t n = T->n_buf;
    PSFM_CUDA(cudaMemcpyAsync(uv12, T->buv.p, 4 * n * sizeof(double), cudaMemcpyDeviceToHost, T->st));
    PSFM_CUDA(cudaMemcpyAsync(ref1, T->bref1.p, 2 * n * sizeof(double), cudaMemcpyDeviceToHost, T->st));
    PSFM_CUDA(cudaMemcpyAsync(ref2, T->bref2.p, 2 * n * sizeof(double), cudaMemcpyDeviceToHost, T->st));
    PSFM_CUDA(cudaMemcpyAsync(scale, T->bscale.p, n * sizeof(double), cudaMemcpyDeviceToHost, T->st));
    T->sync();
    return PSFM_OK;
  }, [&](int code) { return tracker_broken(T, code); });
}

extern "C" int psfm_tracker_set_buffer(psfm_tracker* T, const double* uv12) {
  return guard("psfm_tracker_set_buffer", [&]() -> int {
    int rc = tracker_usable(T, uv12 != nullptr, "psfm_tracker_set_buffer");
    if (rc != PSFM_OK) return rc;
    if (T->n_buf <= 0) return fail("psfm_tracker_set_buffer", PSFM_ERR_INVALID, "no buffered trajectory");
    PSFM_CUDA(cudaMemcpyAsync(T->bout.p, uv12, 4 * (size_t)T->n_buf * sizeof(double), cudaMemcpyHostToDevice, T->st));
    rc = tracker_writeback(T);
    T->sync();        // uv12 is the caller's (possibly pageable) memory
    return rc;
  }, [&](int code) { return tracker_broken(T, code); });
}

extern "C" int psfm_tracker_finish(psfm_tracker* T, int32_t traj_min_len, int64_t* num_trajs, int64_t* num_obs) {
  return guard("psfm_tracker_finish", [&]() -> int {
    int rc = tracker_usable(T, num_trajs && num_obs, "psfm_tracker_finish");
    if (rc != PSFM_OK) return rc;
    if (T->finished) return fail("psfm_tracker_finish", PSFM_ERR_INVALID, "already finished");
    if (T->n_buf > 0) return fail("psfm_tracker_finish", PSFM_ERR_INVALID, "the buffered set of the last frame was not optimised");
    cudaStream_t st = T->st;
    const int t = T->t;
    if (T->n_active) {
      k_clear_active<<<grid_of(T->n_active), 256, 0, st>>>(T->n_active, T->act_id[T->cur].p, T->act_len[T->cur].p, t, T->retired,
                                                            T->rank.p, T->rlen.p, T->rstart.p);
      PSFM_LAUNCH_CHECK();
    }
    T->retired += T->n_active;
    T->n_active = 0;
    const int NT = T->next_id;    // every id is retired now: ranks 0 .. NT-1
    T->finished = true;
    if (NT == 0) { *num_trajs = *num_obs = T->res_trajs = T->res_obs = 0; return PSFM_OK; }
    grow(T->keep, NT, 0, st); grow(T->kpos, NT, 0, st); grow(T->klen, NT, 0, st); grow(T->off, NT, 0, st);
    grow(T->ids, NT, 0, st); grow(T->ptr, (size_t)NT + 1, 0, st);
    k_keep<<<grid_of(NT), 256, 0, st>>>(NT, T->rlen.p, traj_min_len, T->keep.p, T->klen.p);
    PSFM_LAUNCH_CHECK();
    T->scan_flags(T->keep.p, T->kpos.p, NT);
    T->scan(T->klen.p, T->off.p, NT);
    k_emit_ids<<<grid_of(NT), 256, 0, st>>>(NT, T->keep.p, T->kpos.p, T->off.p, T->klen.p, T->ids.p, T->ptr.p, T->totals.p);
    PSFM_LAUNCH_CHECK();
    PSFM_CUDA(cudaMemcpyAsync(T->h_totals, T->totals.p, 2 * sizeof(long long), cudaMemcpyDeviceToHost, st));
    T->sync();
    T->res_trajs = T->h_totals[0];
    T->res_obs = T->h_totals[1];
    grow(T->res_frames, (size_t)T->res_obs, 0, st);
    grow(T->res_xy, 2 * (size_t)T->res_obs, 0, st);
    for (int s = 0; s <= t; ++s) {
      const int n = T->hcnt[s];
      if (!n) continue;
      k_emit_obs<<<grid_of(n), 256, 0, st>>>(n, s, T->hid.p + T->hoff[s], T->hxy.p + 2 * T->hoff[s], T->rank.p, T->keep.p, T->off.p,
                                             T->rstart.p, T->res_frames.p, T->res_xy.p);
      PSFM_LAUNCH_CHECK();
    }
    T->sync();
    *num_trajs = T->res_trajs;
    *num_obs = T->res_obs;
    return PSFM_OK;
  }, [&](int code) { return tracker_broken(T, code); });
}

extern "C" int psfm_tracker_result(psfm_tracker* T, int64_t* ids, int64_t* ptr, int32_t* frame_ids, double* xy) {
  return guard("psfm_tracker_result", [&]() -> int {
    int rc = tracker_usable(T, ids && ptr && frame_ids && xy, "psfm_tracker_result");
    if (rc != PSFM_OK) return rc;
    if (!T->finished) return fail("psfm_tracker_result", PSFM_ERR_INVALID, "call psfm_tracker_finish first");
    const size_t nt = T->res_trajs, m = T->res_obs;
    if (T->next_id == 0) { ptr[0] = 0; return PSFM_OK; }
    PSFM_CUDA(cudaMemcpyAsync(ids, T->ids.p, nt * sizeof(int64_t), cudaMemcpyDeviceToHost, T->st));
    PSFM_CUDA(cudaMemcpyAsync(ptr, T->ptr.p, (nt + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, T->st));
    PSFM_CUDA(cudaMemcpyAsync(frame_ids, T->res_frames.p, m * sizeof(int32_t), cudaMemcpyDeviceToHost, T->st));
    PSFM_CUDA(cudaMemcpyAsync(xy, T->res_xy.p, 2 * m * sizeof(double), cudaMemcpyDeviceToHost, T->st));
    T->sync();
    return PSFM_OK;
  }, [&](int code) { return tracker_broken(T, code); });
}

extern "C" int psfm_tracker_track_npy(psfm_tracker* T, psfm_track_npy** out, int64_t* nbytes) {
  return guard("psfm_tracker_track_npy", [&]() -> int {
    int rc = tracker_usable(T, out && nbytes, "psfm_tracker_track_npy");
    if (rc != PSFM_OK) return rc;
    *out = nullptr;
    *nbytes = 0;
    if (!T->finished) return fail("psfm_tracker_track_npy", PSFM_ERR_INVALID, "call psfm_tracker_finish first");
    // the tracker's ids are retire ranks (< 2^31, int counters), its frame ids times, its ptr an exclusive scan
    track_npy_encode(T->ids.p, T->ptr.p, T->res_frames.p, T->res_xy.p, T->res_trajs, T->st, out, nbytes);
    return PSFM_OK;
  }, [&](int code) { return tracker_broken(T, code); });
}

namespace {

__global__ void k_widen(long long n, const int* in, long long* out) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n) out[i] = in[i];
}

}  // namespace

extern "C" int psfm_tracker_matches(psfm_tracker* T, int32_t num_images, int32_t sample_k, psfm_matches** out,
                                    int64_t* num_pairs, int64_t* num_matches) {
  const char* entry = "psfm_tracker_matches";
  return guard(entry, [&]() -> int {
    int rc = tracker_usable(T, out && num_pairs && num_matches, entry);
    if (rc != PSFM_OK) return rc;
    *out = nullptr;
    if (!T->finished) return fail(entry, PSFM_ERR_INVALID, "call psfm_tracker_finish first");
    if (num_images < T->num_frames) return fail(entry, PSFM_ERR_INVALID, "num_images is below the tracker's number of frames");
    if (sample_k < 1) return fail(entry, PSFM_ERR_INVALID, "sample_k must be >= 1");
    if (T->res_obs > 0x7fffffffLL) return fail(entry, PSFM_ERR_INVALID, "more than 2^31 - 1 samples");
    // the tracker's ptr and xy are read where they are; its int32 frame ids are widened to the build's int64
    psfm::DBuf<long long> frames;
    psfm::TrackSetDev in;
    in.num_trajs = T->res_trajs;
    in.num_obs = T->res_obs;
    if (T->res_obs > 0) {
      frames.alloc((size_t)T->res_obs);
      k_widen<<<grid_of(T->res_obs), 256, 0, T->st>>>(T->res_obs, T->res_frames.p, frames.p);
      PSFM_LAUNCH_CHECK();
      in.tptr = T->ptr.p; in.frames = frames.p; in.xy = T->res_xy.p;
      in.own_frames = &frames;
    }
    rc = psfm::matches_build(entry, in, num_images, sample_k, T->st, out, num_pairs, num_matches);
    return rc == PSFM_OK ? rc : tracker_broken(T, rc);
  }, [&](int code) { return tracker_broken(T, code); });
}

extern "C" void psfm_tracker_destroy(psfm_tracker* T) {
  if (!T) return;
  cudaStreamSynchronize(T->st);
  if (T->h_counts) cudaFreeHost(T->h_counts);
  if (T->h_totals) cudaFreeHost(T->h_totals);
  delete T;
  cudaGetLastError();
}
