// convert.cu — the reconstructed model -> per-image sparse depth maps and their display images (DESIGN.md §4.10).
//
// What sfm/convert.py's save_depth_pose computes per registered image, for the keypoints that have a 3D point:
//   z      = (R X + t)_z, R = qvec2rotmat(qvec) as the reference writes it, qvec not renormalised
//   pixel  = (rint(x), rint(y)) as int32 (out of range or NaN: INT_MIN, what numpy's cast gives on x86-64), clipped
//            to [0, w - 1] x [0, h - 1]
//   depth  = 0 everywhere, then z at every pixel; the last keypoint in keypoint order wins a shared pixel
//   display: valid = depth > 0, v = 1 / (depth + 1), z1 / z2 = numpy's linear percentile 98 / 2 of v[valid],
//            n = clip((v - z2) / (z1 - z2), 0, 1), grey = lut[min(int(float(n) * 256), 255)], NaN: 0; RGBA8 with
//            alpha 255
// The file is compiled with -fmad=false and every product is written out, so the oracle's numpy restatement
// (oracle/convert_oracle.py) reproduces z, v and the percentiles bit for bit:
//   R20 = (2 q3) q1 - (2 q0) q2,  R21 = (2 q2) q3 + (2 q0) q1,  R22 = (1 - 2 (q1 q1)) - 2 (q2 q2)
//   z   = ((R20 X + R21 Y) + R22 Z) + t2
//
// Kernels, per batch of images (grid.y = image of the batch, grid-stride over its keypoints or pixels):
//   k_claim     per keypoint with a point: z and pixel, atomicMax of its batch-local index into the int32 winner map
//   k_winners   per keypoint that won its pixel: depth[pixel] = z; when z > 0, v into the image's segment and a count
//   segmented sort of the valid v (CUB), one segment per image
//   k_percent   per image: the two order statistics at each virtual index and numpy's _lerp
//   k_colour    per pixel: v, n, the LUT and RGBA8
// psfm_convert_create runs the first two kernels without the depth map to count each image's valid pixels, so a
// caller can refuse an image with none before anything is written.  psfm_convert_result runs all five, batch b on
// stream b % 2, and copies the batch's maps to pinned buffers there; the host moves batch b - 1 out of its pinned
// buffers while the device runs batch b.
#include <cub/device/device_segmented_sort.cuh>

#include <algorithm>
#include <chrono>
#include <climits>
#include <vector>

#include "pair_inputs.h"
#include "psfm_common.cuh"

namespace {

using namespace psfm;

// device bytes of one batch slot: winner (4) + depth (8) + RGBA (4) per pixel; z, pixel, v and sorted v per keypoint
constexpr long long kBytesPerPixel = 16, kBytesPerKeypoint = 32;
// images of one batch: grid.y of its launches
constexpr int kMaxBatchImages = 65535;

struct Batch {
  int first, count;                 // images [first, first + count)
  long long kp0, num_kp, num_px;    // keypoints [kp0, kp0 + num_kp), pixels of the batch
};

__device__ __forceinline__ int to_pixel(double x, int size) {
  const double r = rint(x);
  int p = (r >= -2147483648.0 && r < 2147483648.0) ? (int)r : INT_MIN;
  return p < 0 ? 0 : (p > size - 1 ? size - 1 : p);
}

// z of keypoint k (global index) of image i and its pixel inside the image
__device__ __forceinline__ double project(const double* q, const double* t, const double* xyz, int row, double2 xy,
                                          int w, int h, long long* pix) {
  const double q0 = q[0], q1 = q[1], q2 = q[2], q3 = q[3];
  const double r20 = __dsub_rn(__dmul_rn(__dmul_rn(2.0, q3), q1), __dmul_rn(__dmul_rn(2.0, q0), q2));
  const double r21 = __dadd_rn(__dmul_rn(__dmul_rn(2.0, q2), q3), __dmul_rn(__dmul_rn(2.0, q0), q1));
  const double r22 = __dsub_rn(__dsub_rn(1.0, __dmul_rn(2.0, __dmul_rn(q1, q1))), __dmul_rn(2.0, __dmul_rn(q2, q2)));
  const double* X = xyz + 3 * (long long)row;
  const double z = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(r20, X[0]), __dmul_rn(r21, X[1])), __dmul_rn(r22, X[2])), t[2]);
  *pix = (long long)to_pixel(xy.y, h) * w + to_pixel(xy.x, w);
  return z;
}

struct Model {
  const double* qvec;        // [F][4]
  const double* tvec;        // [F][3]
  const int* size;           // [F][2] width, height of each image's camera
  const long long* kptr;     // [F + 1]
  const double2* xy;         // [K]
  const int* row;            // [K]
  const double* xyz;         // [P][3]
};

// grid.y: image first + blockIdx.y; zbuf / pbuf / winner are batch-local (keypoint kp0, pixel offset pix_off[image])
__global__ void k_claim(Model m, int first, long long kp0, const long long* pix_off, double* zbuf, long long* pbuf,
                        int* winner) {
  const int i = first + blockIdx.y;
  const long long a = m.kptr[i], b = m.kptr[i + 1], base = pix_off[blockIdx.y];
  const int w = m.size[2 * i], h = m.size[2 * i + 1];
  for (long long k = a + blockIdx.x * (long long)blockDim.x + threadIdx.x; k < b; k += (long long)gridDim.x * blockDim.x) {
    const int row = m.row[k];
    if (row < 0) continue;
    long long pix;
    const double z = project(m.qvec + 4 * i, m.tvec + 3 * i, m.xyz, row, m.xy[k], w, h, &pix);
    zbuf[k - kp0] = z;
    pbuf[k - kp0] = base + pix;
    atomicMax(winner + base + pix, (int)(k - kp0));
  }
}

// depth (nullable: counting only) and the valid v of every image in its keypoint segment [kptr[i] - kp0, ..)
__global__ void k_winners(Model m, int first, long long kp0, const double* zbuf, const long long* pbuf, const int* winner,
                          double* depth, double* vbuf, int* count) {
  const int i = first + blockIdx.y;
  const long long a = m.kptr[i], b = m.kptr[i + 1];
  for (long long k = a + blockIdx.x * (long long)blockDim.x + threadIdx.x; k < b; k += (long long)gridDim.x * blockDim.x) {
    if (m.row[k] < 0) continue;
    const long long pix = pbuf[k - kp0];
    if (winner[pix] != (int)(k - kp0)) continue;
    const double z = zbuf[k - kp0];
    if (depth) depth[pix] = z;
    if (z > 0.0) {
      const int s = atomicAdd(count + blockIdx.y, 1);
      if (vbuf) vbuf[a - kp0 + s] = __ddiv_rn(1.0, __dadd_rn(z, 1.0));
    }
  }
}

__global__ void k_segment_end(int n, const int* begin, const int* count, int* end) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) end[i] = begin[i] + count[i];
}

// numpy's percentile, method "linear", of the n sorted values s at fraction q (np.percentile's q / 100)
__device__ __forceinline__ double percentile(const double* s, int n, double q) {
  const double vi = __dmul_rn((double)(n - 1), q);
  if (vi >= (double)(n - 1)) return s[n - 1];
  const double lo = floor(vi), g = __dsub_rn(vi, lo);
  const double a = s[(long long)lo], b = s[(long long)lo + 1], d = __dsub_rn(b, a);
  return g >= 0.5 ? __dsub_rn(b, __dmul_rn(d, __dsub_rn(1.0, g))) : __dadd_rn(a, __dmul_rn(d, g));
}

__global__ void k_percent(int n, const int* begin, const int* count, const double* sorted, double* z12) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double* s = sorted + begin[i];
  z12[2 * i] = percentile(s, count[i], 98.0 / 100.0);
  z12[2 * i + 1] = percentile(s, count[i], 2.0 / 100.0);
}

__global__ void k_colour(const long long* pix_off, const int* size, const double* z12, const double* depth,
                         const unsigned char* lut, uchar4* rgba) {
  __shared__ unsigned char s_lut[256];
  for (int j = threadIdx.x; j < 256; j += blockDim.x) s_lut[j] = lut[j];
  __syncthreads();
  const int i = blockIdx.y;
  const long long a = pix_off[i], b = a + (long long)size[2 * i] * size[2 * i + 1];
  const double z1 = z12[2 * i], z2 = z12[2 * i + 1], den = __dsub_rn(z1, z2);
  for (long long p = a + blockIdx.x * (long long)blockDim.x + threadIdx.x; p < b; p += (long long)gridDim.x * blockDim.x) {
    const double v = __ddiv_rn(1.0, __dadd_rn(depth[p], 1.0));
    double n = __ddiv_rn(__dsub_rn(v, z2), den);
    n = n < 0.0 ? 0.0 : (n > 1.0 ? 1.0 : n);           // NaN stays NaN, as np.clip leaves it
    unsigned char c = 0;                                 // the colormap's "bad" colour: black
    if (n == n) {
      const float x = __fmul_rn(__double2float_rn(n), 256.0f);
      c = s_lut[x >= 256.0f ? 255 : (int)x];
    }
    rgba[p] = make_uchar4(c, c, c, 255);
  }
}

// the device buffers of one batch slot, sized for the largest batch
struct Slot {
  cudaStream_t st = nullptr;
  DBuf<int> winner, count, end;
  DBuf<double> depth, zbuf, vbuf, vsort, z12;
  DBuf<long long> pbuf;
  DBuf<unsigned char> rgba, lut, tmp;
  size_t tmp_bytes = 0;
  double* h_depth = nullptr;                        // pinned
  unsigned char* h_rgba = nullptr;
  cudaEvent_t ev[4] = {};
  ~Slot() {
    if (h_depth) cudaFreeHost(h_depth);
    if (h_rgba) cudaFreeHost(h_rgba);
    for (cudaEvent_t e : ev)
      if (e) cudaEventDestroy(e);
    if (st) cudaStreamDestroy(st);
  }
};

double host_ms_since(std::chrono::steady_clock::time_point t0) {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

inline unsigned blocks_for(long long n) { return (unsigned)std::max<long long>(1, std::min<long long>((n + 255) / 256, 64)); }

}  // namespace

struct psfm_convert {
  int F = 0;
  long long K = 0;
  std::vector<long long> kptr;                      // [F + 1]
  std::vector<long long> num_px;                    // [F] pixels of each image
  std::vector<Batch> batches;
  std::vector<long long> valid;                     // [F]
  DBuf<double> qvec, tvec, xy, xyz;
  DBuf<int> size, row;
  DBuf<long long> kptr_d, pix_off_d;                // pix_off_d [F]: each image's first pixel inside its batch
  DBuf<int> seg_begin_d;                            // [F]: each image's first keypoint inside its batch (sort segment)
  unsigned char lut[256];
  Slot slots[2];                                    // psfm_convert_result's, allocated by its first call
  bool slots_ready = false;
  Model model() const {
    return Model{qvec.p, tvec.p, size.p, kptr_d.p, reinterpret_cast<const double2*>(xy.p), row.p, xyz.p};
  }
};

namespace {

// claim + winners of batch b on slot s; depth / vbuf nullable (the counting pass)
void run_claims(const psfm_convert* H, const Batch& b, Slot& s, bool full) {
  long long max_kp = 0;
  for (int i = b.first; i < b.first + b.count; ++i) max_kp = std::max(max_kp, H->kptr[i + 1] - H->kptr[i]);
  PSFM_CUDA(cudaMemsetAsync(s.winner.p, 0xff, sizeof(int) * (size_t)b.num_px, s.st));
  PSFM_CUDA(cudaMemsetAsync(s.count.p, 0, sizeof(int) * (size_t)b.count, s.st));
  if (full) PSFM_CUDA(cudaMemsetAsync(s.depth.p, 0, sizeof(double) * (size_t)b.num_px, s.st));
  const dim3 grid(blocks_for(max_kp), b.count);
  const long long* off = H->pix_off_d.p + b.first;
  k_claim<<<grid, 256, 0, s.st>>>(H->model(), b.first, b.kp0, off, s.zbuf.p, s.pbuf.p, s.winner.p);
  PSFM_LAUNCH_CHECK();
  k_winners<<<grid, 256, 0, s.st>>>(H->model(), b.first, b.kp0, s.zbuf.p, s.pbuf.p, s.winner.p, full ? s.depth.p : nullptr,
                                    full ? s.vbuf.p : nullptr, s.count.p);
  PSFM_LAUNCH_CHECK();
}

void alloc_slot(const psfm_convert* H, Slot& s, bool full) {
  long long px = 0, kp = 0;
  int imgs = 0;
  for (const Batch& b : H->batches) {
    px = std::max(px, b.num_px);
    kp = std::max(kp, b.num_kp);
    imgs = std::max(imgs, b.count);
  }
  PSFM_CUDA(cudaStreamCreateWithFlags(&s.st, cudaStreamNonBlocking));
  s.winner.alloc(px); s.count.alloc(imgs); s.zbuf.alloc(kp); s.pbuf.alloc(kp);
  if (!full) return;
  s.depth.alloc(px); s.rgba.alloc(4 * (size_t)px); s.vbuf.alloc(kp); s.vsort.alloc(kp);
  s.end.alloc(imgs); s.z12.alloc(2 * (size_t)imgs); s.lut.alloc(256);
  PSFM_CUDA(cudaMemcpy(s.lut.p, H->lut, 256, cudaMemcpyHostToDevice));
  PSFM_CUDA(cub::DeviceSegmentedSort::SortKeys(nullptr, s.tmp_bytes, s.vbuf.p, s.vsort.p, (int)std::max(kp, 1LL), imgs,
                                               H->seg_begin_d.p, s.end.p, s.st));
  s.tmp.alloc(s.tmp_bytes);
  PSFM_CUDA(cudaMallocHost((void**)&s.h_depth, sizeof(double) * (size_t)std::max(px, 1LL)));
  PSFM_CUDA(cudaMallocHost((void**)&s.h_rgba, 4 * (size_t)std::max(px, 1LL)));
  for (cudaEvent_t& e : s.ev) PSFM_CUDA(cudaEventCreate(&e));
}

float elapsed(cudaEvent_t a, cudaEvent_t b) {
  float ms = 0.f;
  PSFM_CUDA(cudaEventElapsedTime(&ms, a, b));
  return ms;
}

}  // namespace

extern "C" int psfm_convert_create(int32_t num_cameras, const int32_t* camera_size, int32_t num_images, const double* qvec,
                                   const double* tvec, const int32_t* image_camera, const int64_t* keypoint_ptr,
                                   const double* keypoints, const int32_t* point_row, int64_t num_points,
                                   const double* xyz, const uint8_t* gray_lut, int64_t memory_budget, psfm_convert** out,
                                   int64_t* valid_count, int32_t* batch_ptr, psfm_convert_summary* summary) {
  const char* entry = "psfm_convert_create";
  return guard(entry, [&]() -> int {
    if (!out || !camera_size || !image_camera || !keypoint_ptr || !gray_lut || !valid_count || !batch_ptr ||
        (num_images > 0 && (!qvec || !tvec)))
      return fail(entry, PSFM_ERR_INVALID, "null argument");
    *out = nullptr;
    if (num_cameras < 0 || num_images < 0 || num_points < 0 || memory_budget <= 0)
      return fail(entry, PSFM_ERR_INVALID, "num_cameras, num_images, num_points must be >= 0 and memory_budget > 0");
    for (int c = 0; c < num_cameras; ++c)
      if (camera_size[2 * c] <= 0 || camera_size[2 * c + 1] <= 0 ||
          (long long)camera_size[2 * c] * camera_size[2 * c + 1] > 0x7fffffffLL)
        return fail(entry, PSFM_ERR_INVALID, "camera " + std::to_string(c) + " has a bad size (camera size)");
    int rc = check_keypoint_ptr(entry, num_images, keypoint_ptr);
    if (rc != PSFM_OK) return rc;
    for (int i = 0; i < num_images; ++i)
      if (image_camera[i] < 0 || image_camera[i] >= num_cameras)
        return fail(entry, PSFM_ERR_INVALID, "image " + std::to_string(i) + " has a camera index out of range (camera index)");
    const long long K = keypoint_ptr[num_images];
    if (K > 0x7fffffffLL) return fail(entry, PSFM_ERR_INVALID, "more than 2^31 - 1 keypoints");
    if (K > 0 && (!keypoints || !point_row)) return fail(entry, PSFM_ERR_INVALID, "null argument");
    if (num_points > 0 && !xyz) return fail(entry, PSFM_ERR_INVALID, "null argument");
    for (long long k = 0; k < K; ++k)
      if (point_row[k] < -1 || point_row[k] >= num_points)
        return fail(entry, PSFM_ERR_INVALID, "keypoint " + std::to_string(k) + " has a point row out of range (point row)");
    if ((rc = require_device(entry)) != PSFM_OK) return rc;
    std::unique_ptr<psfm_convert> H(new psfm_convert);
    H->F = num_images;
    H->K = K;
    std::copy(gray_lut, gray_lut + 256, H->lut);
    H->kptr.assign(keypoint_ptr, keypoint_ptr + num_images + 1);
    H->valid.assign(num_images, 0);
    // batches: images in order while both slots' buffers stay inside the budget, at least one image per batch
    std::vector<int> sz(2 * (size_t)num_images);
    std::vector<long long> local_off(num_images, 0);
    std::vector<int> seg_begin(num_images, 0);
    H->num_px.assign(num_images, 0);
    for (int i = 0; i < num_images; ++i) {
      sz[2 * i] = camera_size[2 * image_camera[i]];
      sz[2 * i + 1] = camera_size[2 * image_camera[i] + 1];
      H->num_px[i] = (long long)sz[2 * i] * sz[2 * i + 1];
    }
    for (int i = 0; i < num_images;) {
      Batch b{i, 0, H->kptr[i], 0, 0};
      while (i < num_images) {
        const long long px = H->num_px[i], kp = H->kptr[i + 1] - H->kptr[i];
        if (b.count > 0 && (b.count == kMaxBatchImages ||
                            2 * (kBytesPerPixel * (b.num_px + px) + kBytesPerKeypoint * (b.num_kp + kp)) > memory_budget))
          break;
        local_off[i] = b.num_px;
        seg_begin[i] = (int)b.num_kp;
        b.num_px += px;
        b.num_kp += kp;
        ++b.count;
        ++i;
      }
      H->batches.push_back(b);
    }
    Event e0, e1, e2, e3;
    Slot s;
    const auto t_alloc = std::chrono::steady_clock::now();
    H->qvec.alloc(4 * (size_t)num_images); H->tvec.alloc(3 * (size_t)num_images); H->size.alloc(2 * (size_t)num_images);
    H->kptr_d.alloc(num_images + 1); H->pix_off_d.alloc(num_images); H->seg_begin_d.alloc(num_images);
    H->xy.alloc(2 * (size_t)K); H->row.alloc(K); H->xyz.alloc(3 * (size_t)num_points);
    double alloc_ms = host_ms_since(t_alloc);
    PSFM_CUDA(cudaEventRecord(e0.e, 0));
    H->qvec.upload(qvec, H->qvec.n, nullptr); H->tvec.upload(tvec, H->tvec.n, nullptr); H->size.upload(sz.data(), sz.size(), nullptr);
    H->kptr_d.upload(reinterpret_cast<const long long*>(keypoint_ptr), num_images + 1, nullptr);
    H->pix_off_d.upload(local_off.data(), num_images, nullptr);
    H->seg_begin_d.upload(seg_begin.data(), num_images, nullptr);
    H->xy.upload(keypoints, 2 * (size_t)K, nullptr); H->row.upload(point_row, K, nullptr);
    H->xyz.upload(xyz, 3 * (size_t)num_points, nullptr);
    PSFM_CUDA(cudaEventRecord(e1.e, 0));
    PSFM_CUDA(cudaDeviceSynchronize());
    const auto t_slot = std::chrono::steady_clock::now();
    alloc_slot(H.get(), s, false);
    alloc_ms += host_ms_since(t_slot);
    PSFM_CUDA(cudaEventRecord(e2.e, s.st));
    // the counting pass: the valid pixels of every image, before anything is written
    std::vector<int> cnt;
    for (const Batch& b : H->batches) {
      run_claims(H.get(), b, s, false);
      cnt.resize(b.count);
      PSFM_CUDA(cudaMemcpyAsync(cnt.data(), s.count.p, sizeof(int) * (size_t)b.count, cudaMemcpyDeviceToHost, s.st));
      PSFM_CUDA(cudaStreamSynchronize(s.st));
      for (int j = 0; j < b.count; ++j) H->valid[b.first + j] = cnt[j];
    }
    PSFM_CUDA(cudaEventRecord(e3.e, s.st));
    PSFM_CUDA(cudaEventSynchronize(e3.e));
    if (summary) {
      summary->num_batches = (int32_t)H->batches.size();
      summary->upload_ms = elapsed(e0.e, e1.e);
      summary->kernel_ms = elapsed(e2.e, e3.e);
      summary->d2h_ms = 0.0;
      summary->alloc_ms = alloc_ms;
      summary->host_copy_ms = 0.0;
    }
    std::copy(H->valid.begin(), H->valid.end(), valid_count);
    for (size_t j = 0; j < H->batches.size(); ++j) batch_ptr[j] = H->batches[j].first;
    batch_ptr[H->batches.size()] = num_images;
    *out = H.release();
    return PSFM_OK;
  });
}

extern "C" int psfm_convert_result(psfm_convert* H, int32_t first_batch, int32_t num_batches, double* depth,
                                   uint8_t* rgba, psfm_convert_summary* summary) {
  const char* entry = "psfm_convert_result";
  return guard(entry, [&]() -> int {
    if (!H) return fail(entry, PSFM_ERR_INVALID, "null argument");
    const int nb = (int)H->batches.size();
    if (first_batch < 0 || num_batches < 0 || first_batch > nb || num_batches > nb - first_batch)
      return fail(entry, PSFM_ERR_INVALID, "batches out of range");
    if (num_batches > 0 && (!depth || !rgba)) return fail(entry, PSFM_ERR_INVALID, "null argument");
    const int j0 = first_batch, j1 = first_batch + num_batches;
    for (int j = j0; j < j1; ++j)
      for (int i = H->batches[j].first; i < H->batches[j].first + H->batches[j].count; ++i)
        if (H->valid[i] == 0)
          return fail(entry, PSFM_ERR_INVALID, "image " + std::to_string(i) + " has no valid pixel (no percentile)");
    Slot* slots = H->slots;
    const auto t_alloc = std::chrono::steady_clock::now();
    if (!H->slots_ready && nb > 0) {
      alloc_slot(H, slots[0], true);
      if (nb > 1) alloc_slot(H, slots[1], true);
      H->slots_ready = true;
    }
    const double alloc_ms = host_ms_since(t_alloc);
    // pixel offset of every batch's first image in the caller's buffers
    std::vector<long long> out_off(nb + 1, 0);
    for (int j = j0; j < j1; ++j) out_off[j + 1] = out_off[j] + H->batches[j].num_px;
    double kernel_ms = 0.0, d2h_ms = 0.0, host_copy_ms = 0.0;
    auto drain = [&](int j) {             // batch j's maps from its pinned buffers to the caller's
      Slot& s = slots[j % 2];
      PSFM_CUDA(cudaStreamSynchronize(s.st));
      const Batch& b = H->batches[j];
      const auto t0 = std::chrono::steady_clock::now();
      std::copy(s.h_depth, s.h_depth + b.num_px, depth + out_off[j]);
      std::copy(s.h_rgba, s.h_rgba + 4 * b.num_px, rgba + 4 * out_off[j]);
      host_copy_ms += host_ms_since(t0);
      kernel_ms += elapsed(s.ev[0], s.ev[1]);
      d2h_ms += elapsed(s.ev[1], s.ev[2]);
    };
    for (int j = j0; j < j1; ++j) {
      const Batch& b = H->batches[j];
      Slot& s = slots[j % 2];
      PSFM_CUDA(cudaEventRecord(s.ev[0], s.st));
      run_claims(H, b, s, true);
      // segment of image first + y: its keypoints, [kptr[i] - kp0, kptr[i + 1] - kp0), the valid ones first
      const int* begin = H->seg_begin_d.p + b.first;
      k_segment_end<<<(b.count + 255) / 256, 256, 0, s.st>>>(b.count, begin, s.count.p, s.end.p);
      PSFM_LAUNCH_CHECK();
      size_t bytes = s.tmp_bytes;
      PSFM_CUDA(cub::DeviceSegmentedSort::SortKeys(s.tmp.p, bytes, s.vbuf.p, s.vsort.p, (int)b.num_kp, b.count, begin,
                                                   s.end.p, s.st));
      PSFM_LAUNCH_CHECK();
      k_percent<<<(b.count + 255) / 256, 256, 0, s.st>>>(b.count, begin, s.count.p, s.vsort.p, s.z12.p);
      PSFM_LAUNCH_CHECK();
      long long max_px = 0;
      for (int i = b.first; i < b.first + b.count; ++i) max_px = std::max(max_px, H->num_px[i]);
      k_colour<<<dim3(blocks_for(max_px), b.count), 256, 0, s.st>>>(H->pix_off_d.p + b.first, H->size.p + 2 * b.first, s.z12.p,
                                                                    s.depth.p, s.lut.p, reinterpret_cast<uchar4*>(s.rgba.p));
      PSFM_LAUNCH_CHECK();
      PSFM_CUDA(cudaEventRecord(s.ev[1], s.st));
      PSFM_CUDA(cudaMemcpyAsync(s.h_depth, s.depth.p, sizeof(double) * (size_t)b.num_px, cudaMemcpyDeviceToHost, s.st));
      PSFM_CUDA(cudaMemcpyAsync(s.h_rgba, s.rgba.p, 4 * (size_t)b.num_px, cudaMemcpyDeviceToHost, s.st));
      PSFM_CUDA(cudaEventRecord(s.ev[2], s.st));
      if (j > j0) drain(j - 1);          // batch j - 1's copy overlapped batch j's kernels
    }
    if (j1 > j0) drain(j1 - 1);
    if (summary) {
      summary->num_batches = num_batches;
      summary->upload_ms = 0.0;
      summary->kernel_ms = kernel_ms;
      summary->d2h_ms = d2h_ms;
      summary->alloc_ms = alloc_ms;
      summary->host_copy_ms = host_copy_ms;
    }
    return PSFM_OK;
  });
}

extern "C" void psfm_convert_destroy(psfm_convert* H) {
  delete H;
  cudaGetLastError();
}
