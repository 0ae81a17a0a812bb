// colors.cu — the colour of every 3D point from the images that observe it (DESIGN.md §4.11).
//
// What Reconstruction::ExtractColorsForAllImages (reference base/reconstruction.cc:1250-1300) computes: for every
// observation (a keypoint with a point) of every image that could be read, Bitmap::InterpolateBilinear at
// (X - 0.5, Y - 0.5) (csrc/colors_recalled.cuh); per point the mean of the samples in double, rounded half away from
// zero to uint8, or black when the point has none.  The reference sums in the order of reg_image_ids_, which is not
// defined; here it is fixed: ascending image index, then keypoint index.  No floating-point atomic is used, so two
// runs give the same bytes.  Compiled with -fmad=false, so the interpolation is the oracle's (oracle/colors_oracle.py).
//
//   psfm_colors_create       the observations, compacted in keypoint order (image-major), and a stable radix sort of
//                            them by point row: each point's list in that order (k_point_ptr gives its segment)
//   psfm_colors_add_images   one batch of decoded images: copied into the slot's pinned buffer, uploaded, and k_sample
//                            (one thread per observation of the batch's images) writes a float4 (r, g, b, 1) per
//                            observation, or (0, 0, 0, 0) when the interpolation declines.  Batch b runs on stream
//                            b % 2, so its upload overlaps the previous batch's kernel.  Images never added keep the
//                            (0, 0, 0, 0) of the create call: they contribute nothing.
//   psfm_colors_result       k_mean, one thread per point over its sorted list, and the [P][3] bytes
#include <chrono>
#include <climits>
#include <vector>

#include "colors_recalled.cuh"
#include "pair_inputs.h"
#include "psfm_common.cuh"
#include "radix_sort.cuh"

namespace {

using namespace psfm;

struct ImageMeta {
  long long offset;   // first byte of the image in its batch
  int w, h;
};

__global__ void k_point_ptr(int n, const int* key, long long num_points, int* ptr) {
  const long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (j > n) return;
  const long long prev = j == 0 ? -1 : key[j - 1], cur = j < n ? key[j] : num_points;
  for (long long p = prev + 1; p <= cur; ++p) ptr[p] = (int)j;
}

// observations [o0, o1) belong to the images first .. first + count - 1 of the batch
__global__ void k_sample(long long o0, long long o1, const int* obs_image, const double2* obs_xy, int first,
                         const ImageMeta* meta, const unsigned char* px, float4* colour) {
  for (long long o = o0 + blockIdx.x * (long long)blockDim.x + threadIdx.x; o < o1; o += (long long)gridDim.x * blockDim.x) {
    const ImageMeta m = meta[obs_image[o] - first];
    const double2 xy = obs_xy[o];
    float c[3];
    colour[o] = colors::interpolate_bilinear(px + m.offset, m.w, m.h, xy.x - colors::kPixelCentre,
                                             xy.y - colors::kPixelCentre, c)
                    ? make_float4(c[0], c[1], c[2], 1.0f)
                    : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  }
}

// point p's samples in list order: ascending image, then keypoint
__global__ void k_mean(long long num_points, const int* ptr, const int* order, const float4* colour, unsigned char* rgb) {
  const long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (p >= num_points) return;
  double r = 0.0, g = 0.0, b = 0.0;
  long long n = 0;
  for (int j = ptr[p]; j < ptr[p + 1]; ++j) {
    const float4 c = colour[order[j]];
    if (c.w == 0.0f) continue;
    r += (double)c.x;
    g += (double)c.y;
    b += (double)c.z;
    ++n;
  }
  unsigned char* out = rgb + 3 * p;
  if (n == 0) {
    out[0] = out[1] = out[2] = 0;
    return;
  }
  const double d = (double)n;
  out[0] = (unsigned char)round(r / d);     // round: half away from zero, as std::round
  out[1] = (unsigned char)round(g / d);
  out[2] = (unsigned char)round(b / d);
}

// the buffers of one batch slot, grown to the largest batch it has taken
struct Slot {
  cudaStream_t st = nullptr;
  DBuf<unsigned char> px;
  DBuf<ImageMeta> meta;
  unsigned char* h_px = nullptr;          // pinned
  ImageMeta* h_meta = nullptr;
  size_t px_cap = 0, meta_cap = 0;
  cudaEvent_t ev[3] = {};                 // before the upload, after it, after k_sample
  bool pending = false;                   // a batch's events are not yet counted
  ~Slot() {
    if (h_px) cudaFreeHost(h_px);
    if (h_meta) cudaFreeHost(h_meta);
    for (cudaEvent_t e : ev)
      if (e) cudaEventDestroy(e);
    if (st) cudaStreamDestroy(st);
  }
};

double host_ms_since(std::chrono::steady_clock::time_point t0) {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

float elapsed(cudaEvent_t a, cudaEvent_t b) {
  float ms = 0.f;
  PSFM_CUDA(cudaEventElapsedTime(&ms, a, b));
  return ms;
}

}  // namespace

struct psfm_colors {
  int F = 0;
  long long P = 0, N = 0;                 // points, observations
  std::vector<long long> obs_ptr;         // [F + 1] each image's observations
  std::vector<char> added;                // [F]
  DBuf<int> obs_image, keys, vals, ptr;   // keys / vals: both halves of the sort's double buffers
  DBuf<double> obs_xy;
  DBuf<float4> colour;
  DBuf<unsigned char> rgb;
  const int* order = nullptr;             // the sorted observation indices (one half of vals)
  Slot slots[2];
  int num_batches = 0, num_images = 0;
  double setup_ms = 0.0, upload_ms = 0.0, sample_ms = 0.0, stage_ms = 0.0;
};

namespace {

// the times of the slot's last batch, once its stream has finished
void count_batch(psfm_colors* H, Slot& s) {
  if (!s.pending) return;
  H->upload_ms += elapsed(s.ev[0], s.ev[1]);
  H->sample_ms += elapsed(s.ev[1], s.ev[2]);
  s.pending = false;
}

}  // namespace

extern "C" int psfm_colors_create(int32_t num_images, const int64_t* keypoint_ptr, const double* keypoints,
                                  const int32_t* point_of_keypoint, int64_t num_points, psfm_colors** out,
                                  psfm_colors_summary* summary) {
  const char* entry = "psfm_colors_create";
  return guard(entry, [&]() -> int {
    if (!out || !keypoint_ptr) return fail(entry, PSFM_ERR_INVALID, "null argument");
    *out = nullptr;
    if (num_images < 0 || num_points < 0 || num_points > INT_MAX)
      return fail(entry, PSFM_ERR_INVALID, "num_images must be >= 0 and num_points in [0, 2^31 - 1]");
    int rc = check_keypoint_ptr(entry, num_images, keypoint_ptr);
    if (rc != PSFM_OK) return rc;
    const long long K = keypoint_ptr[num_images];
    if (K > INT_MAX) return fail(entry, PSFM_ERR_INVALID, "more than 2^31 - 1 keypoints");
    if (K > 0 && (!keypoints || !point_of_keypoint)) return fail(entry, PSFM_ERR_INVALID, "null argument");
    for (long long k = 0; k < K; ++k)
      if (point_of_keypoint[k] < -1 || point_of_keypoint[k] >= num_points)
        return fail(entry, PSFM_ERR_INVALID, "keypoint " + std::to_string(k) + " has a point row out of range (point row)");
    if ((rc = require_device(entry)) != PSFM_OK) return rc;
    std::unique_ptr<psfm_colors> H(new psfm_colors);
    H->F = num_images;
    H->P = num_points;
    H->added.assign(num_images, 0);
    H->obs_ptr.assign(num_images + 1, 0);
    std::vector<int> image, row;
    std::vector<double> xy;
    for (int i = 0; i < num_images; ++i) {
      for (long long k = keypoint_ptr[i]; k < keypoint_ptr[i + 1]; ++k) {
        if (point_of_keypoint[k] < 0) continue;
        image.push_back(i);
        row.push_back(point_of_keypoint[k]);
        xy.push_back(keypoints[2 * k]);
        xy.push_back(keypoints[2 * k + 1]);
      }
      H->obs_ptr[i + 1] = (long long)image.size();
    }
    const long long N = H->N = (long long)image.size();
    Event e0, e1;
    PSFM_CUDA(cudaEventRecord(e0, 0));
    H->obs_image.alloc(N); H->obs_xy.alloc(2 * N); H->colour.alloc(N);
    H->keys.alloc(2 * N); H->vals.alloc(2 * N); H->ptr.alloc(num_points + 1); H->rgb.alloc(3 * num_points);
    H->obs_image.upload(image.data(), N, 0);
    H->obs_xy.upload(xy.data(), 2 * N, 0);
    H->keys.upload(row.data(), N, 0);
    H->colour.zero(0);
    std::vector<int> iota(N);
    for (long long o = 0; o < N; ++o) iota[o] = (int)o;
    H->vals.upload(iota.data(), N, 0);
    cub::DoubleBuffer<int> kb(H->keys.p, H->keys.p + N), vb(H->vals.p, H->vals.p + N);
    if (N > 0) sort_pairs(kb, vb, (int)N, key_bits(num_points > 0 ? num_points - 1 : 0));
    H->order = vb.Current();
    k_point_ptr<<<grid_of(N + 1), 256>>>((int)N, kb.Current(), num_points, H->ptr.p);
    PSFM_LAUNCH_CHECK();
    PSFM_CUDA(cudaEventRecord(e1, 0));
    PSFM_CUDA(cudaEventSynchronize(e1));
    H->setup_ms = elapsed(e0, e1);
    for (Slot& s : H->slots) {
      PSFM_CUDA(cudaStreamCreateWithFlags(&s.st, cudaStreamNonBlocking));
      for (cudaEvent_t& e : s.ev) PSFM_CUDA(cudaEventCreate(&e));
    }
    if (summary) {
      *summary = psfm_colors_summary{};
      summary->num_observations = N;
      summary->setup_ms = H->setup_ms;
    }
    *out = H.release();
    return PSFM_OK;
  });
}

extern "C" int psfm_colors_add_images(psfm_colors* H, int32_t first, int32_t count, const int32_t* width,
                                      const int32_t* height, const uint8_t* pixels) {
  const char* entry = "psfm_colors_add_images";
  return guard(entry, [&]() -> int {
    if (!H) return fail(entry, PSFM_ERR_INVALID, "null argument");
    if (count < 0 || first < 0 || first > H->F || count > H->F - first)
      return fail(entry, PSFM_ERR_INVALID, "images [first, first + count) out of range (image index)");
    if (count == 0) return PSFM_OK;
    if (!width || !height || !pixels) return fail(entry, PSFM_ERR_INVALID, "null argument");
    std::vector<ImageMeta> meta(count);
    long long bytes = 0;
    for (int j = 0; j < count; ++j) {
      if (H->added[first + j])
        return fail(entry, PSFM_ERR_INVALID, "image " + std::to_string(first + j) + " was already added (image index)");
      if (width[j] <= 0 || height[j] <= 0)
        return fail(entry, PSFM_ERR_INVALID, "image " + std::to_string(first + j) + " has a zero size (image size)");
      meta[j] = ImageMeta{bytes, width[j], height[j]};
      bytes += 3LL * width[j] * height[j];
    }
    Slot& s = H->slots[H->num_batches % 2];
    PSFM_CUDA(cudaStreamSynchronize(s.st));            // the slot's previous batch no longer reads its buffers
    count_batch(H, s);
    if ((size_t)bytes > s.px_cap) {
      if (s.h_px) PSFM_CUDA(cudaFreeHost(s.h_px));
      s.h_px = nullptr;
      s.px_cap = 0;
      PSFM_CUDA(cudaMallocHost((void**)&s.h_px, bytes));
      s.px.alloc(bytes);
      s.px_cap = bytes;
    }
    if ((size_t)count > s.meta_cap) {
      if (s.h_meta) PSFM_CUDA(cudaFreeHost(s.h_meta));
      s.h_meta = nullptr;
      s.meta_cap = 0;
      PSFM_CUDA(cudaMallocHost((void**)&s.h_meta, sizeof(ImageMeta) * count));
      s.meta.alloc(count);
      s.meta_cap = count;
    }
    const auto t0 = std::chrono::steady_clock::now();
    std::copy(pixels, pixels + bytes, s.h_px);
    std::copy(meta.begin(), meta.end(), s.h_meta);
    H->stage_ms += host_ms_since(t0);
    PSFM_CUDA(cudaEventRecord(s.ev[0], s.st));
    PSFM_CUDA(cudaMemcpyAsync(s.px.p, s.h_px, bytes, cudaMemcpyHostToDevice, s.st));
    PSFM_CUDA(cudaMemcpyAsync(s.meta.p, s.h_meta, sizeof(ImageMeta) * count, cudaMemcpyHostToDevice, s.st));
    PSFM_CUDA(cudaEventRecord(s.ev[1], s.st));
    const long long o0 = H->obs_ptr[first], o1 = H->obs_ptr[first + count];
    k_sample<<<grid_stride_of(o1 - o0), 256, 0, s.st>>>(o0, o1, H->obs_image.p, reinterpret_cast<const double2*>(H->obs_xy.p),
                                                        first, s.meta.p, s.px.p, H->colour.p);
    PSFM_LAUNCH_CHECK();
    PSFM_CUDA(cudaEventRecord(s.ev[2], s.st));
    s.pending = true;
    for (int j = 0; j < count; ++j) H->added[first + j] = 1;
    ++H->num_batches;
    H->num_images += count;
    return PSFM_OK;
  });
}

extern "C" int psfm_colors_result(psfm_colors* H, uint8_t* rgb, psfm_colors_summary* summary) {
  const char* entry = "psfm_colors_result";
  return guard(entry, [&]() -> int {
    if (!H || (H->P > 0 && !rgb)) return fail(entry, PSFM_ERR_INVALID, "null argument");
    for (Slot& s : H->slots) {
      PSFM_CUDA(cudaStreamSynchronize(s.st));
      count_batch(H, s);
    }
    Event e0, e1;
    PSFM_CUDA(cudaEventRecord(e0, 0));
    k_mean<<<grid_of(H->P), 256>>>(H->P, H->ptr.p, H->order, H->colour.p, H->rgb.p);
    PSFM_LAUNCH_CHECK();
    PSFM_CUDA(cudaEventRecord(e1, 0));
    if (H->P > 0) PSFM_CUDA(cudaMemcpy(rgb, H->rgb.p, 3 * (size_t)H->P, cudaMemcpyDeviceToHost));
    PSFM_CUDA(cudaEventSynchronize(e1));
    if (summary) {
      summary->num_batches = H->num_batches;
      summary->num_images = H->num_images;
      summary->num_observations = H->N;
      summary->setup_ms = H->setup_ms;
      summary->upload_ms = H->upload_ms;
      summary->sample_ms = H->sample_ms;
      summary->mean_ms = elapsed(e0, e1);
      summary->stage_ms = H->stage_ms;
    }
    return PSFM_OK;
  });
}

extern "C" void psfm_colors_destroy(psfm_colors* H) {
  delete H;
  cudaGetLastError();
}
