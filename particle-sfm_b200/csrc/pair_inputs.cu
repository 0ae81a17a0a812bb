// pair_inputs.cu — host checks of the image-pair graph (pair_inputs.h).  No device code.
#include "pair_inputs.h"

#include <algorithm>
#include <thread>
#include <vector>

#include "psfm_common.cuh"

namespace psfm {

namespace {

// every match's keypoint indices inside its images' keypoint ranges (host, split over threads: up to 10^9 indices)
bool keypoints_in_range(int64_t R, const int32_t* pair_images, const int64_t* kp_ptr, const int64_t* iptr, const uint32_t* m) {
  const unsigned nt = std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
  std::vector<char> ok(nt, 1);
  const long long N = iptr[R];
  host_fan(nt, [&](unsigned w) {
    const long long lo = N * w / nt, hi = N * (w + 1) / nt;
    if (lo >= hi) return;
    int64_t p = std::upper_bound(iptr, iptr + R + 1, (int64_t)lo) - iptr - 1;
    for (long long i = lo; i < hi;) {
      while (iptr[p + 1] <= i) ++p;
      const long long e = std::min<long long>(hi, iptr[p + 1]);
      const uint64_t na = (uint64_t)(kp_ptr[pair_images[2 * p] + 1] - kp_ptr[pair_images[2 * p]]);
      const uint64_t nb = (uint64_t)(kp_ptr[pair_images[2 * p + 1] + 1] - kp_ptr[pair_images[2 * p + 1]]);
      uint32_t ma = 0, mb = 0;
      bool any = false;
      for (long long k = i; k < e; ++k) {
        ma = std::max(ma, m[2 * k]);
        mb = std::max(mb, m[2 * k + 1]);
        any = true;
      }
      if (any && ((uint64_t)ma >= na || (uint64_t)mb >= nb)) { ok[w] = 0; return; }
      i = e;
    }
  });
  return std::all_of(ok.begin(), ok.end(), [](char c) { return c != 0; });
}

}  // namespace

int check_sizes(const char* entry, int64_t num_images, int64_t num_cameras, int64_t num_pairs) {
  if (num_images < 0 || num_cameras < 0 || num_pairs < 0) return fail(entry, PSFM_ERR_INVALID, "negative size");
  if (num_pairs > 0x7fffffffLL) return fail(entry, PSFM_ERR_INVALID, "more than 2^31 - 1 pairs");
  return PSFM_OK;
}

int check_keypoint_ptr(const char* entry, int32_t num_images, const int64_t* keypoint_ptr) {
  if (keypoint_ptr[0] != 0) return fail(entry, PSFM_ERR_INVALID, "keypoint_ptr[0] must be 0");
  for (int32_t f = 0; f < num_images; ++f)
    if (keypoint_ptr[f + 1] < keypoint_ptr[f]) return fail(entry, PSFM_ERR_INVALID, "keypoint_ptr must be non-decreasing");
  return PSFM_OK;
}

int check_image_cameras(const char* entry, int32_t num_images, const int32_t* image_camera, int32_t num_cameras) {
  for (int32_t f = 0; f < num_images; ++f)
    if (image_camera[f] < 0 || image_camera[f] >= num_cameras)
      return fail(entry, PSFM_ERR_INVALID, "a camera index is outside [0, num_cameras)");
  return PSFM_OK;
}

int check_camera_sizes(const char* entry, int32_t num_cameras, const int32_t* camera_size) {
  for (int32_t i = 0; i < num_cameras; ++i)
    if (!(camera_size[2 * i] > 0 && camera_size[2 * i + 1] > 0)) return fail(entry, PSFM_ERR_INVALID, "a camera size <= 0");
  return PSFM_OK;
}

int check_match_ptr(const char* entry, const char* name, int64_t num_pairs, const int64_t* ptr) {
  if (ptr[0] != 0) return fail(entry, PSFM_ERR_INVALID, std::string(name) + "[0] must be 0");
  for (int64_t p = 0; p < num_pairs; ++p)
    if (ptr[p + 1] < ptr[p]) return fail(entry, PSFM_ERR_INVALID, std::string(name) + " must be non-decreasing");
  return PSFM_OK;
}

int check_pair_images(const char* entry, int64_t num_pairs, const int32_t* pair_images, int32_t num_images) {
  for (int64_t i = 0; i < 2 * num_pairs; ++i)
    if (pair_images[i] < 0 || pair_images[i] >= num_images)
      return fail(entry, PSFM_ERR_INVALID, "an image index is outside [0, num_images)");
  return PSFM_OK;
}

int check_distinct_pairs(const char* entry, int64_t num_pairs, const int32_t* pair_images) {
  std::vector<uint64_t> keys(num_pairs);
  for (int64_t p = 0; p < num_pairs; ++p) {
    const int a = pair_images[2 * p], b = pair_images[2 * p + 1];
    if (a == b) return fail(entry, PSFM_ERR_INVALID, "a pair of an image with itself");
    keys[p] = ((uint64_t)std::min(a, b) << 32) | (uint64_t)std::max(a, b);
  }
  std::sort(keys.begin(), keys.end());
  if (std::adjacent_find(keys.begin(), keys.end()) != keys.end())
    return fail(entry, PSFM_ERR_INVALID, "an unordered image pair is listed twice");
  return PSFM_OK;
}

int check_match_keypoints(const char* entry, int64_t num_pairs, const int32_t* pair_images, const int64_t* keypoint_ptr,
                          const int64_t* ptr, const uint32_t* matches) {
  if (!keypoints_in_range(num_pairs, pair_images, keypoint_ptr, ptr, matches))
    return fail(entry, PSFM_ERR_INVALID, "a keypoint index is outside its image's keypoints");
  return PSFM_OK;
}

}  // namespace psfm
