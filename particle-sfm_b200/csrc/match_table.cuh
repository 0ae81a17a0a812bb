// match_table.cuh — the database match table resident on the device: csrc/handoff.cu builds it from a psfm_matches
// handle (psfm_matches_table), csrc/verification.cu verifies it in place (psfm_match_table_verify).  The arrays are
// those of handoff.MatchTables: images in image_id order, pairs in pair_id order with image 1 the smaller id.
// psfm::matches_build is the handle's construction from a track set already on the device (csrc/handoff.cu), shared
// by psfm_matches_create and psfm_tracker_matches (csrc/tracker.cu).
#pragma once
#include <vector>

#include "../../include/psfm_b200.h"
#include "psfm_common.cuh"

struct psfm_match_table {
  int num_images = 0;
  long long num_keypoints = 0, num_pairs = 0, num_matches = 0;
  std::vector<long long> keypoint_ptr;          // [num_images + 1], host copy
  std::vector<long long> match_ptr;             // [num_pairs + 1], host copy
  std::vector<int> pair_images;                 // [num_pairs][2] image rows, host copy
  psfm::DBuf<long long> d_keypoint_ptr, d_match_ptr;
  psfm::DBuf<float2> keypoints;                 // [num_keypoints] COLMAP origin (x + 0.5, y + 0.5)
  psfm::DBuf<int2> pairs;                       // [num_pairs]
  psfm::DBuf<uint2> matches;                    // [num_matches] (point2D_idx1, point2D_idx2)
};

namespace psfm {

// A track set in device memory: trajectory t owns samples tptr[t] .. tptr[t + 1] (tptr [num_trajs + 1]), with frame
// ids frames [num_obs] (int64) and locations xy [num_obs][2].  A non-null owner is freed by matches_build as soon as
// its array has been read, which keeps the build's peak at the record sort's.
struct TrackSetDev {
  const long long* tptr = nullptr;
  const long long* frames = nullptr;
  const double* xy = nullptr;
  long long num_trajs = 0, num_obs = 0;
  DBuf<long long>* own_tptr = nullptr;
  DBuf<long long>* own_frames = nullptr;
  DBuf<double>* own_xy = nullptr;
};

template <typename T>
inline void drop(DBuf<T>* b) {
  if (b) b->release();
}

// steps 1-7 of csrc/handoff.cu on `st`: the psfm_matches handle of psfm_matches_create for a track set already on the
// device (num_obs < 2^31, sample_k >= 1, num_images >= 0; the caller has checked them and the device)
int matches_build(const char* entry, TrackSetDev& in, int num_images, int sample_k, cudaStream_t st, psfm_matches** out,
                  int64_t* num_pairs, int64_t* num_matches);

}  // namespace psfm
