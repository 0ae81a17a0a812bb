// match_table.cuh — the database match table resident on the device: csrc/handoff.cu builds it from a psfm_matches
// handle (psfm_matches_table), csrc/verification.cu verifies it in place (psfm_match_table_verify).  The arrays are
// those of handoff.MatchTables: images in image_id order, pairs in pair_id order with image 1 the smaller id.
#pragma once
#include <vector>

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
