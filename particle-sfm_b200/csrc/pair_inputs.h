// pair_inputs.h — host checks of the image-pair graph that the pair stages take (two-view poses, pairwise
// translations, rotations, positions, triangulation, verification):
//   keypoint_ptr [F + 1], image_camera [F], camera_size [C][2], pair_images [R][2], a CSR pointer over the matches
//   (inlier_ptr or match_ptr) [R + 1] and the matches [N][2] (keypoint in image 1, keypoint in image 2).
// Each check sets "<entry>: <message>" and returns PSFM_ERR_INVALID on failure, else PSFM_OK.  An entry point calls
// the checks that apply to it, in its own order, and keeps the checks of its own stage.  With one fault in its input
// an entry point names that fault; with several, which one is named first depends on that order.
#pragma once
#include <stdint.h>

namespace psfm {

// "negative size"; "more than 2^31 - 1 pairs"
int check_sizes(const char* entry, int64_t num_images, int64_t num_cameras, int64_t num_pairs);
// keypoint_ptr[0] == 0 and non-decreasing
int check_keypoint_ptr(const char* entry, int32_t num_images, const int64_t* keypoint_ptr);
// every image's camera in [0, num_cameras)
int check_image_cameras(const char* entry, int32_t num_images, const int32_t* image_camera, int32_t num_cameras);
// every camera's width and height > 0
int check_camera_sizes(const char* entry, int32_t num_cameras, const int32_t* camera_size);
// name[0] == 0 and non-decreasing; name is the pointer's argument name (inlier_ptr, match_ptr)
int check_match_ptr(const char* entry, const char* name, int64_t num_pairs, const int64_t* ptr);
// every pair's images in [0, num_images)
int check_pair_images(const char* entry, int64_t num_pairs, const int32_t* pair_images, int32_t num_images);
// no pair of an image with itself, no unordered pair given twice (pair images in range)
int check_distinct_pairs(const char* entry, int64_t num_pairs, const int32_t* pair_images);
// every match's keypoint indices inside its images' keypoints (pointers and pair images valid; multi-threaded)
int check_match_keypoints(const char* entry, int64_t num_pairs, const int32_t* pair_images, const int64_t* keypoint_ptr,
                          const int64_t* ptr, const uint32_t* matches);

}  // namespace psfm
