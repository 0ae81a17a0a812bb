// triangulation_handle.cuh — the resident result of psfm_triangulation_create (triangulation.cu), shared with
// ba_solver.cu: psfm_ba_create_from_triangulation builds the bundle-adjustment problem from the keypoints and
// point3D_of_keypoint kept here without copying them to the host (DESIGN.md §4.9).
#pragma once
#include <vector>

#include "psfm_common.cuh"

struct psfm_triangulation {
  long long P = 0, E = 0, K = 0;
  int F = 0, C = 0;
  psfm_triangulation_summary summary;
  psfm::DBuf<double> xyz;                    // [P][3]
  psfm::DBuf<long long> track_ptr, kp_points; // [P + 1], [K] (point row, -1)
  psfm::DBuf<int> track_image, track_p2d;    // [E]
  psfm::DBuf<long long> kp_ptr;              // [F + 1]
  psfm::DBuf<float2> kps;                    // [K] as stored in the database
  psfm::DBuf<int> img_of;                    // [K] image index of each keypoint
  std::vector<long long> h_kp_ptr;           // [F + 1]
  std::vector<int> image_camera;             // [F]
  std::vector<unsigned char> registered;     // [F]
};

namespace psfm {

// The observations ba.flatten makes of Triangulation.to_reconstruction: every keypoint of a registered image that has
// a point, registered images in ascending index, keypoints in index order.  image_rank [F] (host) gives each
// registered image's problem index and -1 for the others.  Fills obs_image (problem image index), obs_point (point
// row), obs_xy (the keypoint as double) and obs_kp (keypoint index) on `st` and returns their number.
long long triangulation_observations(const psfm_triangulation* h, const int* image_rank, cudaStream_t st,
                                     DBuf<int>& obs_image, DBuf<int>& obs_point, DBuf<double2>& obs_xy, DBuf<int>& obs_kp);

}  // namespace psfm
