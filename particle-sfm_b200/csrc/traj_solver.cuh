// traj_solver.cuh — internal entry into HP1 for other units of the library (the resident tracker stage).
// k_traj_solve itself stays in traj_solver.cu, the one unit compiled with -fmad=false.
#pragma once
#include "psfm_common.cuh"

namespace psfm {
namespace traj {

// HP1 on DEVICE pointers, under the lock of the library's shared HP1 workspace (the one psfm_traj_optimize /
// psfm_traj_optimize_device use).  n > 0.  It runs on `stream` and synchronises it before returning.  A NULL
// `stream` means the workspace's own stream, created cudaStreamNonBlocking: it is ordered after no other work,
// so a caller whose inputs were written on the legacy default stream passes cudaStreamLegacy, not NULL.
int solve_device(const double* d_uv12, const double* d_ref1, const double* d_ref2, const double* d_scale,
                 const float* d_flow12, int n, int w, int h, const psfm_traj_options* opts, double* d_out,
                 psfm_traj_summary* summary, cudaStream_t stream);

}  // namespace traj
}  // namespace psfm
