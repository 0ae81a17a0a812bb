// track_npy.cuh — the device emitter of track.npy's state body (track_npy.cu), shared with the tracker handle.
#pragma once
#include <cuda_runtime.h>

#include "../../include/psfm_b200.h"

namespace psfm {

// the body for T trajectories in DEVICE arrays (ids [T], ptr [T + 1], frame ids and xy of ptr[T] observations), all
// valid (ids in [0, 2^31), frame ids >= 0, ptr monotone from 0), encoded on `st` into a new handle's pinned buffer
void track_npy_encode(const long long* ids, const long long* ptr, const int* frames, const double* xy, long long T, cudaStream_t st,
                      psfm_track_npy** out, int64_t* nbytes);

}  // namespace psfm
