// handoff.cu — track set -> per-image keypoints and pairwise matches on the device (SURVEY.md §8(f) row f-2).
//
// Computes exactly what handoff.traj_to_matches (the array restatement of the reference's traj_to_matches,
// sfm/matches_from_flow.py:51-118) computes.  Everything is integer bookkeeping; the only floating-point values
// are the copied keypoint locations.  Visiting order of the reference: trajectory, then kept sample j, then the
// k loop.  Pipeline (N kept samples, M match records, R image pairs):
//   1. k_count        per sample: its number of match records (closed form), frame range check
//   2. radix sort     (frame, sample) pairs, stable: keypoint index = rank among the samples of the same frame
//   3. scan           int64 exclusive scan of the counts: the visiting position of every sample's first record
//   4. k_records      per sample: its records at their visiting positions, key = a * num_images + b, value =
//                     (src << 32 | dst); visiting order is the lexicographic order of (src, dst)
//   5. radix sort     records by pair key, stable: every pair's records in one run, in visiting order
//   6. k_run_heads    the runs, their keys and first records; the host orders the R runs by (a, first record)
//   7. k_scatter      each record to pair_ptr[rank of its run] + its place in the run, as (kp[src], kp[dst])
// Memory: 32 bytes per record during the sort (keys and values, double-buffered), 24 bytes per record in the
// scatter (sorted values and the int64 output), about 80 bytes per sample besides.
//
// psfm_matches_table then moves the result into the database match table (match_table.cuh), what
// handoff.import_keypoints_matches_arrays followed by MatchTables.from_rows builds on the host:
//   8. k_table_keypoints  per keypoint: float32(x + 0.5) at its image's row in image_id order (16 B in, 8 B out)
//   9. k_table_matches    per kept match: its run's record, columns swapped where the run's source image has the
//                         larger id, as uint32 (16 B in, 8 B out)
// Of the two ordered runs of one image pair the one whose source frame comes first by name is kept: the reference
// visits images in get_image_ids order, which SQLite returns in name order (tests/golden/import_small.npz).
// The host picks one ordered run per unordered pair and orders the pairs by pair_id; the handle's int64 matches and
// double keypoints are freed once the table exists, so the peak stays at or below the record sort's.
//
// Steps 1-7 (psfm::matches_build) start from the track set on the device: psfm_matches_create uploads the host arrays
// and hands them over to be freed as soon as they are read; psfm_tracker_matches (csrc/tracker.cu) passes the finished
// tracker's own arrays, which stay where they are, and runs on the tracker's stream.
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <numeric>
#include <vector>

#include "match_table.cuh"
#include "psfm_common.cuh"
#include "radix_sort.cuh"

namespace {

using namespace psfm;
typedef unsigned long long u64;

// first index in a[0 .. n) with a[idx] > v (a non-decreasing)
__device__ __forceinline__ long long upper_bound_ll(const long long* a, long long n, long long v) {
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (a[mid] <= v) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// the trajectory of kept sample i: its first sample and its number of kept samples
__device__ __forceinline__ void sample_traj(const long long* tptr, long long ntraj, long long i, long long* start, int* n) {
  const long long t = upper_bound_ll(tptr, ntraj + 1, i) - 1;
  *start = tptr[t];
  *n = (int)(tptr[t + 1] - tptr[t]);
}

// matches_from_flow.py:91-103: n <= K: every k != j; otherwise the K targets s * (n // K), minus j itself
__device__ __forceinline__ int match_count(int n, int j, int K) {
  if (n <= K) return n - 1;
  const int stride = n / K;
  return (j % stride == 0 && j / stride < K) ? K - 1 : K;
}

__global__ void k_count(int N, const long long* tptr, long long ntraj, const long long* frames, int num_images, int K,
                        int* frame32, int* iota, long long* cnt, int* bad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > N) return;
  if (i == N) { cnt[N] = 0; return; }
  long long f = frames[i];
  if (f < 0 || f >= num_images) {
    atomicOr(bad, 1);
    f = 0;
  }
  frame32[i] = (int)f;
  iota[i] = i;
  long long start;
  int n;
  sample_traj(tptr, ntraj, i, &start, &n);
  cnt[i] = match_count(n, (int)(i - start), K);
}

// keypoint_ptr[f] = first position of frame f in the frame-sorted samples
__global__ void k_kp_start(int num_images, const int* sframe, int N, long long* kstart) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > num_images) return;
  int lo = 0, hi = N;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (sframe[mid] < f) lo = mid + 1;
    else hi = mid;
  }
  kstart[f] = lo;
}

// keypoint index of sample order[q] and its location at keypoint position q
__global__ void k_kp(int N, const int* sframe, const int* order, const long long* kstart, const double2* xy, int* kp, double2* kxy) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= N) return;
  const int i = order[q];
  kp[i] = (int)(q - kstart[sframe[q]]);
  kxy[q] = xy[i];
}

__global__ void k_records(int N, const long long* tptr, long long ntraj, const int* frame32, const long long* off, int K,
                          int num_images, u64* keys, u64* vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  long long start;
  int n;
  sample_traj(tptr, ntraj, i, &start, &n);
  const int j = (int)(i - start);
  const u64 a = (u64)frame32[i] * (u64)num_images, hi = (u64)i << 32;
  long long p = off[i];
  if (n <= K) {
    for (int k = 0; k < n; ++k) {
      if (k == j) continue;
      const long long dst = start + k;
      keys[p] = a + (u64)frame32[dst];
      vals[p] = hi | (u64)dst;
      ++p;
    }
  } else {
    const int stride = n / K;
    for (int s = 0; s < K; ++s) {
      const int k = s * stride;
      if (k == j) continue;
      const long long dst = start + k;
      keys[p] = a + (u64)frame32[dst];
      vals[p] = hi | (u64)dst;
      ++p;
    }
  }
}

// the first record of every run of equal keys, in no particular order
__global__ void k_run_heads(long long M, const u64* skey, long long* heads, unsigned long long* nheads) {
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < M; q += (long long)gridDim.x * blockDim.x)
    if (q == 0 || skey[q] != skey[q - 1]) heads[atomicAdd(nheads, 1ull)] = q;
}

__global__ void k_run_info(int R, const long long* heads, const u64* skey, const u64* sval, u64* rkey, u64* rfirst) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  rkey[r] = skey[heads[r]];
  rfirst[r] = sval[heads[r]];
}

__global__ void k_scatter(long long M, const long long* run_start, int R, const long long* dest_start, const u64* sval, const int* kp,
                          long long* out) {
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < M; q += (long long)gridDim.x * blockDim.x) {
    const long long r = upper_bound_ll(run_start, R, q) - 1;
    const long long d = dest_start[r] + (q - run_start[r]);
    const u64 v = sval[q];
    out[2 * d] = kp[v >> 32];
    out[2 * d + 1] = kp[v & 0xffffffffull];
  }
}

// keypoint s of the handle (frame-major) -> its row in image_id order, shifted to COLMAP's origin: the double sum
// rounded once to nearest, which is numpy's float64 -> float32 cast
__global__ void k_table_keypoints(long long N, const long long* kstart, int NI, const long long* dst_start,
                                  const double2* kxy, float2* out) {
  for (long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x; s < N; s += (long long)gridDim.x * blockDim.x) {
    const long long f = upper_bound_ll(kstart, (long long)NI + 1, s) - 1;
    const double2 v = kxy[s];
    out[dst_start[f] + (s - kstart[f])] = make_float2(__double2float_rn(__dadd_rn(v.x, 0.5)), __double2float_rn(__dadd_rn(v.y, 0.5)));
  }
}

// match q of the table -> record src[p] + (q - mptr[p]) of the handle, columns swapped when swap[p]
__global__ void k_table_matches(long long M, const long long* mptr, int R, const long long* src, const unsigned char* swap,
                                const long long* in, uint2* out) {
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < M; q += (long long)gridDim.x * blockDim.x) {
    const long long p = upper_bound_ll(mptr, (long long)R + 1, q) - 1;
    const long long r = src[p] + (q - mptr[p]);
    const unsigned a = (unsigned)in[2 * r], b = (unsigned)in[2 * r + 1];
    out[q] = swap[p] ? make_uint2(b, a) : make_uint2(a, b);
  }
}

// of two buffers, free the one a CUB double buffer does not currently point at
template <typename T>
void release_other(DBuf<T>& a, DBuf<T>& b, const T* current) {
  if (current == a.p) b.release();
  else a.release();
}

}  // namespace

struct psfm_matches {
  int num_images = 0;
  long long num_obs = 0, num_matches = 0;
  std::vector<long long> kstart;               // [num_images + 1]
  std::vector<long long> pair_images, pair_ptr;
  DBuf<double> kxy;                            // [num_obs][2] keypoints, image-major
  DBuf<long long> matches;                     // [num_matches][2]
  bool moved = false;                          // kxy and matches were moved into a match table
};

namespace psfm {

int matches_build(const char* entry, TrackSetDev& in, int num_images, int sample_k, cudaStream_t st, psfm_matches** out,
                  int64_t* num_pairs, int64_t* num_matches) {
  const long long N = in.num_obs, num_trajs = in.num_trajs;
  std::unique_ptr<psfm_matches> H(new psfm_matches);
  H->num_images = num_images;
  H->num_obs = N;
  H->kstart.assign((size_t)num_images + 1, 0);
  H->pair_ptr.assign(1, 0);
  if (N == 0) {                                     // empty or all-dynamic track set: nothing to launch
    *out = H.release();
    *num_pairs = *num_matches = 0;
    return PSFM_OK;
  }
  const int n = (int)N, K = sample_k, NI = num_images;
  DBuf<long long> cnt, off, kstart;
  DBuf<int> f32a, f32b, ida, idb, kp, bad;
  f32a.alloc(N); f32b.alloc(N); ida.alloc(N); idb.alloc(N); cnt.alloc(N + 1); bad.alloc(1);
  bad.zero(st);
  k_count<<<grid_of(N + 1), 256, 0, st>>>(n, in.tptr, num_trajs, in.frames, NI, K, f32a.p, ida.p, cnt.p, bad.p);
  PSFM_LAUNCH_CHECK();
  // visiting positions: exclusive int64 scan of the per-sample counts, off[N] = number of records
  off.alloc(N + 1);
  {
    size_t bytes = 0;
    PSFM_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, cnt.p, off.p, n + 1, st));
    DBuf<unsigned char> tmp;
    tmp.alloc(bytes, st);
    PSFM_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, bytes, cnt.p, off.p, n + 1, st));
    PSFM_LAUNCH_CHECK();
  }
  int h_bad = 0;
  long long M = 0;
  PSFM_CUDA(cudaMemcpyAsync(&h_bad, bad.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  PSFM_CUDA(cudaMemcpyAsync(&M, off.p + N, sizeof(long long), cudaMemcpyDeviceToHost, st));
  PSFM_CUDA(cudaStreamSynchronize(st));
  cnt.release();
  drop(in.own_frames);
  if (h_bad) return fail(entry, PSFM_ERR_INVALID, "a frame id is outside [0, num_images)");
  // keypoints: stable sort of the samples by frame
  cub::DoubleBuffer<int> fk(f32a.p, f32b.p), fv(ida.p, idb.p);
  // k_records reads the unsorted frames: sort copies of them
  DBuf<int> frame32;
  frame32.alloc(N);
  PSFM_CUDA(cudaMemcpyAsync(frame32.p, f32a.p, sizeof(int) * (size_t)N, cudaMemcpyDeviceToDevice, st));
  sort_pairs(fk, fv, n, key_bits(NI > 0 ? (u64)(NI - 1) : 0), st);
  kstart.alloc((size_t)NI + 1);
  k_kp_start<<<grid_of((long long)NI + 1), 256, 0, st>>>(NI, fk.Current(), n, kstart.p);
  PSFM_LAUNCH_CHECK();
  kp.alloc(N);
  H->kxy.alloc(2 * (size_t)N);
  k_kp<<<grid_of(N), 256, 0, st>>>(n, fk.Current(), fv.Current(), kstart.p, reinterpret_cast<const double2*>(in.xy), kp.p,
                                   reinterpret_cast<double2*>(H->kxy.p));
  PSFM_LAUNCH_CHECK();
  PSFM_CUDA(cudaMemcpyAsync(H->kstart.data(), kstart.p, sizeof(long long) * ((size_t)NI + 1), cudaMemcpyDeviceToHost, st));
  PSFM_CUDA(cudaStreamSynchronize(st));
  f32a.release(); f32b.release(); ida.release(); idb.release(); drop(in.own_xy);
  H->num_matches = M;
  if (M > 0) {
    // match records at their visiting positions, then stable by pair key
    DBuf<u64> ka, kb, va, vb;
    ka.alloc(M); kb.alloc(M); va.alloc(M); vb.alloc(M);
    k_records<<<grid_of(N), 256, 0, st>>>(n, in.tptr, num_trajs, frame32.p, off.p, K, NI, ka.p, va.p);
    PSFM_LAUNCH_CHECK();
    PSFM_CUDA(cudaStreamSynchronize(st));
    off.release(); frame32.release(); drop(in.own_tptr);
    cub::DoubleBuffer<u64> rk(ka.p, kb.p), rv(va.p, vb.p);
    sort_pairs(rk, rv, (long long)M, key_bits((u64)NI * (u64)NI - 1), st);
    PSFM_CUDA(cudaStreamSynchronize(st));
    release_other(ka, kb, rk.Current());
    release_other(va, vb, rv.Current());
    const u64* skey = rk.Current();
    const u64* sval = rv.Current();
    // runs of equal keys = image pairs
    const long long max_runs = std::min<long long>(M, (long long)NI * NI);
    DBuf<long long> heads;
    DBuf<unsigned long long> nheads;
    heads.alloc(max_runs); nheads.alloc(1);
    nheads.zero(st);
    k_run_heads<<<grid_stride_of(M), 256, 0, st>>>(M, skey, heads.p, nheads.p);
    PSFM_LAUNCH_CHECK();
    unsigned long long R64 = 0;
    PSFM_CUDA(cudaMemcpyAsync(&R64, nheads.p, sizeof(R64), cudaMemcpyDeviceToHost, st));
    PSFM_CUDA(cudaStreamSynchronize(st));
    const int R = (int)R64;
    DBuf<u64> rkey, rfirst;
    rkey.alloc(R); rfirst.alloc(R);
    k_run_info<<<grid_of(R), 256, 0, st>>>(R, heads.p, skey, sval, rkey.p, rfirst.p);
    PSFM_LAUNCH_CHECK();
    std::vector<long long> h_heads(R);
    std::vector<u64> h_key(R), h_first(R);
    PSFM_CUDA(cudaMemcpyAsync(h_heads.data(), heads.p, sizeof(long long) * R, cudaMemcpyDeviceToHost, st));
    PSFM_CUDA(cudaMemcpyAsync(h_key.data(), rkey.p, sizeof(u64) * R, cudaMemcpyDeviceToHost, st));
    PSFM_CUDA(cudaMemcpyAsync(h_first.data(), rfirst.p, sizeof(u64) * R, cudaMemcpyDeviceToHost, st));
    PSFM_CUDA(cudaStreamSynchronize(st));
    if (rk.Current() == ka.p) ka.release();
    else kb.release();
    // runs in sorted-record order (their heads), and the pair list: by image a, then first appearance
    std::vector<int> by_head(R), by_pair(R);
    std::iota(by_head.begin(), by_head.end(), 0);
    std::sort(by_head.begin(), by_head.end(), [&](int x, int y) { return h_heads[x] < h_heads[y]; });
    std::vector<long long> run_len(R);
    for (int r = 0; r < R; ++r)
      run_len[by_head[r]] = (r + 1 < R ? h_heads[by_head[r + 1]] : M) - h_heads[by_head[r]];
    std::iota(by_pair.begin(), by_pair.end(), 0);
    std::sort(by_pair.begin(), by_pair.end(), [&](int x, int y) {
      const u64 ax = h_key[x] / (u64)NI, ay = h_key[y] / (u64)NI;
      return ax != ay ? ax < ay : h_first[x] < h_first[y];
    });
    H->pair_images.resize(2 * (size_t)R);
    H->pair_ptr.assign((size_t)R + 1, 0);
    std::vector<long long> dest(R);
    for (int k = 0; k < R; ++k) {
      const int r = by_pair[k];
      H->pair_images[2 * k] = (long long)(h_key[r] / (u64)NI);
      H->pair_images[2 * k + 1] = (long long)(h_key[r] % (u64)NI);
      dest[r] = H->pair_ptr[k];
      H->pair_ptr[k + 1] = H->pair_ptr[k] + run_len[r];
    }
    std::vector<long long> h_start(R), h_dest(R);
    for (int r = 0; r < R; ++r) { h_start[r] = h_heads[by_head[r]]; h_dest[r] = dest[by_head[r]]; }
    DBuf<long long> d_start, d_dest;
    d_start.alloc(R); d_dest.alloc(R);
    d_start.upload(h_start.data(), R, st); d_dest.upload(h_dest.data(), R, st);
    H->matches.alloc(2 * (size_t)M);
    k_scatter<<<grid_stride_of(M), 256, 0, st>>>(M, d_start.p, R, d_dest.p, sval, kp.p, H->matches.p);
    PSFM_LAUNCH_CHECK();
    PSFM_CUDA(cudaStreamSynchronize(st));
  }
  *num_pairs = (int64_t)(H->pair_ptr.size() - 1);
  *num_matches = M;
  *out = H.release();
  return PSFM_OK;
}

}  // namespace psfm

extern "C" int psfm_matches_create(const int64_t* traj_ptr, int64_t num_trajs, const int64_t* frame_ids, const double* xy,
                                   int32_t num_images, int32_t sample_k, psfm_matches** out, int64_t* num_pairs,
                                   int64_t* num_matches) {
  const char* entry = "psfm_matches_create";
  return guard(entry, [&]() -> int {
    if (!out || !num_pairs || !num_matches || !traj_ptr) return fail(entry, PSFM_ERR_INVALID, "null argument");
    *out = nullptr;
    if (num_trajs < 0 || num_images < 0 || sample_k < 1)
      return fail(entry, PSFM_ERR_INVALID, "num_trajs and num_images must be >= 0, sample_k >= 1");
    if (traj_ptr[0] != 0) return fail(entry, PSFM_ERR_INVALID, "traj_ptr[0] must be 0");
    for (int64_t t = 0; t < num_trajs; ++t)
      if (traj_ptr[t + 1] < traj_ptr[t]) return fail(entry, PSFM_ERR_INVALID, "traj_ptr must be non-decreasing");
    const long long N = traj_ptr[num_trajs];
    if (N > 0x7fffffffLL) return fail(entry, PSFM_ERR_INVALID, "more than 2^31 - 1 samples");
    if (N > 0 && (!frame_ids || !xy)) return fail(entry, PSFM_ERR_INVALID, "null argument");
    int rc = require_device(entry);
    if (rc != PSFM_OK) return rc;
    DBuf<long long> tptr, frames;
    DBuf<double> dxy;
    TrackSetDev in;
    in.num_trajs = num_trajs;
    in.num_obs = N;
    if (N > 0) {
      tptr.alloc((size_t)num_trajs + 1); frames.alloc(N); dxy.alloc(2 * (size_t)N);
      tptr.upload(reinterpret_cast<const long long*>(traj_ptr), tptr.n, nullptr);
      frames.upload(reinterpret_cast<const long long*>(frame_ids), N, nullptr); dxy.upload(xy, 2 * (size_t)N, nullptr);
      in.tptr = tptr.p; in.frames = frames.p; in.xy = dxy.p;
      in.own_tptr = &tptr; in.own_frames = &frames; in.own_xy = &dxy;
    }
    return matches_build(entry, in, num_images, sample_k, nullptr, out, num_pairs, num_matches);
  });
}

extern "C" int psfm_matches_result(const psfm_matches* H, int64_t* keypoint_ptr, double* keypoints, int64_t* pair_images,
                                   int64_t* pair_ptr, int64_t* matches) {
  return guard("psfm_matches_result", [&]() -> int {
    if (H && H->moved && (keypoints || matches))
      return fail("psfm_matches_result", PSFM_ERR_INVALID,
                  "the keypoints and matches were moved into a match table; pass NULL for them");
    if (!H || !keypoint_ptr || !pair_ptr || (H->num_obs && !H->moved && !keypoints) ||
        (H->num_matches && (!pair_images || (!H->moved && !matches))))
      return fail("psfm_matches_result", PSFM_ERR_INVALID, "null argument");
    std::copy(H->kstart.begin(), H->kstart.end(), keypoint_ptr);
    std::copy(H->pair_ptr.begin(), H->pair_ptr.end(), pair_ptr);
    std::copy(H->pair_images.begin(), H->pair_images.end(), pair_images);
    if (H->moved) return PSFM_OK;
    if (H->num_obs)
      PSFM_CUDA(cudaMemcpy(keypoints, H->kxy.p, sizeof(double) * 2 * (size_t)H->num_obs, cudaMemcpyDeviceToHost));
    if (H->num_matches)
      PSFM_CUDA(cudaMemcpy(matches, H->matches.p, sizeof(long long) * 2 * (size_t)H->num_matches, cudaMemcpyDeviceToHost));
    return PSFM_OK;
  });
}

extern "C" void psfm_matches_destroy(psfm_matches* H) {
  delete H;
  cudaGetLastError();
}

extern "C" int psfm_matches_table(psfm_matches* H, const int32_t* image_ids, psfm_match_table** out, int64_t* num_keypoints,
                                  int64_t* num_pairs, int64_t* num_matches) {
  const char* entry = "psfm_matches_table";
  return guard(entry, [&]() -> int {
    if (!H || !out || !num_keypoints || !num_pairs || !num_matches) return fail(entry, PSFM_ERR_INVALID, "null argument");
    *out = nullptr;
    if (H->moved) return fail(entry, PSFM_ERR_INVALID, "the handle's matches were already moved into a match table");
    const int NI = H->num_images;
    if (NI > 0 && !image_ids) return fail(entry, PSFM_ERR_INVALID, "null argument");
    for (int f = 0; f < NI; ++f)
      if (image_ids[f] < 0 || image_ids[f] == 0x7fffffff)
        return fail(entry, PSFM_ERR_INVALID, "an image id is outside [0, 2^31 - 1)");
    std::vector<int> row_frame(NI);                   // frame of every row in image_id order
    std::iota(row_frame.begin(), row_frame.end(), 0);
    std::sort(row_frame.begin(), row_frame.end(), [&](int x, int y) { return image_ids[x] < image_ids[y]; });
    for (int r = 1; r < NI; ++r)
      if (image_ids[row_frame[r]] == image_ids[row_frame[r - 1]]) return fail(entry, PSFM_ERR_INVALID, "an image id is given twice");
    const long long Rh = (long long)H->pair_ptr.size() - 1;
    for (long long k = 0; k < Rh; ++k)
      if (H->pair_images[2 * k] == H->pair_images[2 * k + 1])
        return fail(entry, PSFM_ERR_INVALID, "a trajectory visits one frame twice (a pair of an image with itself)");
    int rc = require_device(entry);
    if (rc != PSFM_OK) return rc;
    std::unique_ptr<psfm_match_table> T(new psfm_match_table);
    T->num_images = NI;
    std::vector<int> row_of(NI);
    for (int r = 0; r < NI; ++r) row_of[row_frame[r]] = r;
    // images: keypoint rows in image_id order
    T->keypoint_ptr.assign((size_t)NI + 1, 0);
    std::vector<long long> dst_start(NI);
    for (int r = 0; r < NI; ++r) {
      const int f = row_frame[r];
      dst_start[f] = T->keypoint_ptr[r];
      T->keypoint_ptr[r + 1] = T->keypoint_ptr[r] + (H->kstart[f + 1] - H->kstart[f]);
    }
    const long long N = T->keypoint_ptr[NI];
    T->num_keypoints = N;
    // pairs: per unordered pair the first run in get_image_ids order (import_feature_matches.py:88-99), which is name
    // order, i.e. frame order: SQLite answers "SELECT name, image_id FROM images" from the unique index on name.  So
    // the run whose source frame is the smaller one, else the other one; its columns are swapped when its source has
    // the larger id (add_matches).  Then pair_id order.
    struct Run { int lo, hi; bool later, swap; long long k; };
    std::vector<Run> runs((size_t)Rh);
    for (long long k = 0; k < Rh; ++k) {
      const long long a = H->pair_images[2 * k], b = H->pair_images[2 * k + 1];
      const int ia = image_ids[a], ib = image_ids[b];
      runs[k] = {std::min(ia, ib), std::max(ia, ib), a > b, ia > ib, k};
    }
    std::sort(runs.begin(), runs.end(), [](const Run& x, const Run& y) {
      return x.lo != y.lo ? x.lo < y.lo : x.hi != y.hi ? x.hi < y.hi : x.later < y.later;
    });
    std::vector<long long> src;
    std::vector<unsigned char> swap;
    T->match_ptr.assign(1, 0);
    for (size_t i = 0; i < runs.size(); ++i) {
      if (i > 0 && runs[i].lo == runs[i - 1].lo && runs[i].hi == runs[i - 1].hi) continue;
      const long long k = runs[i].k;
      const int a = (int)H->pair_images[2 * k], b = (int)H->pair_images[2 * k + 1];
      src.push_back(H->pair_ptr[k]);
      swap.push_back(runs[i].swap);
      T->pair_images.push_back(runs[i].swap ? row_of[b] : row_of[a]);
      T->pair_images.push_back(runs[i].swap ? row_of[a] : row_of[b]);
      T->match_ptr.push_back(T->match_ptr.back() + (H->pair_ptr[k + 1] - H->pair_ptr[k]));
    }
    const int R = (int)src.size();
    const long long M = T->match_ptr[R];
    T->num_pairs = R;
    T->num_matches = M;
    T->d_keypoint_ptr.alloc((size_t)NI + 1);
    T->d_keypoint_ptr.upload(T->keypoint_ptr.data(), (size_t)NI + 1, nullptr);
    T->d_match_ptr.alloc((size_t)R + 1);
    T->d_match_ptr.upload(T->match_ptr.data(), (size_t)R + 1, nullptr);
    T->pairs.alloc(R);
    T->pairs.upload(reinterpret_cast<const int2*>(T->pair_images.data()), R, nullptr);
    T->keypoints.alloc(N);
    T->matches.alloc(M);
    if (N > 0) {
      DBuf<long long> d_kstart, d_dst;
      d_kstart.alloc((size_t)NI + 1); d_dst.alloc(NI);
      d_kstart.upload(H->kstart.data(), (size_t)NI + 1, nullptr);
      d_dst.upload(dst_start.data(), NI, nullptr);
      k_table_keypoints<<<grid_stride_of(N), 256>>>(N, d_kstart.p, NI, d_dst.p, reinterpret_cast<const double2*>(H->kxy.p),
                                                    T->keypoints.p);
      PSFM_LAUNCH_CHECK();
      PSFM_CUDA(cudaDeviceSynchronize());
    }
    if (M > 0) {
      DBuf<long long> d_src;
      DBuf<unsigned char> d_swap;
      d_src.alloc(R); d_swap.alloc(R);
      d_src.upload(src.data(), R, nullptr);
      d_swap.upload(swap.data(), R, nullptr);
      k_table_matches<<<grid_stride_of(M), 256>>>(M, T->d_match_ptr.p, R, d_src.p, d_swap.p, H->matches.p, T->matches.p);
      PSFM_LAUNCH_CHECK();
      PSFM_CUDA(cudaDeviceSynchronize());
    }
    H->kxy.release();
    H->matches.release();
    H->moved = true;
    *num_keypoints = N;
    *num_pairs = R;
    *num_matches = M;
    *out = T.release();
    return PSFM_OK;
  });
}

extern "C" int psfm_match_table_result(const psfm_match_table* T, int64_t* keypoint_ptr, float* keypoints, int32_t* pair_images,
                                       int64_t* match_ptr, uint32_t* matches) {
  return guard("psfm_match_table_result", [&]() -> int {
    if (!T || !keypoint_ptr || !match_ptr || (T->num_keypoints && !keypoints) || (T->num_pairs && !pair_images) ||
        (T->num_matches && !matches))
      return fail("psfm_match_table_result", PSFM_ERR_INVALID, "null argument");
    std::copy(T->keypoint_ptr.begin(), T->keypoint_ptr.end(), keypoint_ptr);
    std::copy(T->match_ptr.begin(), T->match_ptr.end(), match_ptr);
    std::copy(T->pair_images.begin(), T->pair_images.end(), pair_images);
    if (T->num_keypoints)
      PSFM_CUDA(cudaMemcpy(keypoints, T->keypoints.p, sizeof(float2) * (size_t)T->num_keypoints, cudaMemcpyDeviceToHost));
    if (T->num_matches)
      PSFM_CUDA(cudaMemcpy(matches, T->matches.p, sizeof(uint2) * (size_t)T->num_matches, cudaMemcpyDeviceToHost));
    return PSFM_OK;
  });
}

extern "C" void psfm_match_table_destroy(psfm_match_table* T) {
  delete T;
  cudaGetLastError();
}
