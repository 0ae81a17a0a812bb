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
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <numeric>
#include <vector>

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
};

extern "C" int psfm_matches_create(const int64_t* traj_ptr, int64_t num_trajs, const int64_t* frame_ids, const double* xy,
                                   int32_t num_images, int32_t sample_k, psfm_matches** out, int64_t* num_pairs,
                                   int64_t* num_matches) {
  const char* entry = "psfm_matches_create";
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
  psfm_matches* H = new psfm_matches;
  H->num_images = num_images;
  H->num_obs = N;
  H->kstart.assign((size_t)num_images + 1, 0);
  H->pair_ptr.assign(1, 0);
  if (N == 0) {                                     // empty or all-dynamic track set: nothing to launch
    *out = H;
    *num_pairs = *num_matches = 0;
    return PSFM_OK;
  }
  try {
    const int n = (int)N, K = sample_k, NI = num_images;
    DBuf<long long> tptr, frames, cnt, off, kstart;
    DBuf<double> dxy;
    DBuf<int> f32a, f32b, ida, idb, kp, bad;
    tptr.alloc((size_t)num_trajs + 1); frames.alloc(N); dxy.alloc(2 * (size_t)N);
    tptr.upload(reinterpret_cast<const long long*>(traj_ptr), tptr.n, nullptr);
    frames.upload(reinterpret_cast<const long long*>(frame_ids), N, nullptr); dxy.upload(xy, 2 * (size_t)N, nullptr);
    f32a.alloc(N); f32b.alloc(N); ida.alloc(N); idb.alloc(N); cnt.alloc(N + 1); bad.alloc(1);
    bad.zero(nullptr);
    k_count<<<grid_of(N + 1), 256>>>(n, tptr.p, num_trajs, frames.p, NI, K, f32a.p, ida.p, cnt.p, bad.p);
    PSFM_LAUNCH_CHECK();
    frames.release();
    // visiting positions: exclusive int64 scan of the per-sample counts, off[N] = number of records
    off.alloc(N + 1);
    {
      size_t bytes = 0;
      PSFM_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, cnt.p, off.p, n + 1, nullptr));
      DBuf<unsigned char> tmp;
      tmp.alloc(bytes);
      PSFM_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, bytes, cnt.p, off.p, n + 1, nullptr));
      PSFM_LAUNCH_CHECK();
    }
    cnt.release();
    int h_bad = 0;
    long long M = 0;
    PSFM_CUDA(cudaMemcpy(&h_bad, bad.p, sizeof(int), cudaMemcpyDeviceToHost));
    PSFM_CUDA(cudaMemcpy(&M, off.p + N, sizeof(long long), cudaMemcpyDeviceToHost));
    if (h_bad) {
      delete H;
      return fail(entry, PSFM_ERR_INVALID, "a frame id is outside [0, num_images)");
    }
    // keypoints: stable sort of the samples by frame
    cub::DoubleBuffer<int> fk(f32a.p, f32b.p), fv(ida.p, idb.p);
    // k_records reads the unsorted frames: sort copies of them
    DBuf<int> frame32;
    frame32.alloc(N);
    PSFM_CUDA(cudaMemcpy(frame32.p, f32a.p, sizeof(int) * (size_t)N, cudaMemcpyDeviceToDevice));
    sort_pairs(fk, fv, n, key_bits(NI > 0 ? (u64)(NI - 1) : 0));
    kstart.alloc((size_t)NI + 1);
    k_kp_start<<<grid_of((long long)NI + 1), 256>>>(NI, fk.Current(), n, kstart.p);
    PSFM_LAUNCH_CHECK();
    kp.alloc(N);
    H->kxy.alloc(2 * (size_t)N);
    k_kp<<<grid_of(N), 256>>>(n, fk.Current(), fv.Current(), kstart.p, reinterpret_cast<const double2*>(dxy.p), kp.p,
                              reinterpret_cast<double2*>(H->kxy.p));
    PSFM_LAUNCH_CHECK();
    PSFM_CUDA(cudaMemcpy(H->kstart.data(), kstart.p, sizeof(long long) * ((size_t)NI + 1), cudaMemcpyDeviceToHost));
    f32a.release(); f32b.release(); ida.release(); idb.release(); dxy.release();
    H->num_matches = M;
    if (M > 0) {
      // match records at their visiting positions, then stable by pair key
      DBuf<u64> ka, kb, va, vb;
      ka.alloc(M); kb.alloc(M); va.alloc(M); vb.alloc(M);
      k_records<<<grid_of(N), 256>>>(n, tptr.p, num_trajs, frame32.p, off.p, K, NI, ka.p, va.p);
      PSFM_LAUNCH_CHECK();
      off.release(); frame32.release(); tptr.release();
      cub::DoubleBuffer<u64> rk(ka.p, kb.p), rv(va.p, vb.p);
      sort_pairs(rk, rv, (long long)M, key_bits((u64)NI * (u64)NI - 1));
      release_other(ka, kb, rk.Current());
      release_other(va, vb, rv.Current());
      const u64* skey = rk.Current();
      const u64* sval = rv.Current();
      // runs of equal keys = image pairs
      const long long max_runs = std::min<long long>(M, (long long)NI * NI);
      DBuf<long long> heads;
      DBuf<unsigned long long> nheads;
      heads.alloc(max_runs); nheads.alloc(1);
      nheads.zero(nullptr);
      k_run_heads<<<grid_stride_of(M), 256>>>(M, skey, heads.p, nheads.p);
      PSFM_LAUNCH_CHECK();
      unsigned long long R64 = 0;
      PSFM_CUDA(cudaMemcpy(&R64, nheads.p, sizeof(R64), cudaMemcpyDeviceToHost));
      const int R = (int)R64;
      DBuf<u64> rkey, rfirst;
      rkey.alloc(R); rfirst.alloc(R);
      k_run_info<<<grid_of(R), 256>>>(R, heads.p, skey, sval, rkey.p, rfirst.p);
      PSFM_LAUNCH_CHECK();
      std::vector<long long> h_heads(R);
      std::vector<u64> h_key(R), h_first(R);
      PSFM_CUDA(cudaMemcpy(h_heads.data(), heads.p, sizeof(long long) * R, cudaMemcpyDeviceToHost));
      PSFM_CUDA(cudaMemcpy(h_key.data(), rkey.p, sizeof(u64) * R, cudaMemcpyDeviceToHost));
      PSFM_CUDA(cudaMemcpy(h_first.data(), rfirst.p, sizeof(u64) * R, cudaMemcpyDeviceToHost));
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
      d_start.upload(h_start.data(), R, nullptr); d_dest.upload(h_dest.data(), R, nullptr);
      H->matches.alloc(2 * (size_t)M);
      k_scatter<<<grid_stride_of(M), 256>>>(M, d_start.p, R, d_dest.p, sval, kp.p, H->matches.p);
      PSFM_LAUNCH_CHECK();
      PSFM_CUDA(cudaDeviceSynchronize());
    }
    *num_pairs = (int64_t)(H->pair_ptr.size() - 1);
    *num_matches = M;
    *out = H;
    return PSFM_OK;
  } catch (const CudaFail& f) {
    delete H;
    return f.code;
  }
}

extern "C" int psfm_matches_result(const psfm_matches* H, int64_t* keypoint_ptr, double* keypoints, int64_t* pair_images,
                                   int64_t* pair_ptr, int64_t* matches) {
  if (!H || !keypoint_ptr || !pair_ptr || (H->num_obs && !keypoints) || (H->num_matches && (!pair_images || !matches)))
    return fail("psfm_matches_result", PSFM_ERR_INVALID, "null argument");
  try {
    std::copy(H->kstart.begin(), H->kstart.end(), keypoint_ptr);
    std::copy(H->pair_ptr.begin(), H->pair_ptr.end(), pair_ptr);
    std::copy(H->pair_images.begin(), H->pair_images.end(), pair_images);
    if (H->num_obs)
      PSFM_CUDA(cudaMemcpy(keypoints, H->kxy.p, sizeof(double) * 2 * (size_t)H->num_obs, cudaMemcpyDeviceToHost));
    if (H->num_matches)
      PSFM_CUDA(cudaMemcpy(matches, H->matches.p, sizeof(long long) * 2 * (size_t)H->num_matches, cudaMemcpyDeviceToHost));
    return PSFM_OK;
  } catch (const CudaFail& f) { return f.code; }
}

extern "C" void psfm_matches_destroy(psfm_matches* H) {
  delete H;
  cudaGetLastError();
}
