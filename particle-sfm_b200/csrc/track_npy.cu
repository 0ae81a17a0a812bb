// track_npy.cu — the body of track.npy's pickled TrajectorySet state, written on the device (DESIGN.md §4.13).
//
// track.npy is np.save of a 0-d object array holding a particlesfm.TrajectorySet
// (point_trajectory/main_connect_point_trajectories.py:55-62).  Its pickled state is the dict of
// TrajectorySet.as_dict: {id: {"frame_ids": [...], "locations": [...], "labels": [...]}}.  This file writes that
// dict as pickle opcodes, one record per trajectory, in ids order:
//
//   id            K b | M bb | J bbbb                   (BININT1 / BININT2 / BININT, little-endian)
//   }( X"frame_ids" ](   then per frame id  K | M | J   then  e
//      X"locations" ](   then per location  G x G y \x86 (BINFLOAT big-endian, exact bits; TUPLE2)  then  e
//      X"labels"    ](   then per label     \x89 (NEWFALSE)  then  e
//   u
//
// and the whole body is }( records u (a lone } without trajectories).  No memo opcode is used, so the bytes of a
// record depend on that record alone: sizes, an exclusive scan of them, then one warp per record writes it.  The
// host frames the body with the npy header and the pickle opcodes numpy and pickle write around the state
// (point_trajectory.py); the oracle's numpy encoder writes the same bytes (oracle/track_npy_oracle.py).
#include <cub/device/device_scan.cuh>

#include "psfm_common.cuh"
#include "track_npy.cuh"

using namespace psfm;

struct psfm_track_npy {
  uint8_t* host = nullptr;     // pinned, `bytes` long
  int64_t bytes = 0;
};

namespace {

constexpr int kHeadFrames = 2 + 14 + 2;     // }(  X<u32 9>frame_ids  ](
constexpr int kHeadLocations = 1 + 14 + 2;  // e  X<u32 9>locations  ](
constexpr int kHeadLabels = 1 + 11 + 2;     // e  X<u32 6>labels  ](
constexpr int kTail = 2;                    // e u
constexpr int kFixed = kHeadFrames + kHeadLocations + kHeadLabels + kTail;
constexpr int kLocation = 1 + 8 + 1 + 8 + 1;  // G x G y \x86
constexpr int kLabel = 1;                     // \x89

// bytes of the BININT1 / BININT2 / BININT opcode of a non-negative int < 2^31
__device__ __forceinline__ int int_width(long long v) { return v < 256 ? 2 : (v < 65536 ? 3 : 5); }

__device__ __forceinline__ uint8_t* put_int(uint8_t* o, long long v) {
  if (v < 256) {
    o[0] = 'K'; o[1] = (uint8_t)v;
    return o + 2;
  }
  if (v < 65536) {
    o[0] = 'M'; o[1] = (uint8_t)v; o[2] = (uint8_t)(v >> 8);
    return o + 3;
  }
  o[0] = 'J';
  for (int b = 0; b < 4; ++b) o[1 + b] = (uint8_t)(v >> (8 * b));
  return o + 5;
}

__device__ __forceinline__ uint8_t* put_key(uint8_t* o, const char* s, int len) {
  o[0] = 'X'; o[1] = (uint8_t)len; o[2] = 0; o[3] = 0; o[4] = 0;
  for (int i = 0; i < len; ++i) o[5 + i] = (uint8_t)s[i];
  return o + 5 + len;
}

__device__ __forceinline__ void put_binfloat(uint8_t* o, double v) {
  const unsigned long long u = (unsigned long long)__double_as_longlong(v);
  o[0] = 'G';
  for (int b = 0; b < 8; ++b) o[1 + b] = (uint8_t)(u >> (56 - 8 * b));
}

// one thread per record: its byte count
__global__ void k_record_bytes(long long T, const long long* ids, const long long* ptr, const int* frames, long long* bytes) {
  const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= T) return;
  const long long s = ptr[k], e = ptr[k + 1];
  long long n = int_width(ids[k]) + kFixed + (e - s) * (kLocation + kLabel);
  for (long long j = s; j < e; ++j) n += int_width(frames[j]);
  bytes[k] = n;
}

// one warp per record, at body offset 2 + off[k]
__global__ void k_write_records(long long T, const long long* ids, const long long* ptr, const int* frames, const double* xy,
                                const long long* off, uint8_t* body) {
  const long long k = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (k >= T) return;
  const long long s = ptr[k], L = ptr[k + 1] - s;
  uint8_t* o = body + 2 + off[k];
  uint8_t* p = o;
  if (lane == 0) {
    p = put_int(p, ids[k]);
    p[0] = '}'; p[1] = '(';
    p = put_key(p + 2, "frame_ids", 9);
    p[0] = ']'; p[1] = '(';
  }
  const int idw = int_width(ids[k]);
  // frame ids: variable widths, placed by a warp scan in chunks of 32
  uint8_t* fbase = o + idw + kHeadFrames;
  long long run = 0;
  for (long long c = 0; c < L; c += 32) {
    const long long j = c + lane;
    const int f = j < L ? frames[s + j] : 0;
    const int wdt = j < L ? int_width(f) : 0;
    int incl = wdt;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += v;
    }
    if (j < L) put_int(fbase + run + incl - wdt, f);
    run += __shfl_sync(0xffffffffu, incl, 31);
  }
  uint8_t* lhead = fbase + run;
  uint8_t* lbase = lhead + kHeadLocations;
  uint8_t* bhead = lbase + L * kLocation;
  uint8_t* bbase = bhead + kHeadLabels;
  if (lane == 0) {
    lhead[0] = 'e';
    p = put_key(lhead + 1, "locations", 9);
    p[0] = ']'; p[1] = '(';
    bhead[0] = 'e';
    p = put_key(bhead + 1, "labels", 6);
    p[0] = ']'; p[1] = '(';
    bbase[L] = 'e'; bbase[L + 1] = 'u';
  }
  for (long long j = lane; j < L; j += 32) {
    uint8_t* q = lbase + j * kLocation;
    put_binfloat(q, xy[2 * (s + j)]);
    put_binfloat(q + 9, xy[2 * (s + j) + 1]);
    q[18] = 0x86;
    bbase[j] = 0x89;
  }
}

__global__ void k_body_frame(long long T, long long total, uint8_t* body) {
  body[0] = '}';
  if (T) { body[1] = '('; body[2 + total] = 'u'; }
}

}  // namespace

namespace psfm {

void track_npy_encode(const long long* ids, const long long* ptr, const int* frames, const double* xy, long long T,
                      cudaStream_t st, psfm_track_npy** out, int64_t* nbytes) {
  std::unique_ptr<psfm_track_npy, decltype(&psfm_track_npy_destroy)> R(new psfm_track_npy, psfm_track_npy_destroy);
  DBuf<long long> bytes, off;
  DBuf<uint8_t> tmp, body;
  long long sum = 0;
  if (T) {
    bytes.alloc(T, st); off.alloc(T, st);
    k_record_bytes<<<grid_of(T), 256, 0, st>>>(T, ids, ptr, frames, bytes.p);
    PSFM_LAUNCH_CHECK();
    size_t tb = 0;
    PSFM_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, bytes.p, off.p, T, st));
    tmp.alloc(tb, st);
    PSFM_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, tb, bytes.p, off.p, T, st));
    PSFM_LAUNCH_CHECK();
    long long last[2];
    PSFM_CUDA(cudaMemcpyAsync(&last[0], off.p + T - 1, sizeof(long long), cudaMemcpyDeviceToHost, st));
    PSFM_CUDA(cudaMemcpyAsync(&last[1], bytes.p + T - 1, sizeof(long long), cudaMemcpyDeviceToHost, st));
    PSFM_CUDA(cudaStreamSynchronize(st));
    sum = last[0] + last[1];
  }
  R->bytes = T ? 3 + sum : 1;
  body.alloc((size_t)R->bytes, st);
  k_body_frame<<<1, 1, 0, st>>>(T, sum, body.p);
  PSFM_LAUNCH_CHECK();
  if (T) {
    k_write_records<<<grid_of(32 * T), 256, 0, st>>>(T, ids, ptr, frames, xy, off.p, body.p);
    PSFM_LAUNCH_CHECK();
  }
  PSFM_CUDA(cudaMallocHost((void**)&R->host, (size_t)R->bytes));
  PSFM_CUDA(cudaMemcpyAsync(R->host, body.p, (size_t)R->bytes, cudaMemcpyDeviceToHost, st));
  PSFM_CUDA(cudaStreamSynchronize(st));
  *nbytes = R->bytes;
  *out = R.release();
}

}  // namespace psfm

extern "C" int psfm_track_npy_create(const int64_t* ids, const int64_t* ptr, const int32_t* frame_ids, const double* xy,
                                     int64_t num_trajs, int64_t num_obs, psfm_track_npy** out, int64_t* nbytes) {
  const char* entry = "psfm_track_npy_create";
  return guard(entry, [&]() -> int {
    if (!out || !nbytes) return fail(entry, PSFM_ERR_INVALID, "null argument");
    *out = nullptr;
    *nbytes = 0;
    if (num_trajs < 0 || num_obs < 0 || !ptr) return fail(entry, PSFM_ERR_INVALID, "bad sizes");
    if ((num_trajs && !ids) || (num_obs && (!frame_ids || !xy))) return fail(entry, PSFM_ERR_INVALID, "null argument");
    // every check before the device sees a byte: the kernels index with ptr and trust the widths
    if (ptr[0] != 0 || ptr[num_trajs] != num_obs) return fail(entry, PSFM_ERR_INVALID, "ptr must run from 0 to num_obs");
    for (int64_t k = 0; k < num_trajs; ++k) {
      if (ptr[k + 1] < ptr[k]) return fail(entry, PSFM_ERR_INVALID, "ptr is not monotone at trajectory " + std::to_string(k));
      if (ids[k] < 0 || ids[k] > INT32_MAX) return fail(entry, PSFM_ERR_INVALID, "trajectory id outside [0, 2^31): " + std::to_string(ids[k]));
    }
    for (int64_t j = 0; j < num_obs; ++j)
      if (frame_ids[j] < 0) return fail(entry, PSFM_ERR_INVALID, "negative frame id at observation " + std::to_string(j));
    int rc = require_device(entry);
    if (rc != PSFM_OK) return rc;
    DBuf<long long> dids, dptr; DBuf<int> dfr; DBuf<double> dxy;
    dids.alloc(num_trajs); dptr.alloc(num_trajs + 1); dfr.alloc(num_obs); dxy.alloc(2 * num_obs);
    dids.upload((const long long*)ids, num_trajs, nullptr);
    dptr.upload((const long long*)ptr, num_trajs + 1, nullptr);
    dfr.upload(frame_ids, num_obs, nullptr);
    dxy.upload(xy, 2 * num_obs, nullptr);
    track_npy_encode(dids.p, dptr.p, dfr.p, dxy.p, num_trajs, nullptr, out, nbytes);
    return PSFM_OK;
  });
}

extern "C" const uint8_t* psfm_track_npy_data(const psfm_track_npy* h) { return h ? h->host : nullptr; }

extern "C" void psfm_track_npy_destroy(psfm_track_npy* h) {
  if (!h) return;
  if (h->host) cudaFreeHost(h->host);
  delete h;
  cudaGetLastError();
}
