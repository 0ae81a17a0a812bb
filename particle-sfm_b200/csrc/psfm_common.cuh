// psfm_common.cuh — shared helpers of the sm_90a library (error handling, launch
// accounting, block reductions).  Product code: no CPU path lives here.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <exception>
#include <memory>
#include <new>
#include <string>
#include <thread>
#include <vector>

#include "../../include/psfm_b200.h"

namespace psfm {

void set_error(const std::string& msg);
// sets "<entry>: <msg>" as the last error and returns code
int fail(const char* entry, int code, const std::string& msg);
// PSFM_OK, or PSFM_ERR_NO_DEVICE with "<entry>: no CUDA device available (this library has no CPU path)"
int require_device(const char* entry);
extern std::atomic<long long> g_launch_count;

// blocks of `block` threads covering n items, at least one (a grid of zero blocks fails at launch)
inline unsigned grid_of(long long n, int block = 256) { return (unsigned)std::max<long long>(1, (n + block - 1) / block); }
// the same for grid-stride kernels of 256 threads, capped at 16 blocks per SM of the H100's 132
inline unsigned grid_stride_of(long long n) { return (unsigned)std::max<long long>(1, std::min<long long>((n + 255) / 256, 132 * 16)); }

struct CudaFail {
  int code;
};

inline int same_code(int code) { return code; }

// The exception boundary of a C entry point: returns body()'s status and lets no exception out.  CudaFail returns its
// code (its thrower set the message); any other exception sets "<entry>: <what>" and returns PSFM_ERR_HOST.  Only after
// an exception, on_throw(code) runs and its value is returned (by default the code itself).
template <typename Body, typename OnThrow = int (&)(int)>
auto guard(const char* entry, Body&& body, OnThrow&& on_throw = same_code) -> decltype(body()) {
  int code;
  try {
    return body();
  } catch (const CudaFail& f) {
    code = f.code;
  } catch (const std::bad_alloc&) {
    code = fail(entry, PSFM_ERR_HOST, "out of host memory");
  } catch (const std::exception& e) {
    code = fail(entry, PSFM_ERR_HOST, e.what());
  } catch (...) {
    code = fail(entry, PSFM_ERR_HOST, "unknown host exception");
  }
  return on_throw(code);
}

// Runs fn(0) .. fn(nt - 1), fn(0) on the calling thread and the others on threads of their own.  The calls must be
// independent: when a thread cannot be created, the calling thread runs the remaining calls itself.
template <typename Fn>
void host_fan(unsigned nt, Fn&& fn) {
  std::vector<std::thread> th;
  unsigned w = 1;
  try {
    for (; w < nt; ++w) th.emplace_back([&fn, w] { fn(w); });
  } catch (const std::exception&) {}
  for (; w < nt; ++w) fn(w);
  fn(0);
  for (auto& t : th) t.join();
}

#define PSFM_CUDA(expr)                                                                   \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      ::psfm::set_error(std::string(#expr) + ": " + cudaGetErrorString(_e) + " (" +       \
                        __FILE__ + ":" + std::to_string(__LINE__) + ")");                 \
      throw ::psfm::CudaFail{PSFM_ERR_CUDA};                                              \
    }                                                                                     \
  } while (0)

#define PSFM_LAUNCH_CHECK()                  \
  do {                                       \
    ::psfm::g_launch_count.fetch_add(1);     \
    PSFM_CUDA(cudaGetLastError());           \
  } while (0)

// RAII device buffer.  With a stream: stream-ordered allocation from the default memory
// pool (cudaMallocAsync), whose release threshold psfm::keep_pool_memory() raises so that
// create/destroy cycles of a solver re-use the cached blocks instead of paying cudaMalloc.
void keep_pool_memory();

template <typename T>
struct DBuf {
  T* p = nullptr;
  size_t n = 0;
  cudaStream_t st = nullptr;
  bool async = false;
  DBuf() {}
  DBuf(const DBuf&) = delete;
  DBuf& operator=(const DBuf&) = delete;
  ~DBuf() { release(); }
  void release() {
    if (p) {
      if (async) cudaFreeAsync(p, st);
      else cudaFree(p);
    }
    p = nullptr;
    n = 0;
  }
  void alloc(size_t count, cudaStream_t stream = nullptr) {
    release();
    n = count;
    if (count == 0) count = 1;
    if (stream) {
      keep_pool_memory();
      PSFM_CUDA(cudaMallocAsync((void**)&p, count * sizeof(T) + 64, stream));   // slack: bulk copies read whole 16-byte windows
      st = stream;
      async = true;
    } else {
      PSFM_CUDA(cudaMalloc((void**)&p, count * sizeof(T) + 64));
      async = false;
    }
  }
  void upload(const T* h, size_t count, cudaStream_t s) {
    if (count) PSFM_CUDA(cudaMemcpyAsync(p, h, count * sizeof(T), cudaMemcpyHostToDevice, s));
  }
  void zero(cudaStream_t s) { PSFM_CUDA(cudaMemsetAsync(p, 0, (n ? n : 1) * sizeof(T), s)); }
};

// RAII CUDA event (timing enabled) that converts to cudaEvent_t; construction throws CudaFail like PSFM_CUDA
struct Event {
  cudaEvent_t e = nullptr;
  Event() { PSFM_CUDA(cudaEventCreate(&e)); }
  Event(const Event&) = delete;
  Event& operator=(const Event&) = delete;
  ~Event() {
    if (e) cudaEventDestroy(e);
  }
  operator cudaEvent_t() const { return e; }
};

#ifdef __CUDACC__
// ---- warp / block reductions (sum and max), result valid in thread 0 ----
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// sbuf: at least 32 doubles of shared memory; all threads of the block must call.
__device__ __forceinline__ double block_sum(double v, double* sbuf) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) sbuf[wid] = v;
  __syncthreads();
  if (wid == 0) {
    v = (lane < nw) ? sbuf[lane] : 0.0;
    v = warp_sum(v);
  }
  return v;
}
__device__ __forceinline__ double block_max(double v, double* sbuf) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) sbuf[wid] = v;
  __syncthreads();
  if (wid == 0) {
    v = (lane < nw) ? sbuf[lane] : 0.0;
    v = warp_max(v);
  }
  return v;
}
// max of non-negative doubles through their bit pattern (monotone for x >= 0)
__device__ __forceinline__ void atomic_max_nonneg(double* addr, double v) {
  atomicMax((unsigned long long*)addr, (unsigned long long)__double_as_longlong(v));
}
#endif

}  // namespace psfm
