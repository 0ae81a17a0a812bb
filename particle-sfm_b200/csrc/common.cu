// common.cu — error text, device selection, launch accounting of the C ABI.
#include "psfm_common.cuh"

namespace psfm {
static thread_local std::string g_error;
std::atomic<long long> g_launch_count{0};
void set_error(const std::string& msg) { g_error = msg; }
int fail(const char* entry, int code, const std::string& msg) {
  set_error(std::string(entry) + ": " + msg);
  return code;
}
int require_device(const char* entry) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
    cudaGetLastError();
    return fail(entry, PSFM_ERR_NO_DEVICE, "no CUDA device available (this library has no CPU path)");
  }
  return PSFM_OK;
}
void keep_pool_memory() {
  static bool done = false;
  if (done) return;
  int dev = 0;
  cudaMemPool_t pool;
  if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
    unsigned long long thr = ~0ull;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
  }
  done = true;
}
}  // namespace psfm

extern "C" const char* psfm_last_error(void) { return psfm::g_error.c_str(); }
extern "C" int psfm_abi_version(void) { return PSFM_ABI_VERSION; }
extern "C" int psfm_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}
extern "C" int psfm_set_device(int device) {
  return psfm::guard("psfm_set_device", [&]() -> int {
    if (cudaSetDevice(device) != cudaSuccess) {
      psfm::set_error(std::string("cudaSetDevice: ") + cudaGetErrorString(cudaGetLastError()));
      return PSFM_ERR_CUDA;
    }
    return PSFM_OK;
  });
}
extern "C" int64_t psfm_launch_count(void) { return (int64_t)psfm::g_launch_count.load(); }
