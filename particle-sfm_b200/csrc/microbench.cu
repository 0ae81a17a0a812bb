// microbench.cu — measured fp64 roof of the device this library runs on.
//
// An optional MEASURED_PEAKS.json carries an HBM copy bandwidth and a bf16 tensor rate; the
// kernels of this library compute in fp64 (the reference is Ceres: double everywhere), and the
// ones that are not HBM-bound (the Schur-complement pair products, the band factorisation) are
// bounded by the fp64 FMA pipe.  bench.py reports their roofline against THIS measurement:
//   psfm_measure_dfma: sustained DFMA rate of the whole chip (8 independent chains per thread,
//   every SM full) and the latency of one dependent DFMA (single warp, one chain).
#include "psfm_common.cuh"

namespace {

__global__ void __launch_bounds__(256) k_fp64_rate(double* out, int iters, double seed) {
  double a0 = seed + threadIdx.x, a1 = a0 + 1, a2 = a0 + 2, a3 = a0 + 3, a4 = a0 + 4, a5 = a0 + 5, a6 = a0 + 6, a7 = a0 + 7;
  const double m = 1.0 - 1e-9, c = 1e-9;
  for (int i = 0; i < iters; ++i) {
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      a0 = fma(a0, m, c); a1 = fma(a1, m, c); a2 = fma(a2, m, c); a3 = fma(a3, m, c);
      a4 = fma(a4, m, c); a5 = fma(a5, m, c); a6 = fma(a6, m, c); a7 = fma(a7, m, c);
    }
  }
  const double s = ((a0 + a1) + (a2 + a3)) + ((a4 + a5) + (a6 + a7));
  if (s == 12345.678) out[blockIdx.x * blockDim.x + threadIdx.x] = s;   // keeps the chains alive, never true in practice
}

__global__ void k_fp64_latency(long long* cycles, double* sink, int n, double seed) {
  double a = seed;
  const double m = 1.0 - 1e-9, c = 1e-9;
  const long long t0 = clock64();
  for (int i = 0; i < n; ++i) {
#pragma unroll
    for (int u = 0; u < 16; ++u) a = fma(a, m, c);
  }
  const long long t1 = clock64();
  if (threadIdx.x == 0) { cycles[0] = t1 - t0; sink[0] = a; }
}

}  // namespace

// dfma_per_second: fused multiply-adds per second, whole device (x2 = FLOP/s);
// dependent_latency_cycles: SM cycles from one DFMA to the next dependent one.
extern "C" int psfm_measure_dfma(double* dfma_per_second, double* dependent_latency_cycles) {
  return psfm::guard("psfm_measure_dfma", [&]() -> int {
    using namespace psfm;
    const int rc = require_device("psfm_measure_dfma");
    if (rc != PSFM_OK) return rc;
    int dev = 0, sms = 0;
    PSFM_CUDA(cudaGetDevice(&dev));
    PSFM_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const int grid = sms * 8, iters = 2048;
    DBuf<double> out; out.alloc((size_t)grid * 256);
    DBuf<long long> cyc; cyc.alloc(1);
    cudaEvent_t e0, e1;
    PSFM_CUDA(cudaEventCreate(&e0)); PSFM_CUDA(cudaEventCreate(&e1));
    double best = 0.0;
    for (int rep = 0; rep < 5; ++rep) {
      PSFM_CUDA(cudaEventRecord(e0));
      k_fp64_rate<<<grid, 256>>>(out.p, iters, 0.5 + rep);
      PSFM_LAUNCH_CHECK();
      PSFM_CUDA(cudaEventRecord(e1));
      PSFM_CUDA(cudaEventSynchronize(e1));
      float ms = 0.f;
      PSFM_CUDA(cudaEventElapsedTime(&ms, e0, e1));
      const double rate = (double)grid * 256.0 * iters * 64.0 / (ms * 1e-3);
      if (rep > 0 && rate > best) best = rate;      // first launch = warm-up
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    const int nl = 4096;
    k_fp64_latency<<<1, 32>>>(cyc.p, out.p, nl, 0.25);
    PSFM_LAUNCH_CHECK();
    k_fp64_latency<<<1, 32>>>(cyc.p, out.p, nl, 0.75);
    PSFM_LAUNCH_CHECK();
    long long h = 0;
    PSFM_CUDA(cudaMemcpy(&h, cyc.p, sizeof(h), cudaMemcpyDeviceToHost));
    if (dfma_per_second) *dfma_per_second = best;
    if (dependent_latency_cycles) *dependent_latency_cycles = (double)h / (16.0 * nl);
    return PSFM_OK;
  });
}
