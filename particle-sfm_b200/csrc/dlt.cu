// dlt.cu — psfm_null_vectors, the test entry of dlt.cuh's solvers: one solver call per thread on a batch of matrices,
// its raw outputs back.
#include "dlt.cuh"
#include "psfm_common.cuh"

namespace {

using namespace psfm;

constexpr int kBlock = 128;

__host__ __device__ constexpr int in_size(int form) {
  return form == PSFM_NV_JACOBI_3 || form == PSFM_NV_EIGEN_3 ? 9 : form == PSFM_NV_JACOBI_9 ? 81 : 16;
}
__host__ __device__ constexpr int out_size(int form) {
  return form == PSFM_NV_JACOBI_3 ? 18 : form == PSFM_NV_JACOBI_4 ? 32 : form == PSFM_NV_DLT_POINT ? 7
       : form == PSFM_NV_EIGEN_3 ? 3 : form == PSFM_NV_EIGEN_4 ? 4 : 171;
}

template <int N>
__device__ __forceinline__ void load(const double* a, double (&A)[N][N]) {
#pragma unroll
  for (int r = 0; r < N; ++r)
#pragma unroll
    for (int c = 0; c < N; ++c) A[r][c] = a[N * r + c];
}

template <int FORM>
__global__ void __launch_bounds__(kBlock) k_null_vectors(const double* __restrict__ in, long long count, double* __restrict__ out) {
  const long long t = blockIdx.x * (long long)kBlock + threadIdx.x;
  if (t >= count) return;
  const double* a = in + in_size(FORM) * t;
  double* o = out + out_size(FORM) * t;
  if constexpr (FORM == PSFM_NV_JACOBI_3 || FORM == PSFM_NV_JACOBI_4) {
    constexpr int N = FORM == PSFM_NV_JACOBI_3 ? 3 : 4;
    double A[N][N], V[N][N];
    load<N>(a, A);
    one_sided_jacobi<N>(A, V);
#pragma unroll
    for (int r = 0; r < N; ++r)
#pragma unroll
      for (int c = 0; c < N; ++c) { o[N * r + c] = A[r][c]; o[N * N + N * r + c] = V[r][c]; }
  } else if constexpr (FORM == PSFM_NV_DLT_POINT) {
    double A[4][4], B[4][4], v[4], X[3];
    load<4>(a, A);
    load<4>(a, B);
    dlt_point_4x4(A, X);
    dlt_null_vector_4x4(B, v);
    for (int i = 0; i < 3; ++i) o[i] = X[i];
    for (int i = 0; i < 4; ++i) o[3 + i] = v[i];
  } else if constexpr (FORM == PSFM_NV_EIGEN_3 || FORM == PSFM_NV_EIGEN_4) {
    constexpr int N = FORM == PSFM_NV_EIGEN_3 ? 3 : 4;
    double A[N][N], v[N];
    load<N>(a, A);
    smallest_eigenvector<N>(A, v);
    for (int i = 0; i < N; ++i) o[i] = v[i];
  } else {                                     // the local step's solve, A and V in the output
    for (int i = 0; i < 81; ++i) o[i] = a[i];
    const int best = one_sided_jacobi_mem(o, o + 81, 9);
    for (int i = 0; i < 9; ++i) o[162 + i] = o[81 + 9 * i + best];
  }
}

template <int FORM>
void launch(const double* in, long long count, double* out) {
  k_null_vectors<FORM><<<(unsigned)((count + kBlock - 1) / kBlock), kBlock>>>(in, count, out);
  PSFM_LAUNCH_CHECK();
}

}  // namespace

extern "C" int psfm_null_vectors(int32_t form, const double* A, int64_t count, double* out) {
  const char* entry = "psfm_null_vectors";
  return guard(entry, [&]() -> int {
    if (!A || !out) return fail(entry, PSFM_ERR_INVALID, "null argument");
    if (form < PSFM_NV_JACOBI_3 || form > PSFM_NV_JACOBI_9) return fail(entry, PSFM_ERR_INVALID, "unknown form");
    if (count < 1 || count > (1LL << 24)) return fail(entry, PSFM_ERR_INVALID, "needs 1 <= count <= 2^24");
    const int rc = require_device(entry);
    if (rc != PSFM_OK) return rc;
    const int isz[6] = {in_size(0), in_size(1), in_size(2), in_size(3), in_size(4), in_size(5)};
    const int osz[6] = {out_size(0), out_size(1), out_size(2), out_size(3), out_size(4), out_size(5)};
    DBuf<double> d_in, d_out;
    d_in.alloc((size_t)count * isz[form]); d_out.alloc((size_t)count * osz[form]);
    d_in.upload(A, (size_t)count * isz[form], nullptr);
    switch (form) {
      case PSFM_NV_JACOBI_3: launch<PSFM_NV_JACOBI_3>(d_in.p, count, d_out.p); break;
      case PSFM_NV_JACOBI_4: launch<PSFM_NV_JACOBI_4>(d_in.p, count, d_out.p); break;
      case PSFM_NV_DLT_POINT: launch<PSFM_NV_DLT_POINT>(d_in.p, count, d_out.p); break;
      case PSFM_NV_EIGEN_3: launch<PSFM_NV_EIGEN_3>(d_in.p, count, d_out.p); break;
      case PSFM_NV_EIGEN_4: launch<PSFM_NV_EIGEN_4>(d_in.p, count, d_out.p); break;
      default: launch<PSFM_NV_JACOBI_9>(d_in.p, count, d_out.p); break;
    }
    PSFM_CUDA(cudaMemcpy(out, d_out.p, sizeof(double) * (size_t)count * osz[form], cudaMemcpyDeviceToHost));
    return PSFM_OK;
  });
}
