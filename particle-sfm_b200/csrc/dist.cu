// dist.cu — see dist.cuh.  The reference has no multi-GPU code at all (SURVEY.md §2.2);
// this is new design: psfm_dist_get_unique_id / psfm_dist_init build a private NCCL
// communicator (the id bytes travel through the caller's torch.distributed group).
#include "dist.cuh"

#include <dlfcn.h>

#include <algorithm>
#include <cstdlib>
#include <vector>

#include "psfm_common.cuh"

namespace psfm {
namespace dist {

// minimal NCCL ABI (nccl.h 2.27): opaque comm, 128-byte id, enums
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
enum { ncclSuccess = 0 };
enum { ncclSum = 0, ncclProd = 1, ncclMax = 2, ncclMin = 3 };
enum { ncclInt64 = 4, ncclFloat64 = 8 };

static struct {
  void* handle = nullptr;
  int (*GetUniqueId)(ncclUniqueId*) = nullptr;
  int (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*CommDestroy)(ncclComm_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  ncclComm_t comm = nullptr;
  int world = 1, rank = 0;
} g;

static bool load_nccl() {
  if (g.handle) return true;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  for (const char* n : names) {
    g.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (g.handle) break;
  }
  if (!g.handle) {
    set_error(std::string("cannot dlopen libnccl.so.2: ") + dlerror());
    return false;
  }
  g.GetUniqueId = (int (*)(ncclUniqueId*))dlsym(g.handle, "ncclGetUniqueId");
  g.CommInitRank = (int (*)(ncclComm_t*, int, ncclUniqueId, int))dlsym(g.handle, "ncclCommInitRank");
  g.AllReduce = (int (*)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t))dlsym(g.handle, "ncclAllReduce");
  g.CommDestroy = (int (*)(ncclComm_t))dlsym(g.handle, "ncclCommDestroy");
  g.GetErrorString = (const char* (*)(int))dlsym(g.handle, "ncclGetErrorString");
  if (!g.GetUniqueId || !g.CommInitRank || !g.AllReduce || !g.CommDestroy) {
    set_error("libnccl.so.2 lacks a required symbol");
    return false;
  }
  return true;
}

int world_size() { return g.world; }
int rank() { return g.rank; }

// ------------------------------------------------------------------ peer-memory all-reduce (one node, NVLink / NVSwitch)
//
// The collectives of an LM iteration are tiny (4 doubles ... 0.8 MB) and latency-bound: NCCL costs
// 15-30 us per call at 8 ranks.  On one NVSwitch node every rank can LOAD every peer's buffer directly:
// each rank owns a symmetric buffer (cudaMalloc, exported with cudaIpcGetMemHandle, the handles exchanged
// once through the NCCL communicator) and a flag array.  k_p2p_allreduce copies the local operand into the
// rank's symmetric buffer (parity = epoch & 1) and, when the last CTA is done, stores the epoch into
// flags[my_rank] of EVERY peer (system-scope release over NVLink); it then waits until all its own
// flags reach the epoch (acquire) and every rank sums (or max-es) the world's buffers in rank order —
// the same order on every rank, so the replicated results are bit-identical across ranks — and writes
// the result over the local operand.  Two parities make the buffer of epoch k safe to overwrite in epoch
// k+2: passing the barrier of epoch k+1 means every peer has finished reading epoch k.  A wait that
// exceeds ~60 s sets the error flag (no hang on a dead peer).  Falls back to NCCL when IPC set-up fails or
// PSFM_NO_P2P is set.
constexpr int P2P_MAX_WORLD = 16;
constexpr size_t P2P_BYTES = (size_t)8 << 20;       // per parity; operands above this go through NCCL

struct P2P {
  bool ready = false, tried = false;
  double* sym_local = nullptr;                       // [2][P2P_BYTES / 8]
  unsigned long long* flags_local = nullptr;         // [P2P_MAX_WORLD] + [1] publish counter + [1] error
  double* sym[P2P_MAX_WORLD] = {};
  unsigned long long* flags[P2P_MAX_WORLD] = {};
  unsigned long long epoch = 0;
};
static P2P p2p;

struct P2PPtrs {
  double* sym[P2P_MAX_WORLD];
  unsigned long long* flags[P2P_MAX_WORLD];
};

// ONE kernel per all-reduce (a launch costs as much as the whole exchange at this size): every block copies its share
// of the operand into the symmetric buffer; the block that finishes last raises this rank's flag on every peer
// (system-scope release over NVLink); then every block waits until all ranks — its own included, so the in-place
// result never overwrites an operand a sibling block is still copying — have raised theirs, and reduces in rank order.
// The grid (P2P_GRID blocks) is far below one wave, so the spinning blocks cannot starve the publishing ones.
constexpr int P2P_GRID = 32;
__global__ void __launch_bounds__(256) k_p2p_allreduce(double* __restrict__ buf, size_t n, size_t parity_off, P2PPtrs pp, int me, int world,
                                                       unsigned long long epoch, int op_max, unsigned long long* counter,
                                                       unsigned long long* err) {
  double* dst = pp.sym[me] + parity_off;
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (size_t)gridDim.x * 256) dst[i] = buf[i];
  __threadfence_system();
  __syncthreads();
  __shared__ bool last;
  if (threadIdx.x == 0) last = atomicAdd(counter, 1ull) == (unsigned long long)gridDim.x * epoch - 1;   // counter is monotone
  __syncthreads();
  if (last && threadIdx.x < world) {
    __threadfence_system();
    unsigned long long* f = pp.flags[threadIdx.x] + me;
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(f), "l"(epoch) : "memory");
  }
  if (threadIdx.x < world) {
    const unsigned long long* f = pp.flags[me] + threadIdx.x;
    unsigned long long v = 0;
    const long long t0 = clock64();
    for (;;) {
      asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(f) : "memory");
      if (v >= epoch) break;
      if (clock64() - t0 > 120000000000ll) { atomicExch(err, 1ull); break; }   // ~60 s: a peer never arrived (ranks may be seconds apart)
    }
  }
  __syncthreads();
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (size_t)gridDim.x * 256) {
    double acc = __ldcg(pp.sym[0] + parity_off + i);           // L2 / NVLink, never a stale L1 line
    for (int r = 1; r < world; ++r) {
      const double v = __ldcg(pp.sym[r] + parity_off + i);
      acc = op_max ? fmax(acc, v) : acc + v;
    }
    buf[i] = acc;
  }
}

// one-time set-up: symmetric buffers + flags, IPC handles exchanged through NCCL (bit-exact int64 sum of
// one-hot slots); returns false (and stays on NCCL) on any failure
static bool p2p_setup(cudaStream_t stream) {
  if (p2p.tried) return p2p.ready;
  p2p.tried = true;
  if (getenv("PSFM_NO_P2P") || g.world > P2P_MAX_WORLD) return false;
  const int W = g.world;
  if (cudaMalloc((void**)&p2p.sym_local, 2 * P2P_BYTES) != cudaSuccess) { cudaGetLastError(); return false; }
  if (cudaMalloc((void**)&p2p.flags_local, sizeof(unsigned long long) * (P2P_MAX_WORLD + 2)) != cudaSuccess) { cudaGetLastError(); return false; }
  cudaMemset(p2p.flags_local, 0, sizeof(unsigned long long) * (P2P_MAX_WORLD + 2));
  cudaMemset(p2p.sym_local, 0, 2 * P2P_BYTES);
  struct Slot { cudaIpcMemHandle_t sym, flags; };          // 128 bytes
  static_assert(sizeof(Slot) == 128, "two 64-byte IPC handles");
  Slot mine;
  bool ok = cudaIpcGetMemHandle(&mine.sym, p2p.sym_local) == cudaSuccess && cudaIpcGetMemHandle(&mine.flags, p2p.flags_local) == cudaSuccess;
  if (!ok) cudaGetLastError();
  std::vector<Slot> all((size_t)W + 1);
  memset(all.data(), 0, sizeof(Slot) * ((size_t)W + 1));
  if (ok) all[g.rank] = mine;
  long long okflag = ok ? 0 : 1;
  memcpy(&all[W], &okflag, sizeof(okflag));                // last slot: number of ranks that failed
  void* d = nullptr;
  if (cudaMalloc(&d, sizeof(Slot) * ((size_t)W + 1)) != cudaSuccess) { cudaGetLastError(); return false; }
  cudaMemcpyAsync(d, all.data(), sizeof(Slot) * ((size_t)W + 1), cudaMemcpyHostToDevice, stream);
  const int rc = g.AllReduce(d, d, sizeof(Slot) * ((size_t)W + 1) / 8, ncclInt64, ncclSum, g.comm, stream);
  cudaMemcpyAsync(all.data(), d, sizeof(Slot) * ((size_t)W + 1), cudaMemcpyDeviceToHost, stream);
  cudaStreamSynchronize(stream);
  cudaFree(d);
  long long failed = 0;
  memcpy(&failed, &all[W], sizeof(failed));
  if (rc != ncclSuccess || failed != 0) return false;      // same verdict on every rank
  bool open_ok = true;
  for (int r = 0; r < W; ++r) {
    if (r == g.rank) { p2p.sym[r] = p2p.sym_local; p2p.flags[r] = p2p.flags_local; continue; }
    void *a = nullptr, *b = nullptr;
    if (cudaIpcOpenMemHandle(&a, all[r].sym, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess ||
        cudaIpcOpenMemHandle(&b, all[r].flags, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); open_ok = false; break; }
    p2p.sym[r] = (double*)a; p2p.flags[r] = (unsigned long long*)b;
  }
  // every rank must agree before anybody relies on peer loads
  long long bad = open_ok ? 0 : 1;
  void* dflag = nullptr;
  cudaMalloc(&dflag, 8);
  cudaMemcpyAsync(dflag, &bad, 8, cudaMemcpyHostToDevice, stream);
  g.AllReduce(dflag, dflag, 1, ncclInt64, ncclSum, g.comm, stream);
  cudaMemcpyAsync(&bad, dflag, 8, cudaMemcpyDeviceToHost, stream);
  cudaStreamSynchronize(stream);
  cudaFree(dflag);
  p2p.ready = bad == 0;
  return p2p.ready;
}

static bool p2p_allreduce(double* buf, size_t n, int op_max, cudaStream_t stream) {
  if (n * sizeof(double) > P2P_BYTES) return false;
  if (!p2p_setup(stream)) return false;
  const unsigned long long epoch = ++p2p.epoch;
  const size_t off = (epoch & 1) * (P2P_BYTES / sizeof(double));
  P2PPtrs pp;
  for (int r = 0; r < P2P_MAX_WORLD; ++r) { pp.sym[r] = p2p.sym[r]; pp.flags[r] = p2p.flags[r]; }
  // fixed grid: the publish counter advances by P2P_GRID per epoch on every call
  k_p2p_allreduce<<<P2P_GRID, 256, 0, stream>>>(buf, n, off, pp, g.rank, g.world, epoch, op_max, p2p.flags_local + P2P_MAX_WORLD,
                                                p2p.flags_local + P2P_MAX_WORLD + 1);
  g_launch_count.fetch_add(1);
  return cudaGetLastError() == cudaSuccess;
}

static void check(int rc, const char* what) {
  if (rc != ncclSuccess) {
    set_error(std::string(what) + ": " + (g.GetErrorString ? g.GetErrorString(rc) : "nccl error"));
    throw CudaFail{PSFM_ERR_NCCL};
  }
}

void allreduce_sum(double* buf, size_t n, cudaStream_t stream) {
  if (g.world <= 1 || n == 0) return;
  if (p2p_allreduce(buf, n, 0, stream)) return;
  check(g.AllReduce(buf, buf, n, ncclFloat64, ncclSum, g.comm, stream), "ncclAllReduce(sum)");
}
void allreduce_max(double* buf, size_t n, cudaStream_t stream) {
  if (g.world <= 1 || n == 0) return;
  if (p2p_allreduce(buf, n, 1, stream)) return;
  check(g.AllReduce(buf, buf, n, ncclFloat64, ncclMax, g.comm, stream), "ncclAllReduce(max)");
}

}  // namespace dist
}  // namespace psfm

using namespace psfm;

extern "C" int psfm_dist_get_unique_id(uint8_t id[PSFM_NCCL_UNIQUE_ID_BYTES]) {
  return guard("psfm_dist_get_unique_id", [&]() -> int {
    if (!dist::load_nccl()) return PSFM_ERR_NCCL;
    dist::ncclUniqueId u;
    if (dist::g.GetUniqueId(&u) != dist::ncclSuccess) { set_error("ncclGetUniqueId failed"); return PSFM_ERR_NCCL; }
    memcpy(id, u.internal, PSFM_NCCL_UNIQUE_ID_BYTES);
    return PSFM_OK;
  });
}

extern "C" int psfm_dist_init(const uint8_t id[PSFM_NCCL_UNIQUE_ID_BYTES], int32_t rank, int32_t world_size) {
  return guard("psfm_dist_init", [&]() -> int {
    if (world_size < 1 || rank < 0 || rank >= world_size) { set_error("psfm_dist_init: bad rank/world"); return PSFM_ERR_INVALID; }
    if (dist::g.comm) { set_error("psfm_dist_init: already initialised"); return PSFM_ERR_INVALID; }
    if (world_size == 1) { dist::g.world = 1; dist::g.rank = 0; return PSFM_OK; }
    if (!dist::load_nccl()) return PSFM_ERR_NCCL;
    dist::ncclUniqueId u;
    memcpy(u.internal, id, PSFM_NCCL_UNIQUE_ID_BYTES);
    const int rc = dist::g.CommInitRank(&dist::g.comm, world_size, u, rank);
    if (rc != dist::ncclSuccess) {
      set_error(std::string("ncclCommInitRank: ") + (dist::g.GetErrorString ? dist::g.GetErrorString(rc) : "error"));
      dist::g.comm = nullptr;
      return PSFM_ERR_NCCL;
    }
    dist::g.world = world_size;
    dist::g.rank = rank;
    return PSFM_OK;
  });
}

extern "C" int psfm_dist_world_size(void) { return dist::g.world; }
extern "C" int psfm_dist_rank(void) { return dist::g.rank; }
extern "C" void psfm_dist_finalize(void) {
  {
    cudaDeviceSynchronize();
    if (dist::p2p.ready && dist::g.comm) {
      // nobody unmaps / frees a symmetric buffer while a peer's last reduce kernel may still read it
      void* d = nullptr;
      if (cudaMalloc(&d, 8) == cudaSuccess) {
        cudaMemset(d, 0, 8);
        dist::g.AllReduce(d, d, 1, dist::ncclInt64, dist::ncclSum, dist::g.comm, nullptr);
        cudaDeviceSynchronize();
        cudaFree(d);
      }
      unsigned long long err = 0;
      cudaMemcpy(&err, dist::p2p.flags_local + dist::P2P_MAX_WORLD + 1, sizeof(err), cudaMemcpyDeviceToHost);
      if (err) fprintf(stderr, "[psfm dist] a peer-memory all-reduce timed out waiting for a peer (results of that solve are invalid)\n");
    }
    for (int r = 0; r < dist::P2P_MAX_WORLD; ++r) {
      if (r != dist::g.rank && dist::p2p.sym[r]) cudaIpcCloseMemHandle(dist::p2p.sym[r]);
      if (r != dist::g.rank && dist::p2p.flags[r]) cudaIpcCloseMemHandle(dist::p2p.flags[r]);
    }
    if (dist::p2p.sym_local) cudaFree(dist::p2p.sym_local);
    if (dist::p2p.flags_local) cudaFree(dist::p2p.flags_local);
    dist::p2p = dist::P2P();
    cudaGetLastError();
  }
  if (dist::g.comm) dist::g.CommDestroy(dist::g.comm);
  dist::g.comm = nullptr;
  dist::g.world = 1;
  dist::g.rank = 0;
}
