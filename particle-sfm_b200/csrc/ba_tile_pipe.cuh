// ba_tile_pipe.cuh — persistent, software-pipelined form of the tile kernels.
//
// The one-CTA-per-tile kernels of ba_kernels.cuh pay three dependent global-memory latencies
// per tile (tile header -> segment / point lists -> poses) before any arithmetic starts, and
// only 2-3 CTAs fit on an SM to hide them.  Here a CTA is PERSISTENT (grid = SMs x resident
// CTAs) and walks tiles blockIdx.x, blockIdx.x + gridDim.x, ...; every input of tile k+1 travels
// global -> shared as BULK copies (cp.async.bulk, the TMA engine; completion on an mbarrier) into
// the second stage of a two-stage shared-memory buffer while tile k is being computed, and the
// 32-byte header of tile k+2 rides along.  All inputs are single-level contiguous ranges addressed
// from the header alone: the per-segment pose rows are gathered once per linearisation into
// seg_pose by k_seg_pose, the point ranges / segment offsets are stored tile-relative.
//
// Round 1 staged with per-thread cp.async (LDGSTS): ~12 copies per thread and tile, each with its
// 64-bit address arithmetic, loop control and (for the per-point rows) an integer division — the
// ncu source view of the Jacobian sweep showed half of its 1040 instructions per observation in
// that code.  Now ONE warp issues the whole tile: lane j owns copy j (a descriptor built once per
// CTA: global base incl. the SoA row offset, element size, which of {observation, point, segment}
// range it follows, destination offset in the stage), so a tile costs ~45 warp instructions of
// staging instead of ~350 per thread.  A bulk copy needs 16-byte aligned source, destination and
// size: every range is widened to the enclosing 16-byte window; the `lead` (bytes in front of the
// first wanted element) is a function of (base, pt0, cs0) that the consumers recompute.
#pragma once
#include "ba_kernels.cuh"

namespace psfm {
namespace ba {

// ---- mbarrier / bulk-copy primitives (PTX ISA 8.x, sm_90+)
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra.uni WAIT_DONE;\n"
      "bra.uni WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(unsigned dst_smem, const void* src, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(dst_smem), "l"(src),
               "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// Global arrays in pipeline form (built once per problem, seg_pose once per linearisation).  Every array is
// 16-byte aligned at its base and may be over-read by up to 15 bytes at its end (DBuf allocates the slack).
struct PipeSrc {
  const int4* tile_hdr;             // [T][2]  {base, n, pt0, np} {cs0, ns, 0, 0}
  const unsigned short* obs_lseg;   // [M]
  const unsigned short* obs_lpt;    // [M]
  const unsigned short* tile_perm;  // [M]
  const int* pstart_rel;            // [P]     first observation of the point, relative to its tile
  const int* cseg_img;              // [nseg]
  const int* cseg_off32;            // [nseg]  start of the segment in the tile's image order
  const double* seg_pose;           // [nseg][PSFM_SPS]  R (9) | t (3) | pad of the segment's image
  // what the kernel wants staged besides the structure
  const double2* obs_xy;            // [M] or null (16-byte records: the image coordinates, or the residual pairs)
  const double* obs_a;             // [3][M] or null
  const double* X;                  // [3P]
  const double* p6;                 // [6][P] or null   -> spt rows 3..8
  const double* p3a;                // [3][P] or null   -> spt rows 9..11
  const double* p3b;                // [3][P] or null   -> spt rows 12..14
};

// gather pose16 rows per tile segment (after k_pose_table)
__global__ void k_seg_pose(const int* __restrict__ cseg_img, const double* __restrict__ pose16, int nseg,
                           double* __restrict__ seg_pose) {
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (size_t)nseg * 12) return;
  const int s = (int)(t / 12), k = (int)(t % 12);
  seg_pose[(size_t)s * PSFM_SPS + k] = pose16[16 * (size_t)cseg_img[s] + k];
}

// tile-relative structure arrays
__global__ void k_pipe_headers(const int* tile_start, const int* tile_pt, const int* cseg_ptr, int T, int4* hdr) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  hdr[2 * t] = make_int4(tile_start[t], tile_start[t + 1] - tile_start[t], tile_pt[t], tile_pt[t + 1] - tile_pt[t]);
  hdr[2 * t + 1] = make_int4(cseg_ptr[t], cseg_ptr[t + 1] - cseg_ptr[t], 0, 0);
}
__global__ void k_pipe_pstart(const int* tile_start, const int* tile_pt, const int* pt_ptr, int T, int* pstart_rel) {
  const int t = blockIdx.x;
  const int base = tile_start[t], p0 = tile_pt[t], p1 = tile_pt[t + 1];
  for (int p = p0 + threadIdx.x; p < p1; p += blockDim.x) pstart_rel[p] = pt_ptr[p] - base;
}
__global__ void k_pipe_off32(const unsigned short* cseg_off, int nseg, int* off32) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s < nseg) off32[s] = cseg_off[s];
}

// One shared-memory stage: everything a tile reads that comes from global memory.  Region offsets (bytes, all
// multiples of 16) are the same for both stages; the pointers below already include the tile's leads.
template <int TILE>
struct PipeLayout {
  int o_xy, o_a, o_simg, o_xyz, o_spt, o_pstart, o_coff, o_cimg, o_lseg, o_lpt, o_perm, bytes;
  int pstr;          // doubles per spt row (even, >= cap_np + 2)
  __host__ __device__ static int r16(int b) { return (b + 15) & ~15; }
  __host__ __device__ PipeLayout(bool has_xy, bool has_a, int npt, int cns, int cnp) {
    int b = 0;
    o_xy = b; if (has_xy) b += 16 * TILE;
    o_a = b; if (has_a) b += 3 * 8 * (TILE + 2);
    o_simg = b; b += r16(8 * PSFM_SPS * cns);
    o_xyz = b; b += r16(8 * (3 * cnp + 2));
    pstr = (cnp + 3) & ~1;
    o_spt = b; b += (npt > 3 ? npt - 3 : 0) * 8 * pstr;
    o_pstart = b; b += 4 * ((cnp + 8) & ~3);
    o_coff = b; b += 4 * ((cns + 8) & ~3);
    o_cimg = b; b += 4 * ((cns + 8) & ~3);
    o_lseg = b; b += 2 * (TILE + 16);
    o_lpt = b; b += 2 * (TILE + 16);
    o_perm = b; b += 2 * (TILE + 16);
    bytes = r16(b);
  }
};

template <int TILE>
struct PipeStage {
  const double2* xy;            // [TILE]
  const double *a0, *a1, *a2;   // [TILE] each
  double* simg;                 // [cap_ns][PSFM_SPS]
  double* sxyz;                 // [np][3]
  double* spt;                  // row r (>= 3) at spt + r * pstr (+ lead: TileSmem::prow)
  int *pstart, *coff, *cimg;
  const unsigned short *lseg, *lpt, *perm;
  int pstr, plead0, plead1;
  static __host__ __device__ size_t bytes(bool has_xy, bool has_a, int npt, int cns, int cnp) {
    return (size_t)PipeLayout<TILE>(has_xy, has_a, npt, cns, cnp).bytes;
  }
  // mpar / ppar: parity of M and P (SoA row k of an [.][M] array starts at element k * M)
  __device__ __forceinline__ void view(unsigned char* sb, const PipeLayout<TILE>& L, int base, int pt0, int cs0, int mpar, int ppar) {
    xy = reinterpret_cast<const double2*>(sb + L.o_xy);
    const double* ab = reinterpret_cast<const double*>(sb + L.o_a);
    a0 = ab + (base & 1);
    a1 = ab + (TILE + 2) + ((base + mpar) & 1);
    a2 = ab + 2 * (TILE + 2) + (base & 1);
    simg = reinterpret_cast<double*>(sb + L.o_simg);
    sxyz = reinterpret_cast<double*>(sb + L.o_xyz) + (pt0 & 1);
    spt = reinterpret_cast<double*>(sb + L.o_spt) - 3 * (size_t)L.pstr;      // rows are numbered from 3
    pstr = L.pstr; plead0 = pt0 & 1; plead1 = (pt0 + ppar) & 1;
    pstart = reinterpret_cast<int*>(sb + L.o_pstart) + (pt0 & 3);
    coff = reinterpret_cast<int*>(sb + L.o_coff) + (cs0 & 3);
    cimg = reinterpret_cast<int*>(sb + L.o_cimg) + (cs0 & 3);
    lseg = reinterpret_cast<const unsigned short*>(sb + L.o_lseg) + (base & 7);
    lpt = reinterpret_cast<const unsigned short*>(sb + L.o_lpt) + (base & 7);
    perm = reinterpret_cast<const unsigned short*>(sb + L.o_perm) + (base & 7);
  }
};

// Copy descriptor of one lane of the issuing warp (registers, built once per CTA)
struct PipeDesc {
  const unsigned char* g;   // global base (incl. the SoA row offset); null: this lane copies nothing
  int esz;                  // bytes per element
  int kind;                 // 0: observation range (base, n)  1: point range (pt0, np)  2: segment range (cs0, ns)  3: tile header
  int mul;                  // elements per range unit (3 for X: three doubles per point)
  int dst;                  // byte offset in the stage
};

template <int TILE>
__device__ __forceinline__ PipeDesc pipe_desc(const TileCtx& tc, const PipeSrc& ps, const PipeLayout<TILE>& L, int lane) {
  PipeDesc d;
  d.g = nullptr; d.esz = 0; d.kind = 0; d.mul = 1; d.dst = 0;
  const size_t M = (size_t)tc.M, P = (size_t)tc.P;
  auto set = [&](const void* g, int esz, int kind, int mul, int dst) { d.g = reinterpret_cast<const unsigned char*>(g); d.esz = esz; d.kind = kind; d.mul = mul; d.dst = dst; };
  if (lane == 0) { if (ps.obs_xy) set(ps.obs_xy, 16, 0, 1, L.o_xy); }
  else if (lane <= 3) { if (ps.obs_a) set(ps.obs_a + (size_t)(lane - 1) * M, 8, 0, 1, L.o_a + (lane - 1) * 8 * (TILE + 2)); }
  else if (lane == 4) set(ps.obs_lseg, 2, 0, 1, L.o_lseg);
  else if (lane == 5) set(ps.obs_lpt, 2, 0, 1, L.o_lpt);
  else if (lane == 6) set(ps.tile_perm, 2, 0, 1, L.o_perm);
  else if (lane == 7) set(ps.pstart_rel, 4, 1, 1, L.o_pstart);
  else if (lane == 8) set(ps.cseg_off32, 4, 2, 1, L.o_coff);
  else if (lane == 9) set(ps.cseg_img, 4, 2, 1, L.o_cimg);
  else if (lane == 10) set(ps.seg_pose, 8 * PSFM_SPS, 2, 1, L.o_simg);
  else if (lane == 11) set(ps.X, 8, 1, 3, L.o_xyz);
  else if (lane <= 17) { if (ps.p6) set(ps.p6 + (size_t)(lane - 12) * P, 8, 1, 1, L.o_spt + (lane - 12) * 8 * L.pstr); }
  else if (lane <= 20) { if (ps.p3a) set(ps.p3a + (size_t)(lane - 18) * P, 8, 1, 1, L.o_spt + (6 + lane - 18) * 8 * L.pstr); }
  else if (lane <= 23) { if (ps.p3b) set(ps.p3b + (size_t)(lane - 21) * P, 8, 1, 1, L.o_spt + (9 + lane - 21) * 8 * L.pstr); }
  else if (lane == 24) set(ps.tile_hdr, 32, 3, 1, 0);
  return d;
}

// warp 0 issues the bulk copies of one tile (header h0 / h1) into the stage at stage_smem (shared-space address);
// lane 24 fetches the header of tile `hdr_tile` (or nothing when hdr_tile < 0) into hdr_dst
__device__ __forceinline__ void pipe_issue(const PipeDesc d, const int4 h0, const int4 h1, unsigned stage_smem, unsigned hdr_dst,
                                           int hdr_tile, unsigned long long* bar) {
  int start = d.kind == 0 ? h0.x : (d.kind == 1 ? h0.z : (d.kind == 2 ? h1.x : hdr_tile));
  int cnt = d.kind == 0 ? h0.y : (d.kind == 1 ? h0.w : (d.kind == 2 ? h1.y : (hdr_tile >= 0 ? 1 : 0)));
  if (d.g == nullptr) cnt = 0;
  const unsigned char* src = d.g + (size_t)start * d.mul * d.esz;
  const unsigned lead = (unsigned)(reinterpret_cast<uintptr_t>(src) & 15);
  const unsigned bytes = cnt > 0 ? ((lead + (unsigned)(cnt * d.mul * d.esz) + 15u) & ~15u) : 0u;
  const unsigned total = __reduce_add_sync(0xffffffffu, bytes);
  if ((threadIdx.x & 31) == 0) mbar_expect_tx(bar, total);
  __syncwarp();
  if (bytes) bulk_g2s(d.kind == 3 ? hdr_dst : stage_smem + (unsigned)d.dst, src - lead, bytes, bar);
}

// Drives the pipeline.  body(ti, stage, tile) computes one tile from a ready stage; it may
// use barriers and must be called by every thread.  Shared memory that is not staged (reduction
// scratch) is carved by the caller after the two stages.
template <int TILE, typename Body>
__device__ __forceinline__ void pipe_run(const TileCtx& tc, const PipeSrc& ps, unsigned char* stage_base, int4 (*hdr_ring)[2],
                                         unsigned long long* bars, const int npt, const int cns, const int cnp, Body body) {
  const int tid = threadIdx.x;
  int tile = blockIdx.x;
  if (tile >= tc.T) return;
  const bool has_xy = ps.obs_xy != nullptr, has_a = ps.obs_a != nullptr;
  const PipeLayout<TILE> L(has_xy, has_a, npt, cns, cnp);
  const int mpar = tc.M & 1, ppar = tc.P & 1;
  const bool issuer = tid < 32;
  // the descriptors live in shared memory (the pair loop of the Schur kernel has no registers to spare)
  __shared__ PipeDesc sdesc[32];
  if (issuer) sdesc[tid] = pipe_desc<TILE>(tc, ps, L, tid);
  if (tid == 0) { mbar_init(&bars[0], 1); mbar_init(&bars[1], 1); mbar_fence_init(); }
  __syncthreads();
  const unsigned sb0 = smem_u32(stage_base);
  int4 h0 = __ldg(ps.tile_hdr + 2 * (size_t)tile), h1 = __ldg(ps.tile_hdr + 2 * (size_t)tile + 1);
  if (issuer) {
    const int next = tile + gridDim.x;
    pipe_issue(sdesc[tid], h0, h1, sb0, smem_u32(&hdr_ring[1][0]), next < tc.T ? next : -1, &bars[0]);
  }
  for (int it = 0;; ++it) {
    const int cur = it & 1;
    mbar_wait(&bars[cur], (unsigned)((it >> 1) & 1));
    const int ntile = tile + gridDim.x, nntile = ntile + gridDim.x;
    int4 n0 = make_int4(0, 0, 0, 0), n1 = n0;
    if (ntile < tc.T) {
      n0 = hdr_ring[(it + 1) & 3][0];
      n1 = hdr_ring[(it + 1) & 3][1];
      if (issuer)
        pipe_issue(sdesc[tid], n0, n1, sb0 + (unsigned)((cur ^ 1) * L.bytes), smem_u32(&hdr_ring[(it + 2) & 3][0]), nntile < tc.T ? nntile : -1,
                   &bars[cur ^ 1]);
    }
    TileInfo ti;
    ti.base = h0.x; ti.n = h0.y; ti.pt0 = h0.z; ti.np = h0.w; ti.cs0 = h1.x; ti.ns = h1.y;
    PipeStage<TILE> st;
    st.view(stage_base + (size_t)cur * L.bytes, L, ti.base, ti.pt0, ti.cs0, mpar, ppar);
    if (tid == 0) { st.pstart[ti.np] = ti.n; st.coff[ti.ns] = ti.n; }
    body(ti, st, tile);
    __syncthreads();        // everybody is done with this stage before it is refilled (next iteration's issue)
    if (ntile >= tc.T) break;
    tile = ntile; h0 = n0; h1 = n1;
  }
}

// point a TileSmem view at a stage
template <int TILE>
__device__ __forceinline__ void view_stage(TileSmem<TILE>& sm, const PipeStage<TILE>& st) {
  sm.simg = st.simg; sm.spt = st.spt; sm.sxyz = st.sxyz; sm.pstart = st.pstart; sm.coff = st.coff; sm.cimg = st.cimg;
  sm.perm = const_cast<unsigned short*>(st.perm);
  sm.pstr = st.pstr; sm.plead0 = st.plead0; sm.plead1 = st.plead1;
}

// ------------------------------------------------------------------ pipelined Jacobian sweep

template <int TILE, bool ROT>
__global__ void __launch_bounds__(TILE, (TILE == 256 ? 3 : 1)) k_linearize_p(const TileCtx tc, const PipeSrc ps, const LinArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ __align__(16) int4 hdr_ring[4][2];
  __shared__ __align__(8) unsigned long long bars[2];
  const int cns = tc.cap_ns, cnp = tc.cap_np;
  const size_t sb = PipeStage<TILE>::bytes(true, false, 3, cns, cnp);
  TileSmem<TILE> sm;
  sm.cap_ns = cns; sm.cap_np = cnp;
  sm.sv = reinterpret_cast<double*>(smem_raw + 2 * sb);
  sm.sw = nullptr;
  sm.sred = sm.sv + 18 * PSFM_SVS;
  sm.sx = nullptr;
  double* racc = sm.sred + 9 * 32;          // [3][TILE] running sums of this CTA's threads
  for (int k = 0; k < 3; ++k) racc[k * TILE + threadIdx.x] = 0.0;
  pipe_run<TILE>(tc, ps, smem_raw, hdr_ring, bars, 3, cns, cnp, [&](const TileInfo& ti, const PipeStage<TILE>& s, int tile) {
    view_stage<TILE>(sm, s);
    const int tid = threadIdx.x;
    const bool act = tid < ti.n;
    int ls = 0, lp = 0;
    double2 xy = make_double2(0.0, 0.0);
    if (act) { ls = s.lseg[tid]; lp = s.lpt[tid]; xy = s.xy[tid]; }
    linearize_tile<TILE, ROT>(tc, a, sm, ti, act, ls, lp, xy, tile, racc);
  });
  if ((int)blockIdx.x < tc.T) linearize_flush<TILE>(a, racc, sm.sred);
}

template <int TILE>
inline size_t pipe_smem_linearize(int cns, int cnp) {
  return 2 * PipeStage<TILE>::bytes(true, false, 3, cns, cnp) + sizeof(double) * (18 * (TILE + 1) + 9 * 32 + 3 * TILE);
}


// ------------------------------------------------------------------ pipelined back-substitution
//
// Stage = r (the 16-byte slot of xy), D (a), segment poses, per point X | H~ | w^ (12 rows).  The scaled camera
// step xs (6 F + 3 doubles) is small: the persistent CTA keeps the WHOLE vector in shared memory and every tile
// gathers its segments' rows from there.
template <int TILE, bool ROT>
__global__ void __launch_bounds__(TILE, (TILE == 256 ? 3 : 1)) k_back_substitute_p(const TileCtx tc, const PipeSrc ps, const BackArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ __align__(16) int4 hdr_ring[4][2];
  __shared__ __align__(8) unsigned long long bars[2];
  const int cns = tc.cap_ns, cnp = tc.cap_np;
  const size_t sb = PipeStage<TILE>::bytes(true, true, 12, cns, cnp);
  TileSmem<TILE> sm;
  sm.cap_ns = cns; sm.cap_np = cnp;
  sm.sv = reinterpret_cast<double*>(smem_raw + 2 * sb);
  sm.sw = sm.sv + 3 * PSFM_SVS;
  sm.sred = sm.sw + 4 * (size_t)cnp;
  sm.sx = sm.sred + 9 * 32;
  double* xs_all = sm.sx + 6 * (size_t)cns;
  const int nxs = 6 * tc.F + 3 * tc.C;
  for (int j = threadIdx.x; j < nxs; j += TILE) xs_all[j] = __ldg(a.xs + j);
  double xk[3] = {0, 0, 0};
  double inv_f = 0.0;
  if (a.intr >= 1) {
    xk[0] = __ldg(a.xs + 6 * (size_t)tc.F); xk[1] = __ldg(a.xs + 6 * (size_t)tc.F + 1); xk[2] = __ldg(a.xs + 6 * (size_t)tc.F + 2);
    inv_f = 1.0 / __ldg(a.K);
  }
  // [3][TILE] running sums of this CTA's threads, 16-byte aligned (ptxas then needs 107 instead of 121 registers at TILE 512)
  double* racc = reinterpret_cast<double*>((reinterpret_cast<uintptr_t>(xs_all + nxs) + 15) & ~(uintptr_t)15);
  for (int k = 0; k < 3; ++k) racc[k * TILE + threadIdx.x] = 0.0;
  __syncthreads();
  pipe_run<TILE>(tc, ps, smem_raw, hdr_ring, bars, 12, cns, cnp, [&](const TileInfo& ti, const PipeStage<TILE>& s, int tile) {
    view_stage<TILE>(sm, s);
    const int tid = threadIdx.x;
    const bool act = tid < ti.n;
    int ls = 0, lp = 0;
    double a00 = 0, a02 = 0, a12 = 0, r0 = 0, r1 = 0;
    if (act) {
      ls = s.lseg[tid]; lp = s.lpt[tid];
      a00 = s.a0[tid]; a02 = s.a1[tid]; a12 = s.a2[tid];
      const double2 rr = s.xy[tid];
      r0 = rr.x; r1 = rr.y;
    }
    for (int j = tid; j < ti.ns * 6; j += TILE) {
      const int sg = j / 6, k = j - 6 * sg;
      sm.sx[k * cns + sg] = xs_all[6 * s.cimg[sg] + k];
    }
    __syncthreads();
    back_substitute_tile<TILE, ROT>(tc, a, sm, ti, act, ls, lp, a00, a02, a12, r0, r1, xk, inv_f, racc);
  });
  if ((int)blockIdx.x < tc.T) {
    double v[3] = {racc[threadIdx.x], racc[TILE + threadIdx.x], racc[2 * TILE + threadIdx.x]};
    const double s = block_sum_multi<3>(v, sm.sred);
    if (threadIdx.x < 3) atomicAdd(a.acc + threadIdx.x, s);
  }
}

// nxs: length of the scaled camera step (6 F + 3 C)
template <int TILE>
inline size_t pipe_smem_back_substitute(int cns, int cnp, int nxs) {
  return 2 * PipeStage<TILE>::bytes(true, true, 12, cns, cnp) +
         sizeof(double) * (3 * (TILE + 1) + 4 * (size_t)cnp + 9 * 32 + 6 * (size_t)cns + (size_t)nxs + 2 + 3 * TILE);
}

}  // namespace ba
}  // namespace psfm
