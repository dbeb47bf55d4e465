// Advect-diffuse right-hand side on multi-level meshes, per-block lab loader on the WENO line core (DESIGN.md 7.1 step 1).
//
// STATUS: like csrc/amr_ops.cu — compiled for sm_90a, its logic also checked on the CPU through tests/host_emu/ (cooperative
// thread emulation).  cup2d_amr_advect_diffuse_rhs_fast gives the same result as the table-gather
// baseline cup2d_amr_advect_diffuse_rhs.
//
// One warp owns four blocks.  Per block two padded planes (u, v: 14 rows x 15) in shared memory hold the lab:
//   interior      the block itself (1 KB, coalesced)
//   face ghosts   3 layers behind each of the 4 faces (the stencil of KernelAdvectDiffuse is cross-shaped: main.cpp:5441-5503
//                 reads +-3 along the axes only): same-level neighbour -> copy; domain wall -> the wall-adjacent cell with
//                 the normal component negated (main.cpp:3144-3154); coarser / finer neighbour -> left to the table pass
//   table pass    blocks that have a non-same-level neighbour get their ghost rows from the compact ghost-stencil table of
//                 the host plan (cup2d_amr_plan_ghosts): value = sum_e w[e] * vel[src[e]]
// then the x pass (lanes = 4 blocks x 8 rows) and the y pass (lanes = 4 blocks x 8 columns) of weno.cuh, exactly the
// arithmetic of the uniform-grid kernel (advect.cu) with the cell size of the block.  Warps never synchronise with each
// other.  Blocks with a coarse-fine face also store their face fluxes dfac*(inner - ghost) (main.cpp:5515-5569) for the
// correction kernel below, which is the coarse-face formulation of fillcases (see amr_ops.cu) reading those buffers.
#include "sim.h"
#include "weno.cuh"
#include <map>
#include <algorithm>
#include <vector>
#include "amr.h"

extern "C" {
int64_t cup2d_amr_plan_irregular(cup2d_amr_plan *p, int32_t *blocks_out);
int64_t cup2d_amr_plan_ghosts(cup2d_amr_plan *p, int which, int64_t *nrows, int64_t *rowptr, int32_t *dst, int32_t *src_block,
                              int32_t *src_cellcomp, double *weight);
int cup2d_amr_plan_neighbours(cup2d_amr_plan *p, int32_t *out);
}

namespace cup2d {

constexpr int AF_WARPS = 4;                // warps per CTA
constexpr int AF_NT = 32 * AF_WARPS;
constexpr int AF_BPW = 4;                  // blocks per warp
constexpr int AF_PS = 15;                  // plane row stride (odd: lanes along y are conflict-free)
constexpr int AF_PLANE = 14 * AF_PS;       // doubles per component plane
constexpr int AF_RS = 9;                   // partial-result row stride
constexpr int AF_BLK = 2 * AF_PLANE + 2 * 8 * AF_RS; // doubles of shared memory per block: su, sv, Ru, Rv
constexpr int AF_SMEM = AF_WARPS * AF_BPW * AF_BLK * 8; // 72 192 B per CTA -> 3 CTAs/SM

__global__ void __launch_bounds__(AF_NT)
amr_advect_fast_kernel(const double *__restrict__ vel, double *__restrict__ out, const int4 *__restrict__ nbr4,
                       const int *__restrict__ irr_of, const GhostDev gt, const double *__restrict__ hb,
                       const FluxBuf faceflux, int nb, double nu, double dt) {
  extern __shared__ __align__(16) double af_smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int q = lane >> 3, r = lane & 7;
  const int b0 = (blockIdx.x * AF_WARPS + warp) * AF_BPW; // first block of this warp
  if (b0 >= nb) return;
  double *base = af_smem + (size_t)warp * AF_BPW * AF_BLK;
  const double2 *vel2 = reinterpret_cast<const double2 *>(vel);

  // ---- load: interior + same-level / wall face ghosts of the warp's (up to) four blocks ----
  for (int qq = 0; qq < AF_BPW; qq++) {
    const int k = b0 + qq;
    if (k >= nb) break;
    double *su = base + qq * AF_BLK, *sv = su + AF_PLANE;
    for (int i = lane; i < 64; i += 32) {
      const double2 v = vel2[(size_t)k * 64 + i];
      const int p = ((i >> 3) + 3) * AF_PS + (i & 7) + 3;
      su[p] = v.x;
      sv[p] = v.y;
    }
    const int4 nbk = nbr4[k];
    for (int g = lane; g < 96; g += 32) { // face f, position t along it, layer d = 1..3 behind it
      const int f = g / 24, t = g % 8, d = (g % 24) / 8 + 1;
      const int nbf = f == 0 ? nbk.x : f == 1 ? nbk.y : f == 2 ? nbk.z : nbk.w;
      if (nbf < -1) continue; // coarser / finer: the table pass writes this ghost
      int ix, iy, sx, sy; // ghost position (block-relative) and source cell
      if (f < 2) {
        ix = f == 0 ? -d : 7 + d, iy = t;
        sx = nbf >= 0 ? (f == 0 ? 8 - d : d - 1) : (f == 0 ? 0 : 7), sy = t;
      } else {
        ix = t, iy = f == 2 ? -d : 7 + d;
        sx = t, sy = nbf >= 0 ? (f == 2 ? 8 - d : d - 1) : (f == 2 ? 0 : 7);
      }
      double2 v = vel2[(size_t)(nbf >= 0 ? nbf : k) * 64 + sy * 8 + sx];
      if (nbf < 0) { // wall: normal component negated, tangential copied
        if (f < 2) v.x = -v.x; else v.y = -v.y;
      }
      const int p = (iy + 3) * AF_PS + ix + 3;
      su[p] = v.x;
      sv[p] = v.y;
    }
  }
  __syncwarp();
  // ---- table pass: ghost rows of the blocks with a coarser / finer neighbour ----
  for (int qq = 0; qq < AF_BPW; qq++) {
    const int k = b0 + qq;
    if (k >= nb) break;
    const int qi = irr_of[k];
    if (qi < 0) continue;
    double *su = base + qq * AF_BLK;
    for (int64_t row = gt.grow[qi] + lane; row < gt.grow[qi + 1]; row += 32) {
      double acc = 0.0;
      for (int64_t e = gt.rowptr[row]; e < gt.rowptr[row + 1]; e++) acc += gt.w[e] * vel[(size_t)gt.sb[e] * 128 + gt.sc[e]];
      const int cc = gt.dst[row] % (14 * 14 * 2); // (lab row * 14 + lab column) * 2 + component
      const int comp = cc & 1, lx = (cc >> 1) % 14, ly = (cc >> 1) / 14;
      su[comp * AF_PLANE + ly * AF_PS + lx] = acc;
    }
  }
  __syncwarp();
  const int k = b0 + q;
  const bool live = k < nb;
  double *su = base + q * AF_BLK, *sv = su + AF_PLANE, *Ru = sv + AF_PLANE, *Rv = Ru + 8 * AF_RS;
  const double h = live ? hb[k] : 1.0;
  const double dfac = nu * dt, afac3 = -dt * h * (1.0 / 3.0); // main.cpp:5446-5447; weno_line delivers 3 x the differences
  // ---- face fluxes of the blocks with a coarse-fine face: lane = (face q', position r) of block qq ----
  for (int qq = 0; qq < AF_BPW; qq++) {
    const int kk = b0 + qq;
    if (kk >= nb) break;
    const int qi = irr_of[kk];
    if (qi < 0) continue;
    const double *pu = base + qq * AF_BLK, *pv = pu + AF_PLANE;
    const int f = q, t = r;
    int ix, iy, gx, gy;
    if (f < 2) ix = f == 0 ? 0 : 7, iy = t, gx = f == 0 ? -1 : 8, gy = t;
    else ix = t, iy = f == 2 ? 0 : 7, gx = t, gy = f == 2 ? -1 : 8;
    const int pi = (iy + 3) * AF_PS + ix + 3, pg = (gy + 3) * AF_PS + gx + 3;
    double *ff = faceflux.p + (size_t)(faceflux.by_block ? kk : qi) * faceflux.stride + (f * 8 + t) * 2;
    ff[0] = dfac * (pu[pi] - pu[pg]);
    ff[1] = dfac * (pv[pi] - pv[pg]);
  }
  // (lanes of a partial last warp keep running on their unused planes and simply do not store)
  // ---- x pass: lane = row r of block q ----
  weno_line(su + (r + 3) * AF_PS, sv + (r + 3) * AF_PS, 1,
            [&](int c, double U, double, double du, double dv, double D2u, double D2v) { // du, dv: 3 x the differences
              const double aU = afac3 * U;
              Ru[r * AF_RS + c] = fma(aU, du, dfac * D2u);
              Rv[r * AF_RS + c] = fma(aU, dv, dfac * D2v);
            });
  __syncwarp();
  // ---- y pass: lane = column r of block q; advecting component is v ----
  double2 *outp = reinterpret_cast<double2 *>(out) + (size_t)(live ? k : 0) * 64 + r;
  weno_line(sv + (r + 3), su + (r + 3), AF_PS, [&](int c, double V, double, double dv, double du, double D2v, double D2u) {
    const double aV = afac3 * V;
    double2 o;
    o.x = Ru[c * AF_RS + r] + fma(aV, du, dfac * D2u);
    o.y = Rv[c * AF_RS + r] + fma(aV, dv, dfac * D2v);
    if (live) outp[c * 8] = o;
  });
}

// ---- the +-1 stencils (pressure_rhs, pressure_rhs1, pressureCorrectionKernel): 10x10 labs, one warp = four blocks ----
constexpr int A1_WARPS = 2, A1_NT = 64, A1_PS = 11, A1_PLANE = 10 * A1_PS;

// the whole warp loads the +-1 lab of block k into DIM planes: interior, one ghost layer per face from the neighbour
// table (vector fields: normal component negated at walls, main.cpp:3144-3154; scalars: copied, main.cpp:3239-3244), then
// the ghost rows of the compact table if the block has a coarser / finer neighbour.  Ends with a __syncwarp.
template <int DIM>
__device__ __forceinline__ void load_lab1(double *pl, const double *__restrict__ field, int k, const int4 nbk, int qi,
                                          const GhostDev &gt, int lane) {
  for (int i = lane; i < 64; i += 32)
    for (int d = 0; d < DIM; d++) pl[d * A1_PLANE + ((i >> 3) + 1) * A1_PS + (i & 7) + 1] = field[((size_t)k * 64 + i) * DIM + d];
  {
    const int f = lane >> 3, t = lane & 7;
    const int nbf = f == 0 ? nbk.x : f == 1 ? nbk.y : f == 2 ? nbk.z : nbk.w;
    if (nbf >= -1) {
      int ix, iy, sx, sy;
      if (f < 2) ix = f == 0 ? -1 : 8, iy = t, sx = nbf >= 0 ? (f == 0 ? 7 : 0) : (f == 0 ? 0 : 7), sy = t;
      else ix = t, iy = f == 2 ? -1 : 8, sx = t, sy = nbf >= 0 ? (f == 2 ? 7 : 0) : (f == 2 ? 0 : 7);
      for (int d = 0; d < DIM; d++) {
        double v = field[((size_t)(nbf >= 0 ? nbf : k) * 64 + sy * 8 + sx) * DIM + d];
        if (DIM == 2 && nbf < 0 && d == (f < 2 ? 0 : 1)) v = -v;
        pl[d * A1_PLANE + (iy + 1) * A1_PS + ix + 1] = v;
      }
    }
  }
  __syncwarp();
  if (qi >= 0)
    for (int64_t row = gt.grow[qi] + lane; row < gt.grow[qi + 1]; row += 32) {
      double acc = 0.0;
      for (int64_t e = gt.rowptr[row]; e < gt.rowptr[row + 1]; e++) acc += gt.w[e] * field[(size_t)gt.sb[e] * 64 * DIM + gt.sc[e]];
      const int cc = gt.dst[row] % (10 * 10 * DIM);
      const int d = cc % DIM, lx = (cc / DIM) % 10, ly = (cc / DIM) / 10;
      pl[d * A1_PLANE + ly * A1_PS + lx] = acc;
    }
  __syncwarp();
}
__device__ __forceinline__ void face_pos(int f, int t, int &pi, int &pg) { // inner cell and ghost behind face f at position t
  int ix, iy, gx, gy;
  if (f < 2) ix = f == 0 ? 0 : 7, iy = t, gx = f == 0 ? -1 : 8, gy = t;
  else ix = t, iy = f == 2 ? 0 : 7, gx = t, gy = f == 2 ? -1 : 8;
  pi = (iy + 1) * A1_PS + ix + 1, pg = (gy + 1) * A1_PS + gx + 1;
}

// tmp = pressure_rhs(vel, u_def, chi) (main.cpp:6105-6139) + the face fluxes of main.cpp:6152-6205
__global__ void __launch_bounds__(A1_NT)
amr_div_fast_kernel(const double *__restrict__ vel, const double *__restrict__ udef, const double *__restrict__ chi,
                    double *__restrict__ tmp, const int4 *__restrict__ nbr4, const int *__restrict__ irr_of, const GhostDev gt,
                    const double *__restrict__ hb, const FluxBuf faceflux, int nb, double dt) {
  __shared__ double s_lab[A1_WARPS * 4 * 4 * A1_PLANE];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, q = lane >> 3, r = lane & 7;
  const int b0 = (blockIdx.x * A1_WARPS + warp) * 4;
  if (b0 >= nb) return;
  double *base = s_lab + warp * 4 * 4 * A1_PLANE;
  for (int qq = 0; qq < 4 && b0 + qq < nb; qq++) {
    const int k = b0 + qq;
    load_lab1<2>(base + qq * 4 * A1_PLANE, vel, k, nbr4[k], irr_of[k], gt, lane);
    load_lab1<2>(base + qq * 4 * A1_PLANE + 2 * A1_PLANE, udef, k, nbr4[k], irr_of[k], gt, lane);
  }
  for (int qq = 0; qq < 4 && b0 + qq < nb; qq++) { // face fluxes: lane = (face q, position r)
    const int k = b0 + qq, qi = irr_of[k];
    if (qi < 0) continue;
    const double *vu = base + qq * 4 * A1_PLANE, *uu = vu + 2 * A1_PLANE;
    const double fac = 0.5 * hb[k] / dt;
    int pi, pg;
    face_pos(q, r, pi, pg);
    const int c = q < 2 ? 0 : 1;
    const double sv = vu[c * A1_PLANE + pg] + vu[c * A1_PLANE + pi], su = uu[c * A1_PLANE + pg] + uu[c * A1_PLANE + pi];
    const int ix = q < 2 ? (q == 0 ? 0 : 7) : r, iy = q < 2 ? r : (q == 2 ? 0 : 7);
    const double x = chi[(size_t)k * 64 + iy * 8 + ix];
    faceflux.p[(size_t)(faceflux.by_block ? k : qi) * faceflux.stride + q * 8 + r] =
        (q & 1) == 0 ? fac * sv - (fac * x) * su : -fac * sv + (fac * x) * su;
  }
  const int k = b0 + q;
  if (k >= nb) return;
  const double *vu = base + q * 4 * A1_PLANE, *vv = vu + A1_PLANE, *uu = vv + A1_PLANE, *uv = uu + A1_PLANE;
  const double fac = 0.5 * hb[k] / dt;
  const int row = (r + 1) * A1_PS + 1;
  for (int i = 0; i < 8; i++) {
    const int p = row + i;
    const double dv = ((vu[p + 1] - vu[p - 1]) + vv[p + A1_PS]) - vv[p - A1_PS];
    const double du = ((uu[p + 1] - uu[p - 1]) + uv[p + A1_PS]) - uv[p - A1_PS];
    const size_t cell = (size_t)k * 64 + r * 8 + i;
    tmp[cell] = fac * dv - fac * chi[cell] * du;
  }
}

// MODE 0: tmp -= lap(p) (main.cpp:6209-6230) + face fluxes (6243-6283);  MODE 1: tmpV = pressureCorrectionKernel(p) (6021-6043)
template <int MODE>
__global__ void __launch_bounds__(A1_NT)
amr_scalar_fast_kernel(const double *__restrict__ p, double *__restrict__ out, const int4 *__restrict__ nbr4,
                       const int *__restrict__ irr_of, const GhostDev gt, const double *__restrict__ hb,
                       const FluxBuf faceflux, int nb, double dt) {
  __shared__ double s_lab[A1_WARPS * 4 * A1_PLANE];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, q = lane >> 3, r = lane & 7;
  const int b0 = (blockIdx.x * A1_WARPS + warp) * 4;
  if (b0 >= nb) return;
  double *base = s_lab + warp * 4 * A1_PLANE;
  for (int qq = 0; qq < 4 && b0 + qq < nb; qq++) load_lab1<1>(base + qq * A1_PLANE, p, b0 + qq, nbr4[b0 + qq], irr_of[b0 + qq], gt, lane);
  if (MODE == 0)
    for (int qq = 0; qq < 4 && b0 + qq < nb; qq++) {
      const int qi = irr_of[b0 + qq];
      if (qi < 0) continue;
      int pi, pg;
      face_pos(q, r, pi, pg);
      const double *m = base + qq * A1_PLANE;
      faceflux.p[(size_t)(faceflux.by_block ? b0 + qq : qi) * faceflux.stride + q * 8 + r] = m[pg] - m[pi];
    }
  const int k = b0 + q;
  if (k >= nb) return;
  const double *m = base + q * A1_PLANE;
  const int row = (r + 1) * A1_PS + 1;
  const double pfac = -0.5 * dt * hb[k];
  for (int i = 0; i < 8; i++) {
    const int c = row + i;
    const size_t cell = (size_t)k * 64 + r * 8 + i;
    if (MODE == 0) out[cell] -= (((m[c - 1] + m[c + 1]) + m[c - A1_PS]) + m[c + A1_PS]) - 4 * m[c];
    else {
      out[2 * cell] = pfac * (m[c + 1] - m[c - 1]);
      out[2 * cell + 1] = pfac * (m[c + A1_PS] - m[c - A1_PS]);
    }
  }
}

// fillcases per coarse face from the stored face fluxes (see amr_fluxcorr_kernel in amr_ops.cu for the formulation)
template <int DIM>
__global__ void amr_fluxcorr_faces_kernel(const CoarseFace *__restrict__ cf, int ncf, const FluxBuf faceflux,
                                          const int *__restrict__ irr_of, double *__restrict__ result) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ncf * 8 * DIM) return;
  const int comp = i % DIM, t = (i / DIM) % 8;
  const CoarseFace f = cf[i / (8 * DIM)];
  auto flux = [&](int blk, int face, int pos) {
    return faceflux.p[(size_t)(faceflux.by_block ? blk : irr_of[blk]) * faceflux.stride + (face * 8 + pos) * DIM + comp];
  };
  double acc = flux(f.coarse, f.face, t);
  const int fb = f.fine[t >> 2];
  if (fb >= 0) {
    const int t2 = 2 * (t & 3);
    acc += flux(fb, f.face ^ 1, t2) + flux(fb, f.face ^ 1, t2 + 1);
  }
  const int ix = f.face < 2 ? (f.face == 0 ? 0 : 7) : t, iy = f.face < 2 ? t : (f.face == 2 ? 0 : 7);
  double *dst = result + ((size_t)f.coarse * 64 + iy * 8 + ix) * DIM + comp;
  double v = *dst + acc;
  if (DIM == 2 && f.fine[0] >= 0 && f.fine[1] >= 0 && 2 * t + comp >= 9) v += acc; // second pass of fillcase1 (DESIGN.md 7.1, property 3)
  *dst = v;
}

// single-rank contexts: a buffer per irregular block; distributed contexts: inside a field array that is free at that point
// (advect: tmp, 64 doubles per block; pressure kernels: vold, 128 per block), refreshed across ranks before fillcases
template <int DIM> static FluxBuf flux_buf(cup2d_amr *a) {
  if (!a->dist) return FluxBuf{a->d_faceflux, 32 * DIM, 0};
  return DIM == 2 ? FluxBuf{a->f[CUP2D_TMP], 64, 1} : FluxBuf{a->f[CUP2D_VOLD], 128, 1};
}
template <int DIM> static int fluxcorr_faces(cup2d_amr *a, double *result) {
  { // the fine side of a coarse face may live on another rank
    const int rc = amr_dist_refresh(a, DIM == 2 ? CUP2D_TMP : CUP2D_VOLD);
    if (rc) return rc;
  }
  for (int dir = 0; dir < 2; dir++) { // x faces, then y faces (fillcases order)
    const int n = a->ncf[dir] * 8 * DIM;
    if (n == 0) continue;
    amr_fluxcorr_faces_kernel<DIM><<<(n + 127) / 128, 128, 0, a->stream>>>(a->d_cf[dir], a->ncf[dir], flux_buf<DIM>(a), a->d_irr_of,
                                                                         result);
  }
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

static int fast_constants() {
  CUP2D_CUDA(cudaMemcpyToSymbol(cW, hW, sizeof hW));
  CUP2D_CUDA(cudaFuncSetAttribute(amr_advect_fast_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, AF_SMEM));
  return CUP2D_OK;
}

static int fast_setup(cup2d_amr *a) {
  if (a->d_faceflux || a->dist) return CUP2D_OK; // distributed contexts get their tables from amr_fast_setup_dist
  const int64_t nb = a->nb;
  std::vector<int32_t> n8(8 * nb), n4(4 * nb), irr_of(nb, -1);
  if (cup2d_amr_plan_neighbours(a->plan, n8.data())) return CUP2D_EINVAL;
  for (int64_t k = 0; k < nb; k++) { // order of the 8: (-1,-1),(0,-1),(1,-1),(-1,0),(1,0),(-1,1),(0,1),(1,1)
    const int pick[4] = {3, 4, 1, 6};  // W, E, S, N
    for (int j = 0; j < 4; j++) n4[4 * k + j] = n8[8 * k + pick[j]] < -1 ? -2 : n8[8 * k + pick[j]];
  }
  const int64_t nirr = cup2d_amr_plan_irregular(a->plan, nullptr);
  std::vector<int32_t> irr(std::max<int64_t>(nirr, 1));
  cup2d_amr_plan_irregular(a->plan, irr.data());
  for (int64_t qi = 0; qi < nirr; qi++) irr_of[irr[qi]] = (int32_t)qi;
  a->nirr = nirr;
  auto up = [](auto **d, const auto &h) -> cudaError_t {
    using T = typename std::remove_reference<decltype(h[0])>::type;
    cudaError_t e = cudaMalloc(d, std::max<size_t>(h.size(), 1) * sizeof(T));
    if (e != cudaSuccess) return e;
    return cudaMemcpy(*d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice);
  };
  const int ncell[3] = {14 * 14 * 2, 10 * 10 * 2, 10 * 10};
  for (int which = 0; which < 3; which++) {
    int64_t nrows = 0;
    const int64_t nnz = cup2d_amr_plan_ghosts(a->plan, which, &nrows, nullptr, nullptr, nullptr, nullptr, nullptr);
    if (nnz < 0) return CUP2D_EINVAL;
    std::vector<int64_t> rp(nrows + 1), grow(nirr + 1, nrows);
    std::vector<int32_t> dst(std::max<int64_t>(nrows, 1)), sb(std::max<int64_t>(nnz, 1)), sc(std::max<int64_t>(nnz, 1));
    std::vector<double> w(std::max<int64_t>(nnz, 1));
    cup2d_amr_plan_ghosts(a->plan, which, &nrows, rp.data(), dst.data(), sb.data(), sc.data(), w.data());
    for (int64_t row = nrows - 1; row >= 0; row--) grow[dst[row] / ncell[which]] = row; // rows are grouped by block, in order
    for (int64_t qi = nirr - 1; qi >= 0; qi--) grow[qi] = std::min(grow[qi], grow[qi + 1]); // blocks without rows
    GhostDev &g = a->gt[which];
    CUP2D_CUDA(up(&g.grow, grow));
    CUP2D_CUDA(up(&g.rowptr, rp));
    CUP2D_CUDA(up(&g.dst, dst));
    CUP2D_CUDA(up(&g.sb, sb));
    CUP2D_CUDA(up(&g.sc, sc));
    CUP2D_CUDA(up(&g.w, w));
  }
  CUP2D_CUDA(up(&a->d_nbr4, n4));
  CUP2D_CUDA(up(&a->d_irr_of, irr_of));
  CUP2D_CUDA(cudaMalloc(&a->d_faceflux, std::max<int64_t>(nirr, 1) * 64 * sizeof(double)));
  return fast_constants();
}

} // namespace cup2d

int amr_fast_tables(cup2d_amr *a) { return cup2d::fast_setup(a); }

// Tables of a DISTRIBUTED context: the plan knows the whole mesh; this rank keeps what concerns its blocks [b0, b1) and
// names every block by its local slot (own blocks first, then the halo slots of the field arrays): slot_of[global block] or -1.
int amr_fast_setup_dist(cup2d_amr *a, const std::vector<int32_t> &slot_of, int64_t b0, int64_t b1) {
  using namespace cup2d;
  const int64_t nglob = (int64_t)slot_of.size(), nloc = b1 - b0;
  auto up = [](auto **d, const auto &h) -> cudaError_t {
    using T = typename std::remove_reference<decltype(h[0])>::type;
    cudaError_t e = cudaMalloc(d, std::max<size_t>(h.size(), 1) * sizeof(T));
    if (e != cudaSuccess) return e;
    return cudaMemcpy(*d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice);
  };
  auto slot = [&](int32_t g) -> int32_t {
    if (g < 0) return g;
    return slot_of[g]; // -1 would mean a block the halo set missed: caught below
  };
  std::vector<int32_t> n8(8 * nglob), n4(4 * nloc);
  if (cup2d_amr_plan_neighbours(a->plan, n8.data())) return CUP2D_EINVAL;
  for (int64_t k = 0; k < nloc; k++) {
    const int pick[4] = {3, 4, 1, 6}; // W, E, S, N
    for (int j = 0; j < 4; j++) {
      const int32_t g = n8[8 * (b0 + k) + pick[j]];
      n4[4 * k + j] = g < -1 ? -2 : slot(g);
      if (g >= 0 && n4[4 * k + j] < 0) return CUP2D_EINVAL;
    }
  }
  const int64_t nirr_g = cup2d_amr_plan_irregular(a->plan, nullptr);
  std::vector<int32_t> irr(std::max<int64_t>(nirr_g, 1)), irr_of(nloc, -1), local_of_irr(std::max<int64_t>(nirr_g, 1), -1);
  cup2d_amr_plan_irregular(a->plan, irr.data());
  int64_t nirr = 0;
  for (int64_t qi = 0; qi < nirr_g; qi++)
    if (irr[qi] >= b0 && irr[qi] < b1) {
      local_of_irr[qi] = (int32_t)nirr;
      irr_of[irr[qi] - b0] = (int32_t)nirr++;
    }
  a->nirr = nirr;
  const int ncell[3] = {14 * 14 * 2, 10 * 10 * 2, 10 * 10};
  for (int which = 0; which < 3; which++) {
    int64_t nrows_g = 0;
    const int64_t nnz_g = cup2d_amr_plan_ghosts(a->plan, which, &nrows_g, nullptr, nullptr, nullptr, nullptr, nullptr);
    if (nnz_g < 0) return CUP2D_EINVAL;
    std::vector<int64_t> rp_g(nrows_g + 1);
    std::vector<int32_t> dst_g(std::max<int64_t>(nrows_g, 1)), sb_g(std::max<int64_t>(nnz_g, 1)), sc_g(std::max<int64_t>(nnz_g, 1));
    std::vector<double> w_g(std::max<int64_t>(nnz_g, 1));
    cup2d_amr_plan_ghosts(a->plan, which, &nrows_g, rp_g.data(), dst_g.data(), sb_g.data(), sc_g.data(), w_g.data());
    std::vector<int64_t> rp(1, 0);
    std::vector<int32_t> dst, sb, sc;
    std::vector<double> w;
    for (int64_t row = 0; row < nrows_g; row++) {
      const int32_t ql = local_of_irr[dst_g[row] / ncell[which]];
      if (ql < 0) continue;
      dst.push_back(ql * ncell[which] + dst_g[row] % ncell[which]);
      for (int64_t e = rp_g[row]; e < rp_g[row + 1]; e++) {
        const int32_t sl = slot(sb_g[e]);
        if (sl < 0) return CUP2D_EINVAL;
        sb.push_back(sl);
        sc.push_back(sc_g[e]);
        w.push_back(w_g[e]);
      }
      rp.push_back((int64_t)w.size());
    }
    const int64_t nrows = (int64_t)dst.size();
    std::vector<int64_t> grow(nirr + 1, nrows);
    for (int64_t row = nrows - 1; row >= 0; row--) grow[dst[row] / ncell[which]] = row;
    for (int64_t qi = nirr - 1; qi >= 0; qi--) grow[qi] = std::min(grow[qi], grow[qi + 1]);
    GhostDev &g = a->gt[which];
    CUP2D_CUDA(up(&g.grow, grow));
    CUP2D_CUDA(up(&g.rowptr, rp));
    CUP2D_CUDA(up(&g.dst, dst));
    CUP2D_CUDA(up(&g.sb, sb));
    CUP2D_CUDA(up(&g.sc, sc));
    CUP2D_CUDA(up(&g.w, w));
  }
  CUP2D_CUDA(up(&a->d_nbr4, n4));
  CUP2D_CUDA(up(&a->d_irr_of, irr_of));
  // coarse faces whose COARSE block is ours (the fine side may be a halo slot)
  const int64_t nf = cup2d_amr_plan_faces(a->plan, nullptr);
  std::vector<int32_t> rec(5 * std::max<int64_t>(nf, 1));
  cup2d_amr_plan_faces(a->plan, rec.data());
  std::map<std::pair<int, int>, CoarseFace> byface;
  for (int64_t r = 0; r < nf; r++) {
    const int fine = rec[5 * r], kc = rec[5 * r + 2], fc = rec[5 * r + 3], half = rec[5 * r + 4];
    if (kc < b0 || kc >= b1) continue;
    auto it = byface.find({kc, fc});
    if (it == byface.end()) it = byface.emplace(std::make_pair(kc, fc), CoarseFace{(int)(kc - b0), fc, {-1, -1}}).first;
    it->second.fine[half] = slot(fine);
    if (it->second.fine[half] < 0) return CUP2D_EINVAL;
  }
  std::vector<CoarseFace> lists[2];
  for (auto &e : byface) lists[e.second.face < 2 ? 0 : 1].push_back(e.second);
  for (int d = 0; d < 2; d++) {
    a->ncf[d] = (int)lists[d].size();
    if (!lists[d].empty()) CUP2D_CUDA(up(&a->d_cf[d], lists[d]));
  }
  return fast_constants();
}

using namespace cup2d;

extern "C" {

/* tmpV = KernelAdvectDiffuse(vel), flux-corrected (main.cpp:6611-6617): same result as cup2d_amr_advect_diffuse_rhs */
int cup2d_amr_advect_diffuse_rhs_fast(cup2d_amr *a, double dt) {
  if (!a) {
    set_error("null cup2d_amr handle");
    return CUP2D_EINVAL;
  }
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc = fast_setup(a);
  if (rc) return rc;
  if ((rc = amr_dist_refresh(a, CUP2D_VEL))) return rc;
  const int per_cta = AF_WARPS * AF_BPW;
  const int grid = (int)((a->nb + per_cta - 1) / per_cta);
  amr_advect_fast_kernel<<<grid, AF_NT, AF_SMEM, a->stream>>>(
      a->f[CUP2D_VEL], a->f[CUP2D_TMPV], reinterpret_cast<const int4 *>(a->d_nbr4), a->d_irr_of, a->gt[0], a->d_h,
      flux_buf<2>(a), (int)a->nb, a->nu, dt);
  CUP2D_CUDA(cudaGetLastError());
  return fluxcorr_faces<2>(a, a->f[CUP2D_TMPV]);
}

/* same results as cup2d_amr_pressure_rhs / cup2d_amr_pressure_gradient through per-block +-1 labs in shared memory */
int cup2d_amr_pressure_rhs_fast(cup2d_amr *a, double dt, int with_laplacian) {
  if (!a) {
    set_error("null cup2d_amr handle");
    return CUP2D_EINVAL;
  }
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc = fast_setup(a);
  if (rc) return rc;
  if ((rc = amr_dist_refresh(a, CUP2D_VEL)) || (rc = amr_dist_refresh(a, CUP2D_TMPV))) return rc;
  const int grid = (int)((a->nb + A1_WARPS * 4 - 1) / (A1_WARPS * 4));
  const int4 *nbr4 = reinterpret_cast<const int4 *>(a->d_nbr4);
  amr_div_fast_kernel<<<grid, A1_NT, 0, a->stream>>>(a->f[CUP2D_VEL], a->f[CUP2D_TMPV], a->f[CUP2D_CHI], a->f[CUP2D_TMP], nbr4,
                                                     a->d_irr_of, a->gt[1], a->d_h, flux_buf<1>(a), (int)a->nb, dt);
  CUP2D_CUDA(cudaGetLastError());
  if ((rc = fluxcorr_faces<1>(a, a->f[CUP2D_TMP])) || !with_laplacian) return rc;
  return cup2d_amr_laplacian_fast(a, dt);
}

/* tmp -= lap(pold), flux-corrected (main.cpp:7022-7027) */
int cup2d_amr_laplacian_fast(cup2d_amr *a, double dt) {
  if (!a) {
    set_error("null cup2d_amr handle");
    return CUP2D_EINVAL;
  }
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc = fast_setup(a);
  if (rc) return rc;
  if ((rc = amr_dist_refresh(a, CUP2D_POLD))) return rc;
  const int grid = (int)((a->nb + A1_WARPS * 4 - 1) / (A1_WARPS * 4));
  amr_scalar_fast_kernel<0><<<grid, A1_NT, 0, a->stream>>>(a->f[CUP2D_POLD], a->f[CUP2D_TMP], reinterpret_cast<const int4 *>(a->d_nbr4),
                                                           a->d_irr_of, a->gt[2], a->d_h, flux_buf<1>(a), (int)a->nb, dt);
  CUP2D_CUDA(cudaGetLastError());
  return fluxcorr_faces<1>(a, a->f[CUP2D_TMP]);
}

/* route the operator entry points (and with them cup2d_amr_step) through the fast kernels of this file */
int cup2d_amr_set_fast(cup2d_amr *a, int on) {
  if (!a) return CUP2D_EINVAL;
  if (a->dist && !on) {
    set_error("cup2d_amr_set_fast: a distributed context has the fast kernels only");
    return CUP2D_ESTATE;
  }
  a->fast = on != 0;
  return CUP2D_OK;
}

int cup2d_amr_pressure_gradient_fast(cup2d_amr *a, double dt) {
  if (!a) {
    set_error("null cup2d_amr handle");
    return CUP2D_EINVAL;
  }
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc = fast_setup(a);
  if (rc) return rc;
  if ((rc = amr_dist_refresh(a, CUP2D_PRES))) return rc;
  const int grid = (int)((a->nb + A1_WARPS * 4 - 1) / (A1_WARPS * 4));
  amr_scalar_fast_kernel<1><<<grid, A1_NT, 0, a->stream>>>(a->f[CUP2D_PRES], a->f[CUP2D_TMPV], reinterpret_cast<const int4 *>(a->d_nbr4),
                                                           a->d_irr_of, a->gt[2], a->d_h, flux_buf<1>(a), (int)a->nb, dt);
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

} // extern "C"
