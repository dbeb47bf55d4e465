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
#include <algorithm>
#include <vector>
#include "amr.h"

namespace cup2d {

constexpr int AF_WARPS = 4;                // warps per CTA
constexpr int AF_NT = 32 * AF_WARPS;
constexpr int AF_BPW = 4;                  // blocks per warp
constexpr int AF_PS = 15;                  // plane row stride (odd: lanes along y are conflict-free)
constexpr int AF_PLANE = 14 * AF_PS;       // doubles per component plane
constexpr int AF_RS = 9;                   // partial-result row stride
constexpr int AF_BLK = 2 * AF_PLANE + 2 * 8 * AF_RS; // doubles of shared memory per block: su, sv, Ru, Rv
constexpr int AF_SMEM = AF_WARPS * AF_BPW * AF_BLK * 8; // 72 192 B per CTA -> 3 CTAs/SM

template <class DT>
__global__ void __launch_bounds__(AF_NT)
amr_advect_fast_kernel(const double *__restrict__ vel, double *__restrict__ out, const int4 *__restrict__ nbr4,
                       const int *__restrict__ irr_of, const GhostDev gt, const double *__restrict__ hb,
                       const FluxBuf faceflux, int nb, double nu, DT dt_arg) {
  const double dt = dt_arg.get();
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
template <class DT>
__global__ void __launch_bounds__(A1_NT)
amr_div_fast_kernel(const double *__restrict__ vel, const double *__restrict__ udef, const double *__restrict__ chi,
                    double *__restrict__ tmp, const int4 *__restrict__ nbr4, const int *__restrict__ irr_of, const GhostDev gt,
                    const double *__restrict__ hb, const FluxBuf faceflux, int nb, DT dt_arg) {
  const double dt = dt_arg.get();
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
template <int MODE, class DT>
__global__ void __launch_bounds__(A1_NT)
amr_scalar_fast_kernel(const double *__restrict__ p, double *__restrict__ out, const int4 *__restrict__ nbr4,
                       const int *__restrict__ irr_of, const GhostDev gt, const double *__restrict__ hb,
                       const FluxBuf faceflux, int nb, DT dt_arg) {
  const double dt = dt_arg.get();
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

// adapt()'s tagging (amr_vorticity_kernel + amr_tag_block_kernel of amr_ops.cu) without the full per-cell tables.  Does
// block k's {-4,-4,5,5,tensorial} chi lab hold a positive value within `off` cells of the block?  Lanes stride over the lab
// cells: own cells directly; on a regular block the ghosts from the 8-neighbour table with the scalar wall clamp (as fo_labs
// in amr_forces.cu); on an irregular block the compact kind-3 rows, each summed in row order as amr_gather_kernel sums it.
// Ghost cells the plan leaves unwritten are 0 in the full table and never fire.  Every lane gets the answer.
__device__ __forceinline__ bool chi_fires(const double *__restrict__ chi, int k, int qi, int off, const int *__restrict__ nbr8,
                                          const GhostDev &gc, int lane) {
  auto inside = [off](int gx, int gy) { return gx >= -off && gx < 8 + off && gy >= -off && gy < 8 + off; };
  const int *n8 = nbr8 + (size_t)k * 8; // (-1,-1),(0,-1),(1,-1),(-1,0),(1,0),(-1,1),(0,1),(1,1)
  int hit = 0;
  for (int c = lane; c < 256; c += 32) {
    const int gx = (c & 15) - 4, gy = (c >> 4) - 4;
    if (!inside(gx, gy)) continue;
    const int ox = gx < 0 ? -1 : gx > 7, oy = gy < 0 ? -1 : gy > 7;
    if (ox == 0 && oy == 0) {
      hit |= chi[(size_t)k * 64 + gy * 8 + gx] > 0.0;
      continue;
    }
    if (qi >= 0) continue; // irregular: the ghost rows below
    const bool wx = ox != 0 && n8[ox < 0 ? 3 : 4] == -1, wy = oy != 0 && n8[oy < 0 ? 1 : 6] == -1;
    const int cx = wx ? (ox < 0 ? 0 : 7) : gx, cy = wy ? (oy < 0 ? 0 : 7) : gy;
    const int qx = cx < 0 ? -1 : cx > 7, qy = cy < 0 ? -1 : cy > 7;
    const int b = qx == 0 && qy == 0 ? k : n8[(qy + 1) * 3 + (qx + 1) - ((qy + 1) * 3 + (qx + 1) > 4)];
    hit |= chi[(size_t)b * 64 + (cy & 7) * 8 + (cx & 7)] > 0.0;
  }
  if (qi >= 0)
    for (int64_t row = gc.grow[qi] + lane; row < gc.grow[qi + 1]; row += 32) {
      const int c = gc.dst[row] % 256;
      if (!inside((c & 15) - 4, (c >> 4) - 4)) continue;
      double acc = 0.0;
      for (int64_t e = gc.rowptr[row]; e < gc.rowptr[row + 1]; e++) acc += gc.w[e] * chi[(size_t)gc.sb[e] * 64 + gc.sc[e]];
      hit |= acc > 0.0;
    }
  for (int m = 16; m; m >>= 1) hit |= __shfl_xor_sync(0xffffffffu, hit, m);
  return hit != 0;
}

// tmp = KernelVorticity(vel) (main.cpp:3343-3366) with GradChiOnTmp's 2 Rtol in the four centre cells of the blocks whose chi
// lab is positive within 4 cells (blocks of the finest level) or 2 (the others) (4631-4656); linf[k] = max |tmp| over block k
// (4693-4697).  One warp owns four blocks: the +-1 lab of vel from load_lab1 (compact kind-1 rows), the chi test, then lane
// (q, r) computes row r of block q in amr_vorticity_kernel's expression order.  Given ghost rows in the full tables' term
// order, bit for bit the result of the table path.
__global__ void __launch_bounds__(A1_NT)
amr_tags_fast_kernel(const double *__restrict__ vel, const double *__restrict__ chi, double *__restrict__ tmp,
                     const int4 *__restrict__ nbr4, const int *__restrict__ nbr8, const int *__restrict__ irr_of,
                     const GhostDev gv, const GhostDev gc, const double *__restrict__ hb, double h_finest, double rtol,
                     double *__restrict__ linf, int nb) {
  __shared__ double s_lab[A1_WARPS * 4 * 2 * A1_PLANE];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, q = lane >> 3, r = lane & 7;
  const int b0 = (blockIdx.x * A1_WARPS + warp) * 4;
  if (b0 >= nb) return;
  double *base = s_lab + warp * 4 * 2 * A1_PLANE;
  bool fire = false; // block b0 + q
  for (int qq = 0; qq < 4 && b0 + qq < nb; qq++) {
    const int k = b0 + qq, qi = irr_of[k];
    load_lab1<2>(base + qq * 2 * A1_PLANE, vel, k, nbr4[k], qi, gv, lane);
    const bool f = chi_fires(chi, k, qi, hb[k] == h_finest ? 4 : 2, nbr8, gc, lane);
    if (qq == q) fire = f;
  }
  const int k = b0 + q;
  const bool live = k < nb;
  const double *u = base + q * 2 * A1_PLANE, *v = u + A1_PLANE;
  const double i2h = 0.5 / (live ? hb[k] : 1.0);
  const int row = (r + 1) * A1_PS + 1;
  double m = 0.0;
  for (int i = 0; i < 8; i++) {
    const int p = row + i;
    double t = i2h * (((u[p - A1_PS] - u[p + A1_PS]) + v[p + 1]) - v[p - 1]);
    if (fire && (r == 3 || r == 4) && (i == 3 || i == 4)) t = 2 * rtol;
    if (live) tmp[(size_t)k * 64 + r * 8 + i] = t;
    m = fmax(m, fabs(t));
  }
  for (int s = 4; s; s >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, s)); // the 8 rows of block q
  if (live && r == 0) linf[k] = m;
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
  CUP2D_CUDA(cudaFuncSetAttribute(amr_advect_fast_kernel<ByValue>, cudaFuncAttributeMaxDynamicSharedMemorySize, AF_SMEM));
  CUP2D_CUDA(cudaFuncSetAttribute(amr_advect_fast_kernel<OnDevice>, cudaFuncAttributeMaxDynamicSharedMemorySize, AF_SMEM));
  return CUP2D_OK;
}

int plan_ghosts(cup2d_amr *a, int which, PlanGhosts &g) {
  int64_t nrows = 0;
  const int64_t nnz = cup2d_amr_plan_ghosts(a->plan, which, &nrows, nullptr, nullptr, nullptr, nullptr, nullptr);
  if (nnz < 0) return CUP2D_EINVAL;
  g.rowptr.resize(nrows + 1), g.dst.resize(nrows), g.sb.resize(nnz), g.sc.resize(nnz), g.w.resize(nnz);
  cup2d_amr_plan_ghosts(a->plan, which, &nrows, g.rowptr.data(), g.dst.data(), g.sb.data(), g.sc.data(), g.w.data());
  return CUP2D_OK;
}
int plan_neighbours(cup2d_amr *a, std::vector<int32_t> &n8) {
  n8.resize(8 * a->nglobal);
  return cup2d_amr_plan_neighbours(a->plan, n8.data()) ? CUP2D_EINVAL : CUP2D_OK;
}
std::vector<int32_t> plan_irregular(cup2d_amr *a) {
  std::vector<int32_t> irr(cup2d_amr_plan_irregular(a->plan, nullptr));
  cup2d_amr_plan_irregular(a->plan, irr.data());
  return irr;
}
std::vector<int32_t> plan_faces(cup2d_amr *a) {
  std::vector<int32_t> rec(5 * cup2d_amr_plan_faces(a->plan, nullptr));
  cup2d_amr_plan_faces(a->plan, rec.data());
  return rec;
}

// plain contexts build the tables on first use; distributed ones have them from cup2d_amr_create_ranks
static int fast_setup(cup2d_amr *a) { return a->d_faceflux || a->dist ? CUP2D_OK : amr_fast_build(a); }

} // namespace cup2d

int amr_fast_tables(cup2d_amr *a) { return cup2d::fast_setup(a); }

// The plan's rows of the irregular blocks in [gbegin, gbegin + nb), renumbered to the context's irregular list (local
// position * ncell + lab entry), every source by its slot.  source_order: each row's terms in ascending (block, cell) of the
// whole list, the order of the full per-cell tables (cup2d_amr_plan_stencil), into gt_src[which]; the plan's compact rows
// hold the same terms in the order of the block their pattern was made from.
int amr_ghost_rows(cup2d_amr *a, int which, bool source_order) {
  using namespace cup2d;
  const int64_t b0 = a->gbegin, b1 = a->gbegin + a->nb;
  const int ncell = GHOST_NCELL[which];
  const std::vector<int32_t> irr = plan_irregular(a);
  std::vector<int32_t> local_of_irr(irr.size(), -1);
  int64_t nirr = 0;
  for (size_t qi = 0; qi < irr.size(); qi++)
    if (irr[qi] >= b0 && irr[qi] < b1) local_of_irr[qi] = (int32_t)nirr++;
  PlanGhosts all, g;
  int rc = plan_ghosts(a, which, all);
  if (rc) return rc;
  g.rowptr.reserve(all.rowptr.size()), g.dst.reserve(all.dst.size());
  g.sb.reserve(all.sb.size()), g.sc.reserve(all.sc.size()), g.w.reserve(all.w.size());
  g.rowptr.push_back(0);
  std::vector<int64_t> terms;
  for (size_t row = 0; row < all.dst.size(); row++) {
    const int32_t ql = local_of_irr[all.dst[row] / ncell];
    if (ql < 0) continue;
    g.dst.push_back(ql * ncell + all.dst[row] % ncell);
    terms.clear();
    for (int64_t e = all.rowptr[row]; e < all.rowptr[row + 1]; e++) terms.push_back(e);
    if (source_order)
      std::sort(terms.begin(), terms.end(), [&](int64_t x, int64_t y) {
        return all.sb[x] != all.sb[y] ? all.sb[x] < all.sb[y] : all.sc[x] < all.sc[y];
      });
    for (int64_t e : terms) {
      const int32_t sl = a->slot(all.sb[e]);
      if (sl < 0) {
        set_error("distributed context: a lab source lies outside the halo set");
        return CUP2D_EINVAL;
      }
      g.sb.push_back(sl);
      g.sc.push_back(all.sc[e]);
      g.w.push_back(all.w[e]);
    }
    g.rowptr.push_back((int64_t)g.w.size());
  }
  const int64_t nrows = (int64_t)g.dst.size();
  std::vector<int64_t> grow(nirr + 1, nrows);
  for (int64_t row = nrows - 1; row >= 0; row--) grow[g.dst[row] / ncell] = row; // rows are grouped by block, in order
  for (int64_t qi = nirr - 1; qi >= 0; qi--) grow[qi] = std::min(grow[qi], grow[qi + 1]); // blocks without rows
  GhostDev &d = source_order ? a->gt_src[which] : a->gt[which];
  CUP2D_CUDA(upload(&d.rowptr, g.rowptr));
  CUP2D_CUDA(upload(&d.dst, g.dst));
  CUP2D_CUDA(upload(&d.sb, g.sb));
  CUP2D_CUDA(upload(&d.sc, g.sc));
  CUP2D_CUDA(upload(&d.w, g.w));
  CUP2D_CUDA(upload(&d.grow, grow)); // last: marks the table complete
  return CUP2D_OK;
}

// The fast kernels' tables of the blocks [gbegin, gbegin + nb), every block named by its slot (a distributed context's own
// blocks first, then its halo slots).  The face fluxes of a distributed context travel in a field (flux_buf), so only a
// plain context gets a buffer for them.
int amr_fast_build(cup2d_amr *a) {
  using namespace cup2d;
  const int64_t b0 = a->gbegin, nb = a->nb;
  std::vector<int32_t> n8, n4(4 * nb), irr_of(nb, -1);
  int rc = plan_neighbours(a, n8);
  if (rc) return rc;
  for (int64_t k = 0; k < nb; k++) { // order of the 8: (-1,-1),(0,-1),(1,-1),(-1,0),(1,0),(-1,1),(0,1),(1,1)
    const int pick[4] = {3, 4, 1, 6};  // W, E, S, N
    for (int j = 0; j < 4; j++) {
      const int32_t g = n8[8 * (b0 + k) + pick[j]];
      n4[4 * k + j] = g < -1 ? -2 : g < 0 ? g : a->slot(g);
      if (g >= 0 && n4[4 * k + j] < 0) return CUP2D_EINVAL; // a block the halo set missed
    }
  }
  int64_t nirr = 0;
  for (int32_t g : plan_irregular(a))
    if (g >= b0 && g < b0 + nb) irr_of[g - b0] = (int32_t)nirr++;
  a->nirr = nirr;
  for (int which = 0; which < 3; which++)
    if ((rc = amr_ghost_rows(a, which))) return rc;
  CUP2D_CUDA(upload(&a->d_nbr4, n4));
  CUP2D_CUDA(upload(&a->d_irr_of, irr_of));
  if (!a->dist) CUP2D_CUDA(cudaMalloc(&a->d_faceflux, std::max<int64_t>(nirr, 1) * 64 * sizeof(double)));
  return fast_constants();
}

int amr_advect_rhs_fast(cup2d_amr *a, double dt, const double *ddt) {
  using namespace cup2d;
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc = fast_setup(a);
  if (rc) return rc;
  if ((rc = amr_dist_refresh(a, CUP2D_VEL))) return rc;
  const int per_cta = AF_WARPS * AF_BPW;
  const int grid = (int)((a->nb + per_cta - 1) / per_cta);
  with_scalar(dt, ddt, [&](auto d) {
    amr_advect_fast_kernel<<<grid, AF_NT, AF_SMEM, a->stream>>>(
        a->f[CUP2D_VEL], a->f[CUP2D_TMPV], reinterpret_cast<const int4 *>(a->d_nbr4), a->d_irr_of, a->gt[0], a->d_h,
        flux_buf<2>(a), (int)a->nb, a->nu, d);
    return 0;
  });
  CUP2D_CUDA(cudaGetLastError());
  return fluxcorr_faces<2>(a, a->f[CUP2D_TMPV]);
}

int amr_pressure_rhs_fast(cup2d_amr *a, double dt, int with_laplacian, const double *ddt) {
  using namespace cup2d;
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc = fast_setup(a);
  if (rc) return rc;
  if ((rc = amr_dist_refresh(a, CUP2D_VEL)) || (rc = amr_dist_refresh(a, CUP2D_TMPV))) return rc;
  const int grid = (int)((a->nb + A1_WARPS * 4 - 1) / (A1_WARPS * 4));
  const int4 *nbr4 = reinterpret_cast<const int4 *>(a->d_nbr4);
  with_scalar(dt, ddt, [&](auto d) {
    amr_div_fast_kernel<<<grid, A1_NT, 0, a->stream>>>(a->f[CUP2D_VEL], a->f[CUP2D_TMPV], a->f[CUP2D_CHI], a->f[CUP2D_TMP], nbr4,
                                                       a->d_irr_of, a->gt[1], a->d_h, flux_buf<1>(a), (int)a->nb, d);
    return 0;
  });
  CUP2D_CUDA(cudaGetLastError());
  if ((rc = fluxcorr_faces<1>(a, a->f[CUP2D_TMP])) || !with_laplacian) return rc;
  return cup2d_amr_laplacian_fast(a, dt);
}

int amr_pressure_gradient_fast(cup2d_amr *a, double dt, const double *ddt) {
  using namespace cup2d;
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc = fast_setup(a);
  if (rc) return rc;
  if ((rc = amr_dist_refresh(a, CUP2D_PRES))) return rc;
  const int grid = (int)((a->nb + A1_WARPS * 4 - 1) / (A1_WARPS * 4));
  with_scalar(dt, ddt, [&](auto d) {
    amr_scalar_fast_kernel<1><<<grid, A1_NT, 0, a->stream>>>(a->f[CUP2D_PRES], a->f[CUP2D_TMPV], reinterpret_cast<const int4 *>(a->d_nbr4),
                                                             a->d_irr_of, a->gt[2], a->d_h, flux_buf<1>(a), (int)a->nb, d);
    return 0;
  });
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

// The tables of the 16 x 16 {-4,-4,5,5,tensorial} labs (the tagging kernel above, the force diagnostics of amr_forces.cu), on
// first use and until a regrid: the fast tables, the 8-neighbour table and the compact ghost rows of kind 3.  A distributed
// context keeps the rows of its own blocks and names every neighbour and source by its local slot.
int amr_lab16_tables(cup2d_amr *a) {
  using namespace cup2d;
  int rc = fast_setup(a);
  if (rc) return rc;
  if (!a->d_nbr8) { // same-level neighbours by slot (the halo set holds them); walls and level jumps keep their codes
    std::vector<int32_t> n8;
    if ((rc = plan_neighbours(a, n8))) return rc;
    n8.erase(n8.begin() + 8 * (a->gbegin + a->nb), n8.end());
    n8.erase(n8.begin(), n8.begin() + 8 * a->gbegin);
    for (auto &g : n8)
      if (g >= 0 && (g = a->slot(g)) < 0) {
        set_error("distributed context: a lab source lies outside the halo set");
        return CUP2D_EINVAL;
      }
    CUP2D_CUDA(upload(&a->d_nbr8, n8));
  }
  return a->gt[3].grow ? CUP2D_OK : amr_ghost_rows(a, 3);
}

// adapt()'s tagging on the fast tables: tmp, and the per-block L-inf in d_part (vel and chi refreshed by the caller).  Its
// ghost rows of kinds 1 and 3 sum their terms in the full tables' order (gt_src), so that every lab value is the baseline's.
int amr_tags_fast(cup2d_amr *a, double rtol, double h_finest) {
  using namespace cup2d;
  int rc = amr_lab16_tables(a);
  if (rc) return rc;
  for (int which : {1, 3})
    if (!a->gt_src[which].grow && (rc = amr_ghost_rows(a, which, true))) return rc;
  const int grid = (int)((a->nb + A1_WARPS * 4 - 1) / (A1_WARPS * 4));
  amr_tags_fast_kernel<<<grid, A1_NT, 0, a->stream>>>(a->f[CUP2D_VEL], a->f[CUP2D_CHI], a->f[CUP2D_TMP], reinterpret_cast<const int4 *>(a->d_nbr4),
                                                      a->d_nbr8, a->d_irr_of, a->gt_src[1], a->gt_src[3], a->d_h, h_finest, rtol, a->d_part, (int)a->nb);
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

using namespace cup2d;

extern "C" {

/* tmpV = KernelAdvectDiffuse(vel), flux-corrected (main.cpp:6611-6617): same result as cup2d_amr_advect_diffuse_rhs */
int cup2d_amr_advect_diffuse_rhs_fast(cup2d_amr *a, double dt) {
  if (!a) {
    set_error("null cup2d_amr handle");
    return CUP2D_EINVAL;
  }
  return amr_advect_rhs_fast(a, dt, nullptr);
}

/* same results as cup2d_amr_pressure_rhs / cup2d_amr_pressure_gradient through per-block +-1 labs in shared memory */
int cup2d_amr_pressure_rhs_fast(cup2d_amr *a, double dt, int with_laplacian) {
  if (!a) {
    set_error("null cup2d_amr handle");
    return CUP2D_EINVAL;
  }
  return amr_pressure_rhs_fast(a, dt, with_laplacian, nullptr);
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
                                                           a->d_irr_of, a->gt[2], a->d_h, flux_buf<1>(a), (int)a->nb, ByValue{dt});
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
  return amr_pressure_gradient_fast(a, dt, nullptr);
}

} // extern "C"
