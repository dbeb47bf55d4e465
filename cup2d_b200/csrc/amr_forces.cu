// Surface normals and force diagnostics on a multi-level mesh (main.cpp:3774-3828 and 5573-5746 with the reductions of
// 7188-7284) on the obstacle blocks the device holds, so that a caller no longer downloads vel, pres and chi for them.
//
// cup2d_amr_surface(a, n): ComputeSurfaceNormals as ongrid() calls it (4470), on chi and tmp as they stand.  Kernel:
//   amr_surface_kernel  one CTA per (shape, obstacle block), one thread per cell: the +-1 labs of chi and tmp as
//                       PutChiOnGrid builds its lab (csrc/amr_ongrid.cu: same-level copies, wall rules, the plan's kind-2 ghost
//                       rows at level jumps), then the reference's tests (|grad chi|^2 < 1e-12, |D| > EPS, h = h0 / 2^level);
//                       the points are compacted in (iy, ix) order into the block's 64 slots, the count per block alongside.
//   The reference reads its lab rows without their offset (3796-3801): cell (x0, y0) takes the chi / tmp differences at
//   (x0 +- 1, y0 - 1) and (x0 - 1, y0 +- 1), so cells (0,0), (7,0) and (0,7) read a corner ghost of the cross-shaped lab.  No
//   rule writes those corners on a block away from the walls; the reference's BlockLab keeps there what the last block loaded
//   with a wall ghost left, which is chi = 0 and tmp = -1 while the bodies stay away from the walls.  Those are the values
//   used here; corners the wall rule writes are the wall rule's.
//   One host wait, for the counts (the host scans them into each shape's offsets).
// cup2d_amr_forces(a, n, shapes, out): KernelComputeForces and the reductions.  Kernels:
//   amr_forces_kernel   one CTA per (shape, obstacle block), one thread per surface point: the vector lab of vel and the
//                       scalar lab of chi, both {-4,-4,5,5,tensorial} (16 x 16, plan kinds 6 and 3), in shared memory: regular
//                       blocks from the 8-neighbour table with the wall rules, irregular blocks from the compact ghost rows;
//                       each thread the reference's point computation in its expression order; then one thread per accumulated
//                       quantity adds the points in order (the reference's serial chain), and PoutNew (5743).
//   amr_forces_sum_kernel  per shape, one thread per quantity: the blocks in ascending id order (7210-7231), as the reference's
//                       shape sums, which on one rank are its MPI_Allreduce of 19.
//   The four derived quantities (7273-7280) on the host.  One host wait.
// The file is compiled without FMA contraction, device (-fmad=false) and host (-ffp-contract=off) code alike (Makefile), like
// the reference's host build, so every expression rounds as it does there.
#include "sim.h"
#include "amr.h"
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <string>
#include <type_traits>
#include <vector>

extern "C" {
int64_t cup2d_amr_plan_ghosts(cup2d_amr_plan *p, int which, int64_t *nrows, int64_t *rowptr, int32_t *dst, int32_t *src_block,
                              int32_t *src_cellcomp, double *weight);
int cup2d_amr_plan_neighbours(cup2d_amr_plan *p, int32_t *out);
int64_t cup2d_amr_plan_irregular(cup2d_amr_plan *p, int32_t *blocks_out);
}

namespace cup2d {

constexpr int FO_MAXSH = 64;
constexpr int FO_NQ = 18;  // accumulated per point (PoutNew is formed from forcex, forcey)
constexpr double FO_CHI_CORNER = 0.0, FO_TMP_CORNER = -1.0; // the unwritten corner ghosts of the normals' labs (see above)

struct FoShapes {             // every shape's obstacle blocks and surface storage; CTA b belongs to shape s if first[s] <= b < first[s+1]
  const int *ids[FO_MAXSH];
  const double *udef[FO_MAXSH];
  int *ixy[FO_MAXSH], *cnt[FO_MAXSH];
  double *nrm[FO_MAXSH], *skin[FO_MAXSH];
  int first[FO_MAXSH + 1];
  int nshapes;
};
struct FoMotion { double u, v, cx, cy, vu0, vu1; }; // main.cpp:5595-5598

__device__ __forceinline__ void fo_which(const FoShapes &S, int b, int &s, int &k) {
  s = 0;
  while (s + 1 < S.nshapes && S.first[s + 1] <= b) s++;
  k = b - S.first[s];
}

// ComputeSurfaceNormals (main.cpp:3786-3812) for one obstacle block of one shape; thread = cell (x0, y0)
__global__ void __launch_bounds__(64)
amr_surface_kernel(const FoShapes S, const double *__restrict__ chi, const double *__restrict__ tmp, const double *__restrict__ hb,
                   const int4 *__restrict__ nbr4, const int *__restrict__ irr_of, const GhostDev gt) {
  __shared__ double lc[100];
  __shared__ double lt[100];
  __shared__ int s_f[64];
  const int t = threadIdx.x, ix = t & 7, iy = t >> 3;
  int s, k;
  fo_which(S, blockIdx.x, s, k);
  const int id = S.ids[s][k];
  for (int c = t; c < 100; c += 64) lc[c] = FO_CHI_CORNER, lt[c] = FO_TMP_CORNER;
  __syncthreads();
  lc[(iy + 1) * 10 + ix + 1] = chi[(size_t)id * 64 + t];
  lt[(iy + 1) * 10 + ix + 1] = tmp[(size_t)id * 64 + t];
  const int4 nbk = nbr4[id];
  if (t < 32) { // one ghost layer per face: same-level neighbour -> copy, wall -> the wall-adjacent cell (main.cpp:3239-3244)
    const int f = t >> 3, p = t & 7;
    const int nbf = f == 0 ? nbk.x : f == 1 ? nbk.y : f == 2 ? nbk.z : nbk.w;
    if (nbf >= -1) {
      int gx, gy, sx, sy;
      if (f < 2) gx = f == 0 ? -1 : 8, gy = p, sx = nbf >= 0 ? (f == 0 ? 7 : 0) : (f == 0 ? 0 : 7), sy = p;
      else gx = p, gy = f == 2 ? -1 : 8, sx = p, sy = nbf >= 0 ? (f == 2 ? 7 : 0) : (f == 2 ? 0 : 7);
      const size_t src = (size_t)(nbf >= 0 ? nbf : id) * 64 + sy * 8 + sx;
      lc[(gy + 1) * 10 + gx + 1] = chi[src];
      lt[(gy + 1) * 10 + gx + 1] = tmp[src];
    }
  } else if (t < 36 && irr_of[id] < 0) { // corners of a regular block that the wall rule writes (the x walls first, then y)
    const int c = t - 32, gx = c & 1 ? 8 : -1, gy = c & 2 ? 8 : -1;
    const bool wx = (gx < 0 ? nbk.x : nbk.y) == -1, wy = (gy < 0 ? nbk.z : nbk.w) == -1;
    if (wx || wy) {
      const int cx = wx ? (gx < 0 ? 0 : 7) : gx, cy = wy ? (gy < 0 ? 0 : 7) : gy;
      int b = id, px = cx, py = cy;
      if (cx < 0 || cx > 7) b = gx < 0 ? nbk.x : nbk.y, px = gx < 0 ? 7 : 0;
      else if (cy < 0 || cy > 7) b = gy < 0 ? nbk.z : nbk.w, py = gy < 0 ? 7 : 0;
      lc[(gy + 1) * 10 + gx + 1] = chi[(size_t)b * 64 + py * 8 + px];
      lt[(gy + 1) * 10 + gx + 1] = tmp[(size_t)b * 64 + py * 8 + px];
    }
  }
  __syncthreads();
  const int qi = irr_of[id];
  if (qi >= 0) // coarser / finer neighbours: the ghost rows of the plan (kind 2), applied to both fields
    for (int64_t row = gt.grow[qi] + t; row < gt.grow[qi + 1]; row += 64) {
      double ac = 0.0, at = 0.0;
      for (int64_t e = gt.rowptr[row]; e < gt.rowptr[row + 1]; e++) {
        const size_t src = (size_t)gt.sb[e] * 64 + gt.sc[e];
        ac += gt.w[e] * chi[src];
        at += gt.w[e] * tmp[src];
      }
      lc[gt.dst[row] % 100] = ac;
      lt[gt.dst[row] % 100] = at;
    }
  __syncthreads();
  const double h = hb[id], i2h = 0.5 / h, fac = 0.5 * h;
  // main.cpp:3792-3797: lab row y0 (not y0 + 1), columns x0 + 2 and x0
  const double gradHX = lc[10 * iy + ix + 2] - lc[10 * iy + ix];
  const double gradHY = lc[10 * (iy + 2) + ix] - lc[10 * iy + ix];
  bool hit = false;
  double dx = 0, dy = 0, D = 0;
  if (!(gradHX * gradHX + gradHY * gradHY < 1e-12)) {
    const double gradUX = i2h * (lt[10 * iy + ix + 2] - lt[10 * iy + ix]);
    const double gradUY = i2h * (lt[10 * (iy + 2) + ix] - lt[10 * iy + ix]);
    const double gradUSq = (gradUX * gradUX + gradUY * gradUY) + DBL_EPSILON;
    D = fac * (gradHX * gradUX + gradHY * gradUY) / gradUSq;
    if (fabs(D) > DBL_EPSILON) {
      hit = true;
      dx = -D * gradUX, dy = -D * gradUY;
    }
  }
  s_f[t] = hit;
  __syncthreads();
  int pos = 0; // points before this cell in (iy, ix) order
  for (int j = 0; j < t; j++) pos += s_f[j];
  if (hit) {
    const size_t slot = (size_t)k * 64 + pos;
    S.ixy[s][2 * slot] = ix, S.ixy[s][2 * slot + 1] = iy;
    S.nrm[s][3 * slot] = dx, S.nrm[s][3 * slot + 1] = dy, S.nrm[s][3 * slot + 2] = D;
  }
  if (t == 63) S.cnt[s][k] = pos + hit;
}

// the 16 x 16 labs {-4,-4,5,5,tensorial} of vel (vector wall rule) and chi (scalar) of block id; lab index (y + 4) * 16 + x + 4
__device__ __forceinline__ void fo_labs(int id, const double *__restrict__ vel, const double *__restrict__ chi,
                                        const int *__restrict__ nbr8, const int *__restrict__ irr_of, const GhostDev &gv,
                                        const GhostDev &gc, double *lv, double *lx) {
  const int t = threadIdx.x;
  const int qi = irr_of[id];
  const int *n8 = nbr8 + (size_t)id * 8; // (-1,-1),(0,-1),(1,-1),(-1,0),(1,0),(-1,1),(0,1),(1,1)
  for (int c = t; c < 256; c += 64) {
    const int gx = (c & 15) - 4, gy = (c >> 4) - 4;
    const int ox = gx < 0 ? -1 : gx > 7, oy = gy < 0 ? -1 : gy > 7;
    if (ox == 0 && oy == 0) {
      const size_t src = (size_t)id * 64 + gy * 8 + gx;
      lv[2 * c] = vel[2 * src], lv[2 * c + 1] = vel[2 * src + 1], lx[c] = chi[src];
      continue;
    }
    if (qi >= 0) continue; // irregular: the ghost rows below
    // regular block: clamp the directions that face a domain wall (the wall-adjacent cell, normal component negated), then
    // read the cell from the block or its same-level neighbour
    const bool wx = ox != 0 && n8[ox < 0 ? 3 : 4] == -1, wy = oy != 0 && n8[oy < 0 ? 1 : 6] == -1;
    const int cx = wx ? (ox < 0 ? 0 : 7) : gx, cy = wy ? (oy < 0 ? 0 : 7) : gy;
    const int qx = cx < 0 ? -1 : cx > 7, qy = cy < 0 ? -1 : cy > 7;
    const int b = qx == 0 && qy == 0 ? id : n8[(qy + 1) * 3 + (qx + 1) - ((qy + 1) * 3 + (qx + 1) > 4)];
    const size_t src = (size_t)b * 64 + (cy & 7) * 8 + (cx & 7);
    const double u = vel[2 * src], v = vel[2 * src + 1];
    lv[2 * c] = wx ? -u : u, lv[2 * c + 1] = wy ? -v : v, lx[c] = chi[src];
  }
  if (qi < 0) return;
  __syncthreads();
  for (int64_t row = gv.grow[qi] + t; row < gv.grow[qi + 1]; row += 64) {
    double acc = 0.0;
    for (int64_t e = gv.rowptr[row]; e < gv.rowptr[row + 1]; e++) acc += gv.w[e] * vel[(size_t)gv.sb[e] * 128 + gv.sc[e]];
    lv[gv.dst[row] % 512] = acc;
  }
  for (int64_t row = gc.grow[qi] + t; row < gc.grow[qi + 1]; row += 64) {
    double acc = 0.0;
    for (int64_t e = gc.rowptr[row]; e < gc.rowptr[row + 1]; e++) acc += gc.w[e] * chi[(size_t)gc.sb[e] * 64 + gc.sc[e]];
    lx[gc.dst[row] % 256] = acc;
  }
}

// KernelComputeForces (main.cpp:5595-5743) for one obstacle block of one shape; thread = surface point.  part[b][19] in the
// order of quantities[19] (7233-7251)
__global__ void __launch_bounds__(64, 4) // (64) alone makes ptxas spill at 80 registers
amr_forces_kernel(const FoShapes S, const FoMotion *__restrict__ mo, const double *__restrict__ vel, const double *__restrict__ pres,
                  const double *__restrict__ chi, const double *__restrict__ hb, const int2 *__restrict__ ij, const int *__restrict__ nbr8,
                  const int *__restrict__ irr_of, const GhostDev gv, const GhostDev gc, double nu, double *__restrict__ part) {
  __shared__ double lv[512];
  __shared__ double lx[256];
  __shared__ double s_q[FO_NQ * 64];
  const int t = threadIdx.x;
  int s, k;
  fo_which(S, blockIdx.x, s, k);
  const int id = S.ids[s][k], n = S.cnt[s][k];
  const FoMotion m = mo[s];
  if (n > 0) fo_labs(id, vel, chi, nbr8, irr_of, gv, gc, lv, lx);
  __syncthreads();
  if (t < n) {
    const size_t slot = (size_t)k * 64 + t;
    const int ix = S.ixy[s][2 * slot], iy = S.ixy[s][2 * slot + 1];
    const double normX = S.nrm[s][3 * slot], normY = S.nrm[s][3 * slot + 1];
    const double h = hb[id], NUoH = nu / h;
    const int2 b = ij[id];
    const double p0 = (double)(b.x * CUP2D_BS) * h + h * (ix + 0.5), p1 = (double)(b.y * CUP2D_BS) * h + h * (iy + 0.5);
    const double norm = 1.0 / sqrt(normX * normX + normY * normY);
    const double dx = normX * norm, dy = normY * norm;
    int x = ix, y = iy;
    for (int kk = 0; kk < 5; kk++) { // main.cpp:5620-5633
      const int dxi = (int)round(kk * dx), dyi = (int)round(kk * dy);
      if (ix + dxi + 1 >= CUP2D_BS + 5 - 1 || ix + dxi - 1 < -4) continue;
      if (iy + dyi + 1 >= CUP2D_BS + 5 - 1 || iy + dyi - 1 < -4) continue;
      x = ix + dxi, y = iy + dyi;
      if (lx[(y + 4) * 16 + x + 4] < 0.01) break;
    }
    const int sx = normX > 0 ? +1 : -1, sy = normY > 0 ? +1 : -1;
    auto inrange = [](int i) { return i >= -4 && i < CUP2D_BS + 5 - 1; };
    auto L = [&](int xx, int yy, int d) { return lv[2 * ((yy + 4) * 16 + xx + 4) + d]; };
    const double c0 = -137. / 60., c1 = 5., c2 = -5., c3 = 10. / 3., c4 = -5. / 4., c5 = 1. / 5.;
    double dveldx[2], dveldy[2], dveldx2[2], dveldy2[2], dveldxdy[2];
#pragma unroll
    for (int d = 0; d < 2; d++) {
      const double l00 = L(x, y, d);
      if (inrange(x + 5 * sx))
        dveldx[d] = sx * (c0 * l00 + c1 * L(x + sx, y, d) + c2 * L(x + 2 * sx, y, d) + c3 * L(x + 3 * sx, y, d) +
                          c4 * L(x + 4 * sx, y, d) + c5 * L(x + 5 * sx, y, d));
      else if (inrange(x + 2 * sx))
        dveldx[d] = sx * (-1.5 * l00 + 2.0 * L(x + sx, y, d) - 0.5 * L(x + 2 * sx, y, d));
      else
        dveldx[d] = sx * (L(x + sx, y, d) - l00);
      if (inrange(y + 5 * sy))
        dveldy[d] = sy * (c0 * l00 + c1 * L(x, y + sy, d) + c2 * L(x, y + 2 * sy, d) + c3 * L(x, y + 3 * sy, d) +
                          c4 * L(x, y + 4 * sy, d) + c5 * L(x, y + 5 * sy, d));
      else if (inrange(y + 2 * sy))
        dveldy[d] = sy * (-1.5 * l00 + 2.0 * L(x, y + sy, d) - 0.5 * L(x, y + 2 * sy, d));
      else
        dveldy[d] = sx * (L(x, y + sy, d) - l00); // sx, as main.cpp:5679
      dveldx2[d] = L(x - 1, y, d) - 2.0 * l00 + L(x + 1, y, d);
      dveldy2[d] = L(x, y - 1, d) - 2.0 * l00 + L(x, y + 1, d);
      if (inrange(x + 2 * sx) && inrange(y + 2 * sy))
        dveldxdy[d] = sx * sy *
                      (-0.5 * (-1.5 * L(x + 2 * sx, y, d) + 2 * L(x + 2 * sx, y + sy, d) - 0.5 * L(x + 2 * sx, y + 2 * sy, d)) +
                       2 * (-1.5 * L(x + sx, y, d) + 2 * L(x + sx, y + sy, d) - 0.5 * L(x + sx, y + 2 * sy, d)) -
                       1.5 * (-1.5 * l00 + 2 * L(x, y + sy, d) - 0.5 * L(x, y + 2 * sy, d)));
      else
        dveldxdy[d] = sx * sy * (L(x + sx, y + sy, d) - L(x + sx, y, d)) - (L(x, y + sy, d) - l00);
    }
    const double DuDx = dveldx[0] + dveldx2[0] * (ix - x) + dveldxdy[0] * (iy - y);
    const double DvDx = dveldx[1] + dveldx2[1] * (ix - x) + dveldxdy[1] * (iy - y);
    const double DuDy = dveldy[0] + dveldy2[0] * (iy - y) + dveldxdy[0] * (ix - x);
    const double DvDy = dveldy[1] + dveldy2[1] * (iy - y) + dveldxdy[1] * (ix - x);
    const double P = pres[(size_t)id * 64 + iy * 8 + ix];
    const double fXV = NUoH * DuDx * normX + NUoH * DuDy * normY, fXP = -P * normX;
    const double fYV = NUoH * DvDx * normX + NUoH * DvDy * normY, fYP = -P * normY;
    const double fXT = fXV + fXP, fYT = fYV + fYP;
    const double us = L(ix, iy, 0), vs = L(ix, iy, 1);
    const double2 U = reinterpret_cast<const double2 *>(S.udef[s])[(size_t)k * 64 + iy * 8 + ix];
    double *sk = S.skin[s] + slot * 14;
    sk[0] = p0, sk[1] = p1, sk[2] = P, sk[3] = us, sk[4] = vs, sk[5] = dx, sk[6] = dy, sk[7] = (DvDx - DuDy) / h;
    sk[8] = U.x, sk[9] = U.y;
    sk[10] = -P * dx + NUoH * DuDx * dx + NUoH * DuDy * dy;
    sk[11] = -P * dy + NUoH * DvDx * dx + NUoH * DvDy * dy;
    sk[12] = NUoH * DuDx * dx + NUoH * DuDy * dy;
    sk[13] = NUoH * DvDx * dx + NUoH * DvDy * dy;
    const double forcePar = fXT * m.vu0 + fYT * m.vu1;
    const double powOut = fXT * us + fYT * vs, powDef = fXT * U.x + fYT * U.y;
    // the 18 accumulated terms, in the slots of quantities[19] without PoutNew (9); drag is subtracted
    double *sq = s_q + t;
    sq[0 * 64] = normX * vs - normY * us;
    sq[1 * 64] = sqrt(normX * normX + normY * normY);
    sq[2 * 64] = fXT;
    sq[3 * 64] = fXP;
    sq[4 * 64] = fXV;
    sq[5 * 64] = (p0 - m.cx) * fYP - (p1 - m.cy) * fXP;
    sq[6 * 64] = .5 * (forcePar - fabs(forcePar));
    sq[7 * 64] = fXT * m.vu1 - fYT * m.vu0;
    sq[8 * 64] = powOut;
    sq[9 * 64] = powOut < 0.0 ? powOut : 0.0; // std::min((Real)0, powOut)
    sq[10 * 64] = (p0 - m.cx) * fYT - (p1 - m.cy) * fXT;
    sq[11 * 64] = fYT;
    sq[12 * 64] = fYP;
    sq[13 * 64] = fYV;
    sq[14 * 64] = (p0 - m.cx) * fYV - (p1 - m.cy) * fXV;
    sq[15 * 64] = .5 * (forcePar + fabs(forcePar));
    sq[16 * 64] = powDef < 0.0 ? powDef : 0.0; // std::min((Real)0, powDef)
    sq[17 * 64] = powDef;
  }
  __syncthreads();
  double *pb = part + (size_t)blockIdx.x * 19;
  if (t < FO_NQ) { // the reference's per-block chains: each quantity's points in order
    double acc = 0.0;
    const double *sq = s_q + t * 64;
    if (t == 6)
      for (int j = 0; j < n; j++) acc -= sq[j];
    else
      for (int j = 0; j < n; j++) acc += sq[j];
    pb[t < 9 ? t : t + 1] = acc;
  }
  __syncthreads();
  if (t == 0) pb[9] = pb[2] * m.u + pb[12] * m.v; // PoutNew = forcex * u + forcey * v (main.cpp:5743)
}

// main.cpp:7190-7231 per shape: the blocks in ascending id order, one chain per quantity
__global__ void __launch_bounds__(32)
amr_forces_sum_kernel(const FoShapes S, const double *__restrict__ part, double *__restrict__ sums) {
  const int s = blockIdx.x, q = threadIdx.x;
  if (q >= 19) return;
  double acc = 0.0;
  for (int b = S.first[s]; b < S.first[s + 1]; b++) acc += part[(size_t)b * 19 + q];
  sums[(size_t)s * 19 + q] = acc;
}

static int fo_grow(void **p, size_t *cap, size_t bytes) {
  if (bytes <= *cap) return CUP2D_OK;
  cudaFree(*p);
  *p = nullptr, *cap = 0;
  CUP2D_CUDA(cudaMalloc(p, bytes));
  *cap = bytes;
  return CUP2D_OK;
}

// the force labs' tables, on first use and until a regrid: the 8-neighbour table and the compact ghost rows of kinds 6 and 3
static int fo_tables(cup2d_amr *a) {
  int rc = amr_fast_tables(a);
  if (rc) return rc;
  auto up = [](auto **d, const auto &h) -> cudaError_t {
    using T = typename std::remove_reference<decltype(h[0])>::type;
    cudaError_t e = cudaMalloc(d, std::max<size_t>(h.size(), 1) * sizeof(T));
    if (e != cudaSuccess) return e;
    return cudaMemcpy(*d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice);
  };
  if (!a->d_nbr8) {
    std::vector<int32_t> n8((size_t)8 * a->nb);
    if (cup2d_amr_plan_neighbours(a->plan, n8.data())) return CUP2D_EINVAL;
    CUP2D_CUDA(up(&a->d_nbr8, n8));
  }
  const int64_t nirr = cup2d_amr_plan_irregular(a->plan, nullptr);
  for (int which : {3, 6}) {
    GhostDev &g = a->gt[which];
    if (g.grow) continue;
    const int ncell = which == 6 ? 16 * 16 * 2 : 16 * 16;
    int64_t nrows = 0;
    const int64_t nnz = cup2d_amr_plan_ghosts(a->plan, which, &nrows, nullptr, nullptr, nullptr, nullptr, nullptr);
    if (nnz < 0) return CUP2D_EINVAL;
    std::vector<int64_t> rp(nrows + 1), grow(nirr + 1, nrows);
    std::vector<int32_t> dst(std::max<int64_t>(nrows, 1)), sb(std::max<int64_t>(nnz, 1)), sc(std::max<int64_t>(nnz, 1));
    std::vector<double> w(std::max<int64_t>(nnz, 1));
    cup2d_amr_plan_ghosts(a->plan, which, &nrows, rp.data(), dst.data(), sb.data(), sc.data(), w.data());
    for (int64_t row = nrows - 1; row >= 0; row--) grow[dst[row] / ncell] = row; // rows are grouped by block, in order
    for (int64_t qi = nirr - 1; qi >= 0; qi--) grow[qi] = std::min(grow[qi], grow[qi + 1]);
    CUP2D_CUDA(up(&g.rowptr, rp));
    CUP2D_CUDA(up(&g.dst, dst));
    CUP2D_CUDA(up(&g.sb, sb));
    CUP2D_CUDA(up(&g.sc, sc));
    CUP2D_CUDA(up(&g.w, w));
    CUP2D_CUDA(up(&g.grow, grow)); // last: marks the table complete
  }
  return CUP2D_OK;
}

static int fo_check(cup2d_amr *a, int nshapes, const char *who) {
  if (!a || nshapes < 1 || nshapes > FO_MAXSH) {
    set_error(std::string(who) + ": bad arguments (1..64 shapes)");
    return CUP2D_EINVAL;
  }
  if (a->dist || a->nranks > 1) {
    set_error(std::string(who) + ": contexts on several ranks are not supported");
    return CUP2D_ESTATE;
  }
  for (int s = 0; s < nshapes; s++)
    if (s >= (int)a->shapes.size()) {
      set_error(std::string(who) + ": shape " + std::to_string(s) + " has not been set");
      return CUP2D_EINVAL;
    }
  return CUP2D_OK;
}

static FoShapes fo_shapes(cup2d_amr *a, int nshapes) {
  FoShapes S = {};
  S.nshapes = nshapes;
  for (int s = 0; s < nshapes; s++) {
    const cup2d_amr::Shape &sh = a->shapes[s];
    const cup2d_amr::Surface &q = a->surf[s];
    S.ids[s] = sh.d_ids, S.udef[s] = sh.d_udef;
    S.ixy[s] = q.d_ixy, S.cnt[s] = q.d_cnt, S.nrm[s] = q.d_nrm, S.skin[s] = q.d_skin;
    S.first[s + 1] = S.first[s] + sh.nob;
  }
  return S;
}

} // namespace cup2d

using namespace cup2d;

extern "C" {

int cup2d_amr_surface(cup2d_amr *a, int nshapes) {
  int rc = fo_check(a, nshapes, "cup2d_amr_surface");
  if (rc) return rc;
  CUP2D_CUDA(cudaSetDevice(a->device));
  if ((rc = amr_fast_tables(a))) return rc;
  if (a->surf.size() < a->shapes.size()) a->surf.resize(a->shapes.size());
  for (int s = 0; s < nshapes; s++) { // 64 point slots per obstacle block
    cup2d_amr::Surface &q = a->surf[s];
    const int nob = a->shapes[s].nob;
    if (nob > q.cap || !q.d_cnt) {
      cudaFree(q.d_ixy); cudaFree(q.d_cnt); cudaFree(q.d_nrm); cudaFree(q.d_skin);
      q.d_ixy = q.d_cnt = nullptr, q.d_nrm = q.d_skin = nullptr, q.cap = 0;
      const size_t cap = (size_t)std::max(nob, 1);
      CUP2D_CUDA(cudaMalloc(&q.d_ixy, cap * 64 * 2 * sizeof(int)));
      CUP2D_CUDA(cudaMalloc(&q.d_cnt, cap * sizeof(int)));
      CUP2D_CUDA(cudaMalloc(&q.d_nrm, cap * 64 * 3 * sizeof(double)));
      CUP2D_CUDA(cudaMalloc(&q.d_skin, cap * 64 * 14 * sizeof(double)));
      q.cap = (int)cap;
    }
    a->shapes[s].has_surface = false;
  }
  const FoShapes S = fo_shapes(a, nshapes);
  for (int s = 0; s < nshapes; s++) // the skin of the last cup2d_amr_forces call: none yet
    if (a->shapes[s].nob) CUP2D_CUDA(cudaMemsetAsync(a->surf[s].d_skin, 0, (size_t)a->shapes[s].nob * 64 * 14 * sizeof(double), a->stream));
  const int total = S.first[nshapes];
  if (total > 0)
    amr_surface_kernel<<<total, 64, 0, a->stream>>>(S, a->f[CUP2D_CHI], a->f[CUP2D_TMP], a->d_h, reinterpret_cast<const int4 *>(a->d_nbr4),
                                                    a->d_irr_of, a->gt[2]);
  CUP2D_CUDA(cudaGetLastError());
  std::vector<int> cnt(std::max(total, 1));
  for (int s = 0; s < nshapes; s++)
    if (a->shapes[s].nob)
      CUP2D_CUDA(cudaMemcpyAsync(cnt.data() + S.first[s], a->surf[s].d_cnt, (size_t)a->shapes[s].nob * sizeof(int), cudaMemcpyDeviceToHost,
                                 a->stream));
  CUP2D_CUDA(cudaStreamSynchronize(a->stream));
  for (int s = 0; s < nshapes; s++) {
    a->surf[s].cnt.assign(cnt.begin() + S.first[s], cnt.begin() + S.first[s + 1]);
    a->shapes[s].has_surface = true;
  }
  return CUP2D_OK;
}

int64_t cup2d_amr_surface_get(cup2d_amr *a, int shape, int32_t *block, int32_t *ixy, double *normal, double *skin) {
  if (!a || shape < 0 || shape >= (int)a->shapes.size()) {
    set_error("cup2d_amr_surface_get: no such shape");
    return CUP2D_EINVAL;
  }
  if (!a->shapes[shape].has_surface) {
    set_error("cup2d_amr_surface_get: no surface points (cup2d_amr_surface after the shape was last set)");
    return CUP2D_ESTATE;
  }
  const cup2d_amr::Shape &sh = a->shapes[shape];
  const cup2d_amr::Surface &q = a->surf[shape];
  int64_t n = 0;
  for (int c : q.cnt) n += c;
  if (n == 0 || !(block || ixy || normal || skin)) return n;
  CUP2D_CUDA(cudaSetDevice(a->device));
  const size_t ns = (size_t)sh.nob * 64;
  std::vector<int32_t> ids(sh.nob), hixy(ns * 2);
  std::vector<double> hn(normal ? ns * 3 : 0), hs(skin ? ns * 14 : 0);
  CUP2D_CUDA(cudaMemcpyAsync(ids.data(), sh.d_ids, (size_t)sh.nob * sizeof(int), cudaMemcpyDeviceToHost, a->stream));
  CUP2D_CUDA(cudaMemcpyAsync(hixy.data(), q.d_ixy, ns * 2 * sizeof(int), cudaMemcpyDeviceToHost, a->stream));
  if (normal) CUP2D_CUDA(cudaMemcpyAsync(hn.data(), q.d_nrm, ns * 3 * sizeof(double), cudaMemcpyDeviceToHost, a->stream));
  if (skin) CUP2D_CUDA(cudaMemcpyAsync(hs.data(), q.d_skin, ns * 14 * sizeof(double), cudaMemcpyDeviceToHost, a->stream));
  CUP2D_CUDA(cudaStreamSynchronize(a->stream));
  int64_t o = 0;
  for (int k = 0; k < sh.nob; k++)
    for (int j = 0; j < q.cnt[k]; j++, o++) {
      const size_t slot = (size_t)k * 64 + j;
      if (block) block[o] = ids[k];
      if (ixy) ixy[2 * o] = hixy[2 * slot], ixy[2 * o + 1] = hixy[2 * slot + 1];
      if (normal) memcpy(normal + 3 * o, hn.data() + 3 * slot, 3 * sizeof(double));
      if (skin) memcpy(skin + 14 * o, hs.data() + 14 * slot, 14 * sizeof(double));
    }
  return n;
}

int cup2d_amr_forces(cup2d_amr *a, int nshapes, const cup2d_rigid *shapes, double *out) {
  int rc = fo_check(a, nshapes, "cup2d_amr_forces");
  if (rc) return rc;
  if (!shapes || !out) {
    set_error("cup2d_amr_forces: null shapes or out");
    return CUP2D_EINVAL;
  }
  for (int s = 0; s < nshapes; s++)
    if (!a->shapes[s].has_surface) {
      set_error("cup2d_amr_forces: shape " + std::to_string(s) + " has no surface points (cup2d_amr_surface after it was last set)");
      return CUP2D_ESTATE;
    }
  std::vector<FoMotion> mo(nshapes);
  for (int s = 0; s < nshapes; s++) { // main.cpp:5595-5598
    const double u = shapes[s].u, v = shapes[s].v, vel_norm = std::sqrt(u * u + v * v);
    mo[s] = FoMotion{u, v, shapes[s].center_of_mass[0], shapes[s].center_of_mass[1], vel_norm > 0 ? u / vel_norm : 0.0,
                     vel_norm > 0 ? v / vel_norm : 0.0};
  }
  CUP2D_CUDA(cudaSetDevice(a->device));
  if ((rc = fo_tables(a)) || (rc = amr_ensure_ij(a))) return rc;
  const FoShapes S = fo_shapes(a, nshapes);
  const int total = S.first[nshapes];
  const size_t b_part = ((size_t)total * 19 + (size_t)nshapes * 19) * sizeof(double);
  if ((rc = fo_grow((void **)&a->d_fo_part, &a->fo_part_cap, b_part + nshapes * sizeof(FoMotion)))) return rc;
  double *d_sums = a->d_fo_part + (size_t)total * 19;
  FoMotion *d_mo = reinterpret_cast<FoMotion *>(d_sums + (size_t)nshapes * 19);
  CUP2D_CUDA(cudaMemcpyAsync(d_mo, mo.data(), nshapes * sizeof(FoMotion), cudaMemcpyHostToDevice, a->stream));
  if (total > 0)
    amr_forces_kernel<<<total, 64, 0, a->stream>>>(S, d_mo, a->f[CUP2D_VEL], a->f[CUP2D_PRES], a->f[CUP2D_CHI], a->d_h,
                                                   reinterpret_cast<const int2 *>(a->d_ij), a->d_nbr8, a->d_irr_of, a->gt[6],
                                                   a->gt[3], a->nu, a->d_fo_part);
  amr_forces_sum_kernel<<<nshapes, 32, 0, a->stream>>>(S, a->d_fo_part, d_sums);
  CUP2D_CUDA(cudaGetLastError());
  std::vector<double> q19((size_t)nshapes * 19);
  CUP2D_CUDA(cudaMemcpyAsync(q19.data(), d_sums, q19.size() * sizeof(double), cudaMemcpyDeviceToHost, a->stream));
  CUP2D_CUDA(cudaStreamSynchronize(a->stream));
  for (int s = 0; s < nshapes; s++) { // main.cpp:7273-7280
    const double *q = q19.data() + 19 * s;
    double *o = out + 23 * s;
    std::copy(q, q + 19, o);
    const double u = shapes[s].u, v = shapes[s].v;
    const double thrust = q[16], drag = q[6], defPowerBnd = q[17], defPower = q[18];
    const double Pthrust = thrust * std::sqrt(u * u + v * v), Pdrag = drag * std::sqrt(u * u + v * v);
    const double denUnb = Pthrust - std::min(defPower, 0.0), demBnd = Pthrust - defPowerBnd;
    o[19] = Pthrust, o[20] = Pdrag;
    o[21] = Pthrust / std::max(denUnb, DBL_EPSILON);
    o[22] = Pthrust / std::max(demBnd, DBL_EPSILON);
  }
  return CUP2D_OK;
}

} // extern "C"
