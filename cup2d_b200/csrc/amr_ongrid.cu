// Bodies on a multi-level mesh: ongrid()'s rasterisation of fish midlines (main.cpp:4019-4024, 4208-4556) on the device.
//
// cup2d_amr_ongrid(a, n, bodies, out) takes each shape's midline as ongrid() holds it after the kinematics (main.cpp:4208)
// and leaves chi, tmp and every shape's obstacle blocks (ids, chi, dist, udef) on the device, where cup2d_amr_shape_integrals /
// _penalize / _udef_assemble read them.  Host part, O(Nm) per shape: the rotation from the host libm, the AreaSegment boxes
// (main.cpp:3839-3878, 4216-4242) and one upload of midlines and segments.  Kernels (stable names, timed by name):
//   amr_ongrid_scan_kernel     chi = 0, tmp = -1 on every block (4019-4024) and every block against every segment of every shape
//                              (isIntersectingWithAABB, 3879-3909): one bit per shape and block, counts per CTA
//   amr_ongrid_offsets_kernel  exclusive scan of the counts per shape
//   amr_ongrid_compact_kernel  obstacle block ids in ascending block order (the reference's obstacleBlocks[id] order)
//   amr_ongrid_fish_kernel     PutFishOnBlocks (4271-4463): one CTA per obstacle block, one thread per cell; each thread walks
//                              the block's intersecting segments and their points in the reference's order and applies only the
//                              updates that land on its own cell, so the per-cell update sequence, and the result, is the
//                              reference's bit for bit; then u_def / chi, the signed square root of dist and tmp = max(tmp, dist)
//   amr_ongrid_chi_kernel      PutChiOnGrid (3911-3969) from the +-1 lab of tmp (same-level copies, wall copies, the plan's
//                              kind-2 ghost rows at level jumps); per-block Mass / COM partials, summed cell by cell in order
//   amr_ongrid_moments_kernel  the seven sums of 4489-4518 per block, cell by cell in order
//   amr_ongrid_correct_kernel  udef -= (u - a py, v + a px) (4541-4556)
//   amr_udef_blend_kernel      cup2d_amr_udef_blend: vel = vel (1 - chi) + tmpV chi before the time loop (6566-6575)
// The host adds the per-block partials in block order (as cup2d_amr_shape_integrals does).  On a distributed context
// (cup2d_amr_create_ranks) the kernels run over the rank's own blocks, tmp's halo slots are refreshed before the chi kernel
// (the neighbour table and ghost rows name slots), and the rank's partial sums are all-reduced (amr_dist_sum_vec) before
// the host uses them, as the reference's MPI_Allreduce at 4483 and 4520.  This file is compiled without FMA
// contraction (Makefile), like the reference (-O3, no -ffp-contract=fast on x86-64), so every expression rounds as it does there.
#include "sim.h"
#include "amr.h"
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <string>
#include <vector>

namespace cup2d {

constexpr int OG_SEG = 16;    // doubles per segment record: safe, normalI[2], normalJ[2], objBoxLabFr[2][2], objBoxObjFr[2][2], first, last
constexpr int OG_MID = 9;     // midline arrays per shape
constexpr int OG_SCAN = 128;  // blocks per CTA of the scan (one thread per block)
constexpr int OG_MAXSH = 64;

struct OgSegs {               // every shape's segments in the staged buffer
  const double *seg[OG_MAXSH];
  int nseg[OG_MAXSH];
  int nshapes;
};
struct OgShape {              // one shape for the per-shape kernels
  const double *mid, *seg;    // [9][nm], [nseg][OG_SEG]
  int nm, nseg;
  double R00, R01, R10, R11, px, py; // Rmatrix2D of PutFishOnBlocks (host cos / sin), position = center
  double cmx, cmy;            // centre of mass the sums are taken about
};
struct OgIds { int *ids[OG_MAXSH]; };
typedef unsigned long long og_u64;

__device__ __forceinline__ double og_max(double a, double b) { return a < b ? b : a; } // std::max
__device__ __forceinline__ double og_min(double a, double b) { return b < a ? b : a; } // std::min
__device__ __forceinline__ double og_sq(double a) { return a * a; }                   // std::pow(a, 2)

// AreaSegment::isIntersectingWithAABB (main.cpp:3879-3909) for the cell centres start..end of a block
__device__ __forceinline__ bool og_hit(const double *s, double st0, double st1, double en0, double en1) {
  const double w0 = (en0 - st0) / 2 + s[0], w1 = (en1 - st1) / 2 + s[0];
  const double c0 = (en0 + st0) / 2, c1 = (en1 + st1) / 2;
  if (og_min(s[6], c0 + w0) - og_max(s[5], c0 - w0) < 0 || og_min(s[8], c1 + w1) - og_max(s[7], c1 - w1) < 0) return false;
  const double X0 = w0 * s[1], Y0 = w1 * s[2], X1 = w0 * s[3], Y1 = w1 * s[4];
  if (og_min(c0 + X0 + Y0, s[10]) - og_max(c0 - X0 - Y0, s[9]) < 0 ||
      og_min(c1 + X1 + Y1, s[12]) - og_max(c1 - X1 - Y1, s[11]) < 0)
    return false;
  return true;
}

// chi = 0, tmp = -1 on the CTA's OG_SCAN blocks (16 B per cell), then one thread per block tests the segments of every shape
__global__ void __launch_bounds__(OG_SCAN)
amr_ongrid_scan_kernel(double *__restrict__ chi, double *__restrict__ tmp, const int2 *__restrict__ ij, const double *__restrict__ hb,
                       int nb, const OgSegs S, unsigned long long *__restrict__ mask, int *__restrict__ cnt) {
  __shared__ og_u64 s_bits[OG_SCAN];
  const int b0 = blockIdx.x * OG_SCAN, n = min(OG_SCAN, nb - b0);
  double2 *c2 = reinterpret_cast<double2 *>(chi) + (size_t)b0 * 32, *t2 = reinterpret_cast<double2 *>(tmp) + (size_t)b0 * 32;
  for (int i = threadIdx.x; i < n * 32; i += OG_SCAN) {
    c2[i] = make_double2(0.0, 0.0);
    t2[i] = make_double2(-1.0, -1.0);
  }
  unsigned long long bits = 0;
  const int k = b0 + threadIdx.x;
  if (threadIdx.x < n) {
    const double h = hb[k];
    const int2 b = ij[k];
    const double o0 = (double)(b.x * CUP2D_BS) * h, o1 = (double)(b.y * CUP2D_BS) * h;
    const double st0 = o0 + h * 0.5, st1 = o1 + h * 0.5, en0 = o0 + h * (CUP2D_BS - 0.5), en1 = o1 + h * (CUP2D_BS - 0.5);
    for (int s = 0; s < S.nshapes; s++)
      for (int q = 0; q < S.nseg[s]; q++)
        if (og_hit(S.seg[s] + (size_t)q * OG_SEG, st0, st1, en0, en1)) {
          bits |= 1ull << s;
          break;
        }
    mask[k] = bits;
  }
  s_bits[threadIdx.x] = bits;
  __syncthreads();
  if (threadIdx.x < S.nshapes) {
    int c = 0;
    for (int i = 0; i < n; i++) c += (int)((s_bits[i] >> threadIdx.x) & 1);
    cnt[(size_t)threadIdx.x * gridDim.x + blockIdx.x] = c;
  }
}

// cnt[shape][cta] -> exclusive offsets in place, totals[shape]: one CTA per shape, each thread a contiguous chunk of the
// counts, the chunk sums scanned in shared memory
constexpr int OG_OFF_NT = 256;
__global__ void __launch_bounds__(OG_OFF_NT)
amr_ongrid_offsets_kernel(int *__restrict__ cnt, int ncta, int *__restrict__ total) {
  __shared__ int s_sum[OG_OFF_NT];
  int *c = cnt + (size_t)blockIdx.x * ncta;
  const int chunk = (ncta + OG_OFF_NT - 1) / OG_OFF_NT, c0 = min(ncta, (int)threadIdx.x * chunk), c1 = min(ncta, c0 + chunk);
  int acc = 0;
  for (int i = c0; i < c1; i++) acc += c[i];
  s_sum[threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    int run = 0;
    for (int t = 0; t < OG_OFF_NT; t++) {
      const int v = s_sum[t];
      s_sum[t] = run;
      run += v;
    }
    total[blockIdx.x] = run;
  }
  __syncthreads();
  acc = s_sum[threadIdx.x];
  for (int i = c0; i < c1; i++) {
    const int v = c[i];
    c[i] = acc;
    acc += v;
  }
}

__global__ void __launch_bounds__(OG_SCAN)
amr_ongrid_compact_kernel(const unsigned long long *__restrict__ mask, const int *__restrict__ off, int nb, int nshapes, OgIds out) {
  __shared__ og_u64 s_bits[OG_SCAN];
  const int b0 = blockIdx.x * OG_SCAN, n = min(OG_SCAN, nb - b0);
  s_bits[threadIdx.x] = threadIdx.x < n ? mask[b0 + threadIdx.x] : 0ull;
  __syncthreads();
  if (threadIdx.x < nshapes) {
    const int s = threadIdx.x;
    int p = off[(size_t)s * gridDim.x + blockIdx.x];
    for (int i = 0; i < n; i++)
      if ((s_bits[i] >> s) & 1) out.ids[s][p++] = b0 + i;
  }
}

__device__ __forceinline__ void og_to_comp(const OgShape &S, double &x, double &y) { // changeToComputationalFrame
  const double p0 = x, p1 = y;
  x = S.R00 * p0 + S.R01 * p1;
  y = S.R10 * p0 + S.R11 * p1;
  x += S.px;
  y += S.py;
}
__device__ __forceinline__ void og_vel_to_comp(const OgShape &S, double &x, double &y) { // changeVelocityToComputationalFrame
  const double p0 = x, p1 = y;
  x = S.R00 * p0 + S.R01 * p1;
  y = S.R10 * p0 + S.R11 * p1;
}

// PutFishOnBlocks (main.cpp:4283-4461) for the obstacle blocks of one shape; thread = cell (ix, iy)
__global__ void __launch_bounds__(64)
amr_ongrid_fish_kernel(const OgShape S, const int *__restrict__ ids, const int2 *__restrict__ ij, const double *__restrict__ hb,
                       double *__restrict__ tmp, double *__restrict__ odist, double *__restrict__ ochi, double *__restrict__ oudef) {
  const int k = blockIdx.x, t = threadIdx.x, ix = t & 7, iy = t >> 3, nm = S.nm;
  const int id = ids[k];
  const double h = hb[id], invh = 1.0 / h;
  const int2 b = ij[id];
  const double o0 = (double)(b.x * CUP2D_BS) * h, o1 = (double)(b.y * CUP2D_BS) * h;
  const double org0 = o0 + h * 0.5, org1 = o1 + h * 0.5, en0 = o0 + h * (CUP2D_BS - 0.5), en1 = o1 + h * (CUP2D_BS - 0.5);
  const double pc0 = o0 + h * (ix + 0.5), pc1 = o1 + h * (iy + 0.5);
  const double *rX = S.mid, *rY = rX + nm, *norX = rY + nm, *norY = norX + nm, *vX = norY + nm, *vY = vX + nm;
  const double *vNorX = vY + nm, *vNorY = vNorX + nm, *width = vNorY + nm;
  double D = -1, X = 0, U0 = 0, U1 = 0; // this cell's o->dist, o->chi, o->udef
  // pass 1 (4303-4396): the two skin points of every midline point
  for (int q = 0; q < S.nseg; q++) {
    const double *sg = S.seg + (size_t)q * OG_SEG;
    if (!og_hit(sg, org0, org1, en0, en1)) continue;
    const int first = max((int)sg[13], 1), last = min((int)sg[14], nm - 2);
    for (int ss = first; ss <= last; ss++)
      for (int signp = -1; signp <= 1; signp += 2) {
        const double sp = (double)signp;
        double m0 = rX[ss] + width[ss] * sp * norX[ss], m1 = rY[ss] + width[ss] * sp * norY[ss];
        og_to_comp(S, m0, m1);
        const int ia0 = (int)floor((m0 - org0) * invh), ia1 = (int)floor((m1 - org1) * invh);
        if (ia0 + 3 <= 0 || ia0 - 1 >= CUP2D_BS || ia1 + 3 <= 0 || ia1 - 1 >= CUP2D_BS) continue;
        if (ix < ia0 - 2 || ix >= ia0 + 4 || iy < ia1 - 2 || iy >= ia1 + 4) continue;
        double P0 = rX[ss + 1] + width[ss + 1] * sp * norX[ss + 1], P1 = rY[ss + 1] + width[ss + 1] * sp * norY[ss + 1];
        og_to_comp(S, P0, P1);
        double M0 = rX[ss - 1] + width[ss - 1] * sp * norX[ss - 1], M1 = rY[ss - 1] + width[ss - 1] * sp * norY[ss - 1];
        og_to_comp(S, M0, M1);
        double u0 = vX[ss] + width[ss] * sp * vNorX[ss], u1 = vY[ss] + width[ss] * sp * vNorY[ss];
        og_vel_to_comp(S, u0, u1);
        const double dist0 = og_sq(pc0 - m0) + og_sq(pc1 - m1);
        const double distP = og_sq(pc0 - P0) + og_sq(pc1 - P1);
        const double distM = og_sq(pc0 - M0) + og_sq(pc1 - M1);
        if (fabs(D) < og_min(og_min(dist0, distP), distM)) continue;
        const double q0 = pc0 - S.px, q1 = pc1 - S.py; // changeFromComputationalFrame
        const double p0 = S.R00 * q0 + S.R10 * q1, p1 = S.R01 * q0 + S.R11 * q1;
        int close_s = ss, secnd_s = ss + (distP < distM ? 1 : -1);
        double dist1 = dist0;
        if (distP < dist0 || distM < dist0) {
          dist1 = distP < distM ? distP : distM;
          close_s = secnd_s;
          secnd_s = ss;
        }
        const double dSsq = og_sq(rX[close_s] - rX[secnd_s]) + og_sq(rY[close_s] - rY[secnd_s]);
        const double cnt2ML = og_sq(width[close_s]), nxt2ML = og_sq(width[secnd_s]);
        const double safeW = og_max(width[close_s], width[secnd_s]) + 2 * h;
        const double grd2ML = og_sq(p0 - rX[close_s]) + og_sq(p1 - rY[close_s]);
        const double diffH = fabs(width[close_s] - width[secnd_s]);
        double sign2d;
        if (dSsq > diffH * diffH || grd2ML > safeW * safeW) {
          sign2d = grd2ML > cnt2ML ? -1 : 1;
        } else {
          const double corr = 2 * sqrt(cnt2ML * nxt2ML);
          const double Rsq = (cnt2ML + nxt2ML - corr + dSsq) * (cnt2ML + nxt2ML + corr + dSsq) / 4 / dSsq;
          const double maxAx = og_max(cnt2ML, nxt2ML);
          const int idAx1 = cnt2ML > nxt2ML ? close_s : secnd_s, idAx2 = idAx1 == close_s ? secnd_s : close_s;
          const double d = sqrt((Rsq - maxAx) / dSsq);
          const double xc0 = rX[idAx1] + (rX[idAx1] - rX[idAx2]) * d, xc1 = rY[idAx1] + (rY[idAx1] - rY[idAx2]) * d;
          sign2d = og_sq(p0 - xc0) + og_sq(p1 - xc1) > Rsq ? -1 : 1;
        }
        if (fabs(D) > dist1) {
          const double W = 1 - og_min(1.0, sqrt(dist1) * (invh / 3));
          U0 = W * u0;
          U1 = W * u1;
          D = sign2d * dist1;
          X = W;
        }
      }
  }
  // pass 2 (4399-4447): points across the width, bilinear weights
  for (int q = 0; q < S.nseg; q++) {
    const double *sg = S.seg + (size_t)q * OG_SEG;
    if (!og_hit(sg, org0, org1, en0, en1)) continue;
    const int first = max((int)sg[13], 1), last = min((int)sg[14], nm - 2);
    for (int ss = first; ss <= last; ss++) {
      const int Nw = (int)floor(width[ss] / h);
      for (int iw = -Nw + 1; iw < Nw; ++iw) {
        const double offsetW = iw * h;
        double x0 = rX[ss] + offsetW * norX[ss], x1 = rY[ss] + offsetW * norY[ss];
        og_to_comp(S, x0, x1);
        x0 = (x0 - org0) * invh;
        x1 = (x1 - org1) * invh;
        const double ap0 = floor(x0), ap1 = floor(x1);
        const int ia0 = (int)ap0, ia1 = (int)ap1;
        if (ia0 + 2 <= 0 || ia0 >= CUP2D_BS || ia1 + 2 <= 0 || ia1 >= CUP2D_BS) continue;
        const int sx = ix - ia0, sy = iy - ia1;
        if (sx < 0 || sx > 1 || sy < 0 || sy > 1) continue;
        double u0 = vX[ss] + offsetW * vNorX[ss], u1 = vY[ss] + offsetW * vNorY[ss];
        og_vel_to_comp(S, u0, u1);
        const double wx = sx == 0 ? 1 - fabs(x0 - ap0) : 1 - fabs(x0 - (ap0 + 1));
        const double wy = sy == 0 ? 1 - fabs(x1 - ap1) : 1 - fabs(x1 - (ap1 + 1));
        const double wxwy = wy * wx;
        U0 += wxwy * u0;
        U1 += wxwy * u1;
        X += wxwy;
        if (fabs(D + 1) < DBL_EPSILON) D = 1;
      }
    }
  }
  const double normfac = X > DBL_EPSILON ? X : 1;
  U0 /= normfac;
  U1 /= normfac;
  D = D >= 0 ? sqrt(D) : -sqrt(-D);
  double *tp = tmp + (size_t)id * 64 + t;
  *tp = og_max(*tp, D);
  odist[(size_t)k * 64 + t] = D;
  ochi[(size_t)k * 64 + t] = 0;
  reinterpret_cast<double2 *>(oudef)[(size_t)k * 64 + t] = make_double2(U0, U1);
}

// PutChiOnGrid (main.cpp:3914-3968) for the obstacle blocks of one shape: part[k][3] = {Mass, COM_x, COM_y} of block k
__global__ void __launch_bounds__(64)
amr_ongrid_chi_kernel(const OgShape S, const int *__restrict__ ids, const int2 *__restrict__ ij, const double *__restrict__ hb,
                      const double *__restrict__ tmp, double *__restrict__ chi, const double *__restrict__ odist,
                      double *__restrict__ ochi, const int4 *__restrict__ nbr4, const int *__restrict__ irr_of, const GhostDev gt,
                      double *__restrict__ part) {
  __shared__ double lab[100];
  __shared__ double s_m[64];
  __shared__ double s_x[64];
  __shared__ double s_y[64];
  const int k = blockIdx.x, t = threadIdx.x, ix = t & 7, iy = t >> 3;
  const int id = ids[k];
  lab[(iy + 1) * 10 + ix + 1] = tmp[(size_t)id * 64 + t];
  if (t < 32) { // one ghost layer per face: same-level neighbour -> copy, wall -> the wall-adjacent cell (main.cpp:3239-3244)
    const int4 nbk = nbr4[id];
    const int f = t >> 3, p = t & 7;
    const int nbf = f == 0 ? nbk.x : f == 1 ? nbk.y : f == 2 ? nbk.z : nbk.w;
    if (nbf >= -1) {
      int gx, gy, sx, sy;
      if (f < 2) gx = f == 0 ? -1 : 8, gy = p, sx = nbf >= 0 ? (f == 0 ? 7 : 0) : (f == 0 ? 0 : 7), sy = p;
      else gx = p, gy = f == 2 ? -1 : 8, sx = p, sy = nbf >= 0 ? (f == 2 ? 7 : 0) : (f == 2 ? 0 : 7);
      lab[(gy + 1) * 10 + gx + 1] = tmp[(size_t)(nbf >= 0 ? nbf : id) * 64 + sy * 8 + sx];
    }
  }
  __syncthreads();
  const int qi = irr_of[id];
  if (qi >= 0) // coarser / finer neighbours: the ghost rows of the plan (kind 2)
    for (int64_t row = gt.grow[qi] + t; row < gt.grow[qi + 1]; row += 64) {
      double acc = 0.0;
      for (int64_t e = gt.rowptr[row]; e < gt.rowptr[row + 1]; e++) acc += gt.w[e] * tmp[(size_t)gt.sb[e] * 64 + gt.sc[e]];
      lab[gt.dst[row] % 100] = acc;
    }
  __syncthreads();
  const double h = hb[id], h2 = h * h;
  const double dist = odist[(size_t)k * 64 + t];
  double c;
  if (dist > +h || dist < -h) {
    c = dist > 0 ? 1 : 0;
  } else {
    const int x0 = ix + 1, y0 = iy + 1;
    const double distPx = lab[10 * y0 + x0 + 1], distMx = lab[10 * y0 + x0 - 1];
    const double distPy = lab[10 * (y0 + 1) + x0], distMy = lab[10 * (y0 - 1) + x0];
    const double IplusX = og_max(0.0, distPx), IminuX = og_max(0.0, distMx);
    const double IplusY = og_max(0.0, distPy), IminuY = og_max(0.0, distMy);
    const double gradIX = IplusX - IminuX, gradIY = IplusY - IminuY;
    const double gradUX = distPx - distMx, gradUY = distPy - distMy;
    const double gradUSq = (gradUX * gradUX + gradUY * gradUY) + DBL_EPSILON;
    c = (gradIX * gradUX + gradIY * gradUY) / gradUSq;
  }
  ochi[(size_t)k * 64 + t] = c;
  double *cp = chi + (size_t)id * 64 + t;
  *cp = og_max(*cp, c);
  s_m[t] = s_x[t] = s_y[t] = 0;
  if (c > 0) {
    const int2 b = ij[id];
    const double p0 = (double)(b.x * CUP2D_BS) * h + h * (ix + 0.5), p1 = (double)(b.y * CUP2D_BS) * h + h * (iy + 0.5);
    s_x[t] = c * h2 * (p0 - S.cmx);
    s_y[t] = c * h2 * (p1 - S.cmy);
    s_m[t] = c * h2;
  }
  __syncthreads();
  if (t == 0) { // the reference's per-block sums, cell by cell
    double m = 0, x = 0, y = 0;
    for (int j = 0; j < 64; j++) {
      x += s_x[j];
      y += s_y[j];
      m += s_m[j];
    }
    part[(size_t)k * 3] = m;
    part[(size_t)k * 3 + 1] = x;
    part[(size_t)k * 3 + 2] = y;
  }
}

// the seven sums of main.cpp:4492-4518 per obstacle block (cell order), about the corrected centre of mass
__global__ void __launch_bounds__(64)
amr_ongrid_moments_kernel(const OgShape S, const int *__restrict__ ids, const int2 *__restrict__ ij, const double *__restrict__ hb,
                          const double *__restrict__ ochi, const double *__restrict__ oudef, double *__restrict__ part) {
  __shared__ double s[7 * 64];
  const int k = blockIdx.x, t = threadIdx.x, ix = t & 7, iy = t >> 3;
  const int id = ids[k];
  const double h = hb[id], hsq = h * h;
  const double X = ochi[(size_t)k * 64 + t];
  for (int q = 0; q < 7; q++) s[q * 64 + t] = 0;
  if (X > 0) {
    const int2 b = ij[id];
    double p0 = (double)(b.x * CUP2D_BS) * h + h * (ix + 0.5), p1 = (double)(b.y * CUP2D_BS) * h + h * (iy + 0.5);
    const double chi = X * hsq;
    p0 -= S.cmx;
    p1 -= S.cmy;
    const double2 U = reinterpret_cast<const double2 *>(oudef)[(size_t)k * 64 + t];
    s[0 * 64 + t] = chi * p0;
    s[1 * 64 + t] = chi * p1;
    s[2 * 64 + t] = chi;
    s[3 * 64 + t] = chi * (p0 * p0 + p1 * p1);
    s[4 * 64 + t] = chi * U.x;
    s[5 * 64 + t] = chi * U.y;
    s[6 * 64 + t] = chi * (p0 * U.y - p1 * U.x);
  }
  __syncthreads();
  if (t < 7) {
    double acc = 0;
    for (int j = 0; j < 64; j++) acc += s[t * 64 + j];
    part[(size_t)k * 7 + t] = acc;
  }
}

// main.cpp:4541-4556 on every cell of the obstacle blocks
__global__ void __launch_bounds__(64)
amr_ongrid_correct_kernel(const OgShape S, const int *__restrict__ ids, const int2 *__restrict__ ij, const double *__restrict__ hb,
                          double *__restrict__ oudef, double u, double v, double a) {
  const int k = blockIdx.x, t = threadIdx.x, ix = t & 7, iy = t >> 3;
  const int id = ids[k];
  const double h = hb[id];
  const int2 b = ij[id];
  double p0 = (double)(b.x * CUP2D_BS) * h + h * (ix + 0.5), p1 = (double)(b.y * CUP2D_BS) * h + h * (iy + 0.5);
  p0 -= S.cmx;
  p1 -= S.cmy;
  double2 *up = reinterpret_cast<double2 *>(oudef) + (size_t)k * 64 + t;
  double2 U = *up;
  U.x -= u - a * p1;
  U.y -= v + a * p0;
  *up = U;
}

// AreaSegment (main.cpp:3839-3878) of points idx..next_idx of a midline, in the lab frame: the record of OG_SEG doubles
static void og_segment(const cup2d_body &B, int idx, int next_idx, double safe, double cosang, double sinang, double *r) {
  double bb[2][2] = {{1e9, -1e9}, {1e9, -1e9}};
  for (int ss = idx; ss <= next_idx; ++ss) { // main.cpp:4221-4236
    const double xBnd[2] = {B.rX[ss] - B.norX[ss] * B.width[ss], B.rX[ss] + B.norX[ss] * B.width[ss]};
    const double yBnd[2] = {B.rY[ss] - B.norY[ss] * B.width[ss], B.rY[ss] + B.norY[ss] * B.width[ss]};
    const double maxX = std::max(xBnd[0], xBnd[1]), minX = std::min(xBnd[0], xBnd[1]);
    const double maxY = std::max(yBnd[0], yBnd[1]), minY = std::min(yBnd[0], yBnd[1]);
    bb[0][0] = std::min(bb[0][0], minX);
    bb[0][1] = std::max(bb[0][1], maxX);
    bb[1][0] = std::min(bb[1][0], minY);
    bb[1][1] = std::max(bb[1][1], maxY);
  }
  const double w[2] = {(bb[0][1] - bb[0][0]) / 2 + safe, (bb[1][1] - bb[1][0]) / 2 + safe};
  double c[2] = {(bb[0][1] + bb[0][0]) / 2, (bb[1][1] + bb[1][0]) / 2};
  const double R[2][2] = {{cosang, -sinang}, {sinang, cosang}};
  const double p[2] = {c[0], c[1]}, nx[2] = {1, 0}, ny[2] = {0, 1};
  double nI[2], nJ[2];
  for (int i = 0; i < 2; ++i) {
    c[i] = R[i][0] * p[0] + R[i][1] * p[1];
    nI[i] = R[i][0] * nx[0] + R[i][1] * nx[1];
    nJ[i] = R[i][0] * ny[0] + R[i][1] * ny[1];
  }
  c[0] += B.center[0];
  c[1] += B.center[1];
  const double magI = std::sqrt(nI[0] * nI[0] + nI[1] * nI[1]), magJ = std::sqrt(nJ[0] * nJ[0] + nJ[1] * nJ[1]);
  const double invMagI = 1 / magI, invMagJ = 1 / magJ;
  for (int i = 0; i < 2; ++i) {
    nI[i] = std::fabs(nI[i]) * invMagI;
    nJ[i] = std::fabs(nJ[i]) * invMagJ;
  }
  r[0] = safe;
  r[1] = nI[0], r[2] = nI[1], r[3] = nJ[0], r[4] = nJ[1];
  for (int i = 0; i < 2; ++i) {
    const double wx = w[0] * nI[i], wy = w[1] * nJ[i];
    r[5 + 2 * i] = c[i] - wx - wy;
    r[6 + 2 * i] = c[i] + wx + wy;
    r[9 + 2 * i] = c[i] - w[i];
    r[10 + 2 * i] = c[i] + w[i];
  }
  r[13] = idx, r[14] = next_idx, r[15] = 0;
}

// the blend of the initial velocity with the bodies' u_def before the time loop (main.cpp:6566-6575): one CTA of 256 threads
// handles 2 blocks (128 cells x (u, v)) per pass, block-strided; explicit round-to-nearest in the reference's expression order
__global__ void __launch_bounds__(256)
amr_udef_blend_kernel(double *__restrict__ vel, const double *__restrict__ tmpv, const double *__restrict__ chi, int64_t nb) {
  const int64_t n = nb * 128;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) {
    const double x = chi[i >> 1];
    vel[i] = __dadd_rn(__dmul_rn(vel[i], __dsub_rn(1.0, x)), __dmul_rn(tmpv[i], x));
  }
}

// per-call device scratch, grown as needed (freed with the shapes)
static int og_grow(void **p, size_t *cap, size_t bytes) {
  if (bytes <= *cap) return CUP2D_OK;
  cudaFree(*p);
  *p = nullptr, *cap = 0;
  CUP2D_CUDA(cudaMalloc(p, bytes));
  *cap = bytes;
  return CUP2D_OK;
}

} // namespace cup2d

using namespace cup2d;

extern "C" {

int cup2d_amr_ongrid(cup2d_amr *a, int nshapes, const cup2d_body *bodies, double *out) {
  if (!a || nshapes < 1 || nshapes > OG_MAXSH || !bodies || !out) {
    set_error("cup2d_amr_ongrid: bad arguments (1..64 bodies and an output array)");
    return CUP2D_EINVAL;
  }
  if (!a->dist && a->nranks > 1) {
    set_error("cup2d_amr_ongrid: contexts with operators replicated on several ranks (cup2d_amr_set_ranks) are not supported");
    return CUP2D_ESTATE;
  }
  int bpdx = 0, bpdy = 0;
  amr_plan_level_ij(a->plan, &bpdx, &bpdy);
  const double ext[2] = {bpdx * CUP2D_BS * a->h0, bpdy * CUP2D_BS * a->h0};
  for (int s = 0; s < nshapes; s++) {
    const cup2d_body &B = bodies[s];
    if (B.nm < 9 || (B.nm - 1) % ((B.nm - 1) / 8) != 0 || !B.rX || !B.rY || !B.norX || !B.norY || !B.vX || !B.vY || !B.vNorX || !B.vNorY || !B.width) {
      set_error("cup2d_amr_ongrid: body " + std::to_string(s) + " needs nm >= 9 with (nm - 1) divisible by (nm - 1) / 8 (main.cpp:4208-4210) and nine midline arrays");
      return CUP2D_EINVAL;
    }
    if (!(B.center[0] >= 0 && B.center[0] <= ext[0] && B.center[1] >= 0 && B.center[1] <= ext[1])) { // main.cpp:4009-4013
      set_error("cup2d_amr_ongrid: body " + std::to_string(s) + " has its center outside the domain");
      return CUP2D_EINVAL;
    }
  }
  // host part, O(Nm): rotation from the host libm, segments, one staged upload
  std::vector<double> stage;
  std::vector<size_t> mid_off(nshapes), seg_off(nshapes);
  std::vector<int> nseg(nshapes);
  std::vector<double> cosang(nshapes), sinang(nshapes);
  const double safe = 4 * a->hmin; // main.cpp:4212-4215, 4237
  for (int s = 0; s < nshapes; s++) {
    const cup2d_body &B = bodies[s];
    const int nm = B.nm;
    cosang[s] = std::cos(B.orientation);
    sinang[s] = std::sin(B.orientation);
    mid_off[s] = stage.size();
    for (const double *p : {B.rX, B.rY, B.norX, B.norY, B.vX, B.vY, B.vNorX, B.vNorY, B.width}) stage.insert(stage.end(), p, p + nm);
    nseg[s] = (nm - 1) / 8; // main.cpp:4208
    seg_off[s] = stage.size();
    stage.resize(stage.size() + (size_t)nseg[s] * OG_SEG);
    for (int i = 0; i < nseg[s]; ++i)
      og_segment(B, i * (nm - 1) / nseg[s], (i + 1) * (nm - 1) / nseg[s], safe, cosang[s], sinang[s],
                 stage.data() + seg_off[s] + (size_t)i * OG_SEG);
  }
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc = amr_fast_tables(a);
  if (rc || (rc = amr_ensure_ij(a))) return rc;
  const int64_t nb = a->nb;
  const int ncta = (int)((nb + OG_SCAN - 1) / OG_SCAN);
  if ((rc = og_grow((void **)&a->d_og_stage, &a->og_stage_cap, stage.size() * sizeof(double))) ||
      (rc = og_grow((void **)&a->d_og_mask, &a->og_mask_cap, (size_t)nb * sizeof(unsigned long long))) ||
      (rc = og_grow((void **)&a->d_og_cnt, &a->og_cnt_cap, ((size_t)nshapes * ncta + OG_MAXSH) * sizeof(int))))
    return rc;
  // CUDA events around the kernels (cup2d_amr_ongrid_timing); ev(i) is a no-op unless timing is on
  auto ev = [&](int i) { return a->og_timing ? cudaEventRecord((cudaEvent_t)a->og_ev[i], a->stream) : cudaSuccess; };
  CUP2D_CUDA(ev(0));
  CUP2D_CUDA(cudaMemcpyAsync(a->d_og_stage, stage.data(), stage.size() * sizeof(double), cudaMemcpyHostToDevice, a->stream));
  OgSegs segs = {};
  segs.nshapes = nshapes;
  for (int s = 0; s < nshapes; s++) segs.seg[s] = a->d_og_stage + seg_off[s], segs.nseg[s] = nseg[s];
  const int2 *ij = reinterpret_cast<const int2 *>(a->d_ij);
  int *d_total = a->d_og_cnt + (size_t)nshapes * ncta;
  CUP2D_CUDA(ev(1));
  amr_ongrid_scan_kernel<<<ncta, OG_SCAN, 0, a->stream>>>(a->f[CUP2D_CHI], a->f[CUP2D_TMP], ij, a->d_h, (int)nb, segs, a->d_og_mask,
                                                          a->d_og_cnt);
  CUP2D_CUDA(ev(2));
  amr_ongrid_offsets_kernel<<<nshapes, OG_OFF_NT, 0, a->stream>>>(a->d_og_cnt, ncta, d_total);
  CUP2D_CUDA(ev(3));
  CUP2D_CUDA(cudaGetLastError());
  std::vector<int> nob(nshapes);
  CUP2D_CUDA(cudaMemcpyAsync(nob.data(), d_total, nshapes * sizeof(int), cudaMemcpyDeviceToHost, a->stream));
  CUP2D_CUDA(cudaStreamSynchronize(a->stream));
  // per-shape storage (as cup2d_amr_shape_set), plus dist; shapes beyond nshapes are dropped
  for (size_t s = nshapes; s < a->shapes.size(); s++) {
    cup2d_amr::Shape &sh = a->shapes[s];
    cudaFree(sh.d_ids); cudaFree(sh.d_X); cudaFree(sh.d_udef); cudaFree(sh.d_dist);
  }
  a->shapes.resize(nshapes);
  OgIds oids = {};
  std::vector<int64_t> pofs(nshapes + 1, 0); // first partial-sum slot of every shape
  for (int s = 0; s < nshapes; s++) {
    cup2d_amr::Shape &sh = a->shapes[s];
    if (nob[s] > sh.cap || !sh.d_dist) {
      cudaFree(sh.d_ids); cudaFree(sh.d_X); cudaFree(sh.d_udef); cudaFree(sh.d_dist);
      sh.d_ids = nullptr, sh.d_X = sh.d_udef = sh.d_dist = nullptr, sh.cap = 0;
      const int cap = nob[s] + nob[s] / 4 + 16;
      CUP2D_CUDA(cudaMalloc(&sh.d_ids, (size_t)cap * sizeof(int)));
      CUP2D_CUDA(cudaMalloc(&sh.d_X, (size_t)cap * 64 * sizeof(double)));
      CUP2D_CUDA(cudaMalloc(&sh.d_udef, (size_t)cap * 128 * sizeof(double)));
      CUP2D_CUDA(cudaMalloc(&sh.d_dist, (size_t)cap * 64 * sizeof(double)));
      sh.cap = cap;
    }
    sh.nob = nob[s];
    sh.has_dist = sh.ascending = true;
    sh.has_surface = false;
    oids.ids[s] = sh.d_ids;
    pofs[s + 1] = pofs[s] + nob[s];
  }
  const int64_t ntot = pofs[nshapes];
  if ((rc = og_grow((void **)&a->d_og_part, &a->og_part_cap, (size_t)std::max<int64_t>(ntot, 1) * 7 * sizeof(double)))) return rc;
  CUP2D_CUDA(ev(4));
  amr_ongrid_compact_kernel<<<ncta, OG_SCAN, 0, a->stream>>>(a->d_og_mask, a->d_og_cnt, (int)nb, nshapes, oids);
  CUP2D_CUDA(ev(5));
  std::vector<OgShape> S(nshapes);
  for (int s = 0; s < nshapes; s++) {
    const cup2d_body &B = bodies[s];
    S[s] = OgShape{a->d_og_stage + mid_off[s], a->d_og_stage + seg_off[s], B.nm, nseg[s], cosang[s], -sinang[s], sinang[s],
                   cosang[s], B.center[0], B.center[1], B.center_of_mass[0], B.center_of_mass[1]};
  }
  for (int s = 0; s < nshapes; s++) { // shapes in order: tmp is the maximum over all of them before PutChiOnGrid
    const cup2d_amr::Shape &sh = a->shapes[s];
    if (sh.nob)
      amr_ongrid_fish_kernel<<<sh.nob, 64, 0, a->stream>>>(S[s], sh.d_ids, ij, a->d_h, a->f[CUP2D_TMP], sh.d_dist, sh.d_X, sh.d_udef);
  }
  CUP2D_CUDA(ev(6));
  if ((rc = amr_dist_refresh(a, CUP2D_TMP))) return rc; // the +-1 lab of tmp reads the halo slots of a distributed context
  for (int s = 0; s < nshapes; s++) { // Mass / COM partials of every shape, one download
    const cup2d_amr::Shape &sh = a->shapes[s];
    if (sh.nob)
      amr_ongrid_chi_kernel<<<sh.nob, 64, 0, a->stream>>>(S[s], sh.d_ids, ij, a->d_h, a->f[CUP2D_TMP], a->f[CUP2D_CHI], sh.d_dist, sh.d_X,
                                                          reinterpret_cast<const int4 *>(a->d_nbr4), a->d_irr_of, a->gt[2],
                                                          a->d_og_part + 3 * pofs[s]);
  }
  CUP2D_CUDA(ev(7));
  CUP2D_CUDA(cudaGetLastError());
  std::vector<double> hp((size_t)std::max<int64_t>(ntot, 1) * 7);
  CUP2D_CUDA(cudaMemcpyAsync(hp.data(), a->d_og_part, (size_t)ntot * 3 * sizeof(double), cudaMemcpyDeviceToHost, a->stream));
  CUP2D_CUDA(cudaStreamSynchronize(a->stream));
  std::vector<double> sums((size_t)nshapes * 7, 0.0);
  for (int s = 0; s < nshapes; s++) // block order (main.cpp:4476-4482)
    for (int64_t k = pofs[s]; k < pofs[s + 1]; k++)
      for (int q = 0; q < 3; q++) sums[(size_t)s * 3 + q] += hp[(size_t)k * 3 + q];
  if ((rc = amr_dist_sum_vec(a, sums.data(), 3 * nshapes))) return rc; // the ranks' partials, as MPI_Allreduce (4483)
  for (int s = 0; s < nshapes; s++) {
    const double *com = sums.data() + (size_t)s * 3;
    double *o = out + 10 * s;
    o[0] = com[0], o[1] = com[1], o[2] = com[2];
    o[3] = bodies[s].center_of_mass[0] + com[1] / com[0]; // main.cpp:4485-4486
    o[4] = bodies[s].center_of_mass[1] + com[2] / com[0];
    S[s].cmx = o[3], S[s].cmy = o[4];
  }
  CUP2D_CUDA(ev(8));
  for (int s = 0; s < nshapes; s++) { // the seven sums of every shape, one download
    const cup2d_amr::Shape &sh = a->shapes[s];
    if (sh.nob)
      amr_ongrid_moments_kernel<<<sh.nob, 64, 0, a->stream>>>(S[s], sh.d_ids, ij, a->d_h, sh.d_X, sh.d_udef, a->d_og_part + 7 * pofs[s]);
  }
  CUP2D_CUDA(ev(9));
  CUP2D_CUDA(cudaGetLastError());
  CUP2D_CUDA(cudaMemcpyAsync(hp.data(), a->d_og_part, (size_t)ntot * 7 * sizeof(double), cudaMemcpyDeviceToHost, a->stream));
  CUP2D_CUDA(cudaStreamSynchronize(a->stream));
  CUP2D_CUDA(ev(10));
  std::fill(sums.begin(), sums.end(), 0.0);
  for (int s = 0; s < nshapes; s++)
    for (int64_t k = pofs[s]; k < pofs[s + 1]; k++)
      for (int q = 0; q < 7; q++) sums[(size_t)s * 7 + q] += hp[(size_t)k * 7 + q];
  if ((rc = amr_dist_sum_vec(a, sums.data(), 7 * nshapes))) return rc; // as MPI_Allreduce (4520)
  for (int s = 0; s < nshapes; s++) {
    const cup2d_amr::Shape &sh = a->shapes[s];
    const double *q7 = sums.data() + (size_t)s * 7;
    const double m = q7[2], j = q7[3], u = q7[4] / m, v = q7[5] / m, av = q7[6] / j; // main.cpp:4529-4531
    double *o = out + 10 * s;
    o[5] = m, o[6] = j, o[7] = u, o[8] = v, o[9] = av;
    if (sh.nob) amr_ongrid_correct_kernel<<<sh.nob, 64, 0, a->stream>>>(S[s], sh.d_ids, ij, a->d_h, sh.d_udef, u, v, av);
  }
  CUP2D_CUDA(ev(11));
  CUP2D_CUDA(cudaGetLastError());
  CUP2D_CUDA(cudaStreamSynchronize(a->stream));
  a->og_timed = a->og_timing;
  return CUP2D_OK;
}

int cup2d_amr_ongrid_timing(cup2d_amr *a, int on) {
  if (!a) {
    set_error("null cup2d_amr handle");
    return CUP2D_EINVAL;
  }
  CUP2D_CUDA(cudaSetDevice(a->device));
  if (on && !a->og_release) {
    a->og_release = [](cup2d_amr *c) {
      for (auto &e : c->og_ev)
        if (e) cudaEventDestroy((cudaEvent_t)e), e = nullptr;
    };
    for (auto &e : a->og_ev) {
      cudaEvent_t ce = nullptr;
      CUP2D_CUDA(cudaEventCreate(&ce));
      e = (void *)ce;
    }
  }
  a->og_timing = on != 0;
  a->og_timed = false;
  return CUP2D_OK;
}

int cup2d_amr_ongrid_times(cup2d_amr *a, double *ms8) {
  if (!a || !ms8 || !a->og_timed) {
    set_error("cup2d_amr_ongrid_times: no timed cup2d_amr_ongrid call (cup2d_amr_ongrid_timing(a, 1) first)");
    return CUP2D_EINVAL;
  }
  // call, scan, offsets, compact, fish, chi, moments, correct
  const int from[8] = {0, 1, 2, 4, 5, 6, 8, 10}, to[8] = {11, 2, 3, 5, 6, 7, 9, 11};
  for (int q = 0; q < 8; q++) {
    float ms = 0.f;
    CUP2D_CUDA(cudaEventElapsedTime(&ms, (cudaEvent_t)a->og_ev[from[q]], (cudaEvent_t)a->og_ev[to[q]]));
    ms8[q] = ms;
  }
  return CUP2D_OK;
}

int cup2d_amr_shape_get(cup2d_amr *a, int shape, int32_t *ids, double *chi, double *dist, double *udef) {
  if (!a || shape < 0 || shape >= (int)a->shapes.size()) {
    set_error("cup2d_amr_shape_get: no such shape");
    return CUP2D_EINVAL;
  }
  const cup2d_amr::Shape &sh = a->shapes[shape];
  if (dist && !sh.has_dist) {
    set_error("cup2d_amr_shape_get: the shape was set by cup2d_amr_shape_set and has no dist");
    return CUP2D_EINVAL;
  }
  CUP2D_CUDA(cudaSetDevice(a->device));
  if (sh.nob) {
    if (ids) CUP2D_CUDA(cudaMemcpyAsync(ids, sh.d_ids, (size_t)sh.nob * sizeof(int), cudaMemcpyDeviceToHost, a->stream));
    if (chi) CUP2D_CUDA(cudaMemcpyAsync(chi, sh.d_X, (size_t)sh.nob * 64 * sizeof(double), cudaMemcpyDeviceToHost, a->stream));
    if (dist) CUP2D_CUDA(cudaMemcpyAsync(dist, sh.d_dist, (size_t)sh.nob * 64 * sizeof(double), cudaMemcpyDeviceToHost, a->stream));
    if (udef) CUP2D_CUDA(cudaMemcpyAsync(udef, sh.d_udef, (size_t)sh.nob * 128 * sizeof(double), cudaMemcpyDeviceToHost, a->stream));
    CUP2D_CUDA(cudaStreamSynchronize(a->stream));
  }
  return sh.nob;
}

int cup2d_amr_udef_blend(cup2d_amr *a) {
  if (!a) {
    set_error("null cup2d_amr handle");
    return CUP2D_EINVAL;
  }
  CUP2D_CUDA(cudaSetDevice(a->device));
  if (a->nb == 0) return CUP2D_OK;
  const int grid = (int)std::min<int64_t>((a->nb + 1) / 2, AMR_GRID_SMS * 8);
  amr_udef_blend_kernel<<<grid, 256, 0, a->stream>>>(a->f[CUP2D_VEL], a->f[CUP2D_TMPV], a->f[CUP2D_CHI], a->nb);
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

} // extern "C"
