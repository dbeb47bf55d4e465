// Poisson right-hand side of one warp's rows, shared by the stand-alone right-hand-side kernel (pressure.cu) and the kernel
// that starts a step's solve from it (poisson.cu), so that both form b with the same expression in the same order.
#pragma once
#include "rows.cuh"

namespace cup2d {

// ------------------------------------------------------------------------------------------------
// undivided divergence of a vector field on the warp's 32 rows, free-slip ghosts at walls
// (pressure_rhs main.cpp:6105-6139: ((u_E - u_W) + v_N) - v_S, left to right; VectorLab ghosts
// main.cpp:3131-3154: normal component negated)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void rows_div(const double2 (&cf)[8], const double *__restrict__ f, int nvalid,
                                         const int4 nb, int slot, int y, double *sw, int lane,
                                         double (&d)[8]) {
  double2 c[8];
  chunk2_to_rows(sw, nvalid, lane, cf, c);
  if (lane < nvalid) {
    const double2 *f2 = reinterpret_cast<const double2 *>(f);
    double vu[8], vd[8];
    {
      double2 t[8];
      if (y < 7) {
        rows_peek2(sw, lane + 1, t);
#pragma unroll
        for (int i = 0; i < 8; i++) vu[i] = t[i].y;
      } else if (nb.w >= 0) {
        grow_load2(f, nb.w, 0, t);
#pragma unroll
        for (int i = 0; i < 8; i++) vu[i] = t[i].y;
      } else {
#pragma unroll
        for (int i = 0; i < 8; i++) vu[i] = -c[i].y;
      }
      if (y > 0) {
        rows_peek2(sw, lane - 1, t);
#pragma unroll
        for (int i = 0; i < 8; i++) vd[i] = t[i].y;
      } else if (nb.z >= 0) {
        grow_load2(f, nb.z, 7, t);
#pragma unroll
        for (int i = 0; i < 8; i++) vd[i] = t[i].y;
      } else {
#pragma unroll
        for (int i = 0; i < 8; i++) vd[i] = -c[i].y;
      }
    }
    const double uW = nb.x >= 0 ? f2[(size_t)nb.x * 64 + y * 8 + 7].x : -c[0].x;
    const double uE = nb.y >= 0 ? f2[(size_t)nb.y * 64 + y * 8 + 0].x : -c[7].x;
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const double e = i < 7 ? c[i + 1].x : uE;
      const double w = i > 0 ? c[i - 1].x : uW;
      d[i] = ((e - w) + vu[i]) - vd[i];
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; i++) d[i] = 0.0;
  }
}

// out = fac*(div vel) - fac*chi*(div udef) - lap(pold) of rows [row0, row0 + nv) in row layout (lane l: row row0 + l, zero
// beyond nv)     (main.cpp:7011-7027).  sw: per-warp scratch of ROWS_SCRATCH doubles.  All 32 lanes must call.
template <bool HAS_UDEF>
__device__ __forceinline__ void rhs_rows(const double *__restrict__ vel, const double *__restrict__ udef,
                                         const double *__restrict__ chi, const double *__restrict__ pold,
                                         const int4 *__restrict__ nbr, int row0, int nv, double fac, double *sw, int lane,
                                         double (&out)[8]) {
  const int row = row0 + lane, slot = row >> 3, y = row & 7;
  const int4 nb = lane < nv ? nbr[slot] : make_int4(-1, -1, -1, -1);
  double t[8], pc[8];
  // every global load of the chunk is issued up front (memory-level parallelism), then the smem work
  double2 cvel[8], cpold[4];
  chunk2_ld(vel, row0, nv, lane, cvel);
  chunk_ld(pold, row0, nv, lane, cpold);
  rows_div(cvel, vel, nv, nb, slot, y, sw, lane, out);
#pragma unroll
  for (int i = 0; i < 8; i++) out[i] *= fac;
  if (HAS_UDEF) {
    double du[8];
    double2 cud[8];
    chunk2_ld(udef, row0, nv, lane, cud);
    rows_div(cud, udef, nv, nb, slot, y, sw, lane, du);
    rows_load1(chi, row0, nv, sw, lane, t);
#pragma unroll
    for (int i = 0; i < 8; i++) out[i] = out[i] - fac * t[i] * du[i];
  }
  rows_lap_c(cpold, pold, row0, nv, nbr, sw, lane, pc, t);
#pragma unroll
  for (int i = 0; i < 8; i++) out[i] -= t[i];
}

} // namespace cup2d
