// dt control, Poisson right-hand side and pressure correction kernels.
//
// Thread mapping for the block-structured kernels: one lane = one row of 8 cells of one 8x8 block,
// one warp = 4 consecutive blocks.  Global memory is touched only with warp-coalesced 128-bit
// accesses; rows (and the rows of the lanes above/below) come out of a padded per-warp shared-memory
// scratch (rows.cuh).  Neighbour BLOCKS come through d_nbr[slot] = (W,E,S,N), -1 = domain wall, which
// replaces the reference's BlockLab assembly (main.cpp:2270-2440) and ghost fill (main.cpp:3131-3154,
// 3210-3245).
#include "rhs.cuh"
#include "sim.h"

namespace cup2d {

constexpr int NT = 256;
constexpr int WPB = NT / 32;

// ------------------------------------------------------------------------------------------------
// umax = max |vel| over both components (main.cpp:6585-6591)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NT) umax_kernel(const double *__restrict__ vel, size_t n2,
                                                  double *partials, unsigned int *counter,
                                                  Comm comm, double *out) {
  double m = 0;
  const double2 *p = reinterpret_cast<const double2 *>(vel);
  for (size_t i = (size_t)blockIdx.x * NT + threadIdx.x; i < n2; i += (size_t)gridDim.x * NT) {
    const double2 a = p[i];
    m = fmax(m, fmax(fabs(a.x), fabs(a.y)));
  }
  double dummy[1] = {0};
  grid_reduce<1, NT>(dummy, m, partials, counter, comm, [=](const double *, double mx) { out[0] = mx; });
}

int launch_umax_async(cup2d_sim *s) {
  const size_t n2 = (size_t)s->nloc * 64;
  int grid = s->num_sms * 8;
  {
    ProfScope prof(s, KC_UMAX);
    umax_kernel<<<grid, NT, 0, s->stream>>>(s->f[CUP2D_VEL], n2, s->d_partials, s->d_counter, s->comm, s->d_scal);
  }
  s->launches++;
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

// dt rule (main.cpp:6593-6595) and everything derived from dt, on the device, in the host code's operation order
// (explicit round-to-nearest operations: no FMA contraction, so dt is bitwise what cup2d_compute_dt returns)
__global__ void k_step_factors(StepFactors *f, const double *umax_in, double dt_host, double h, double nu, double cfl) {
  double dt = dt_host, umax = 0.0;
  if (umax_in) {
    umax = *umax_in;
    const double dt_diff = __ddiv_rn(__dmul_rn(__dmul_rn(0.25, h), h), __dadd_rn(nu, __dmul_rn(__dmul_rn(0.25, h), umax)));
    const double dt_adv = __ddiv_rn(h, __dadd_rn(umax, 1e-8));
    dt = fmin(dt_diff, __dmul_rn(cfl, dt_adv));
  }
  f->dt = dt;
  f->umax = umax;
  f->afac = __dmul_rn(-dt, h);                                             // launch_advect: -dt * h
  f->dfac = __dmul_rn(nu, dt);                                             //                nu * dt
  f->rhs_fac = __ddiv_rn(__dmul_rn(0.5, h), dt);                           // launch_pressure_rhs: 0.5 * h / dt
  f->corr_fac = __dmul_rn(__dmul_rn(__dmul_rn(-0.5, dt), h), __ddiv_rn(__ddiv_rn(1.0, h), h)); // (-0.5 dt h) * (1/h/h)
}
int launch_step_factors(cup2d_sim *s, double dt_host) {
  k_step_factors<<<1, 1, 0, s->stream>>>(s->d_fac, dt_host > 0 ? nullptr : s->d_scal, dt_host, s->h, s->nu, s->cfl);
  s->launches++;
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

int launch_umax(cup2d_sim *s, double *umax_out) {
  int rc = launch_umax_async(s);
  if (rc) return rc;
  CUP2D_CUDA(cudaMemcpyAsync(s->h_scal, s->d_scal, sizeof(double), cudaMemcpyDeviceToHost, s->stream));
  CUP2D_CUDA(cudaStreamSynchronize(s->stream));
  *umax_out = s->h_scal[0];
  return CUP2D_OK;
}

// tmp = fac*(div vel) - fac*chi*(div udef) - lap(pold);  pres = 0     (main.cpp:7011-7027)
// The stand-alone form (cup2d_pressure_rhs): a time step forms the same b in pressure_rhs_start_kernel (poisson.cu) and
// starts its solve there instead.
template <bool HAS_UDEF>
__global__ void __launch_bounds__(NT)
pressure_rhs_kernel(const double *__restrict__ vel, const double *__restrict__ udef,
                    const double *__restrict__ chi, const double *__restrict__ pold,
                    double *__restrict__ tmp, double *__restrict__ pres, const int4 *__restrict__ nbr,
                    int nrows, double fac) {
  __shared__ __align__(16) double s_scr[WPB * ROWS_SCRATCH];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double *sw = s_scr + warp * ROWS_SCRATCH;
  for (int row0 = (blockIdx.x * WPB + warp) * 32; row0 < nrows; row0 += gridDim.x * WPB * 32) {
    const int nv = min(32, nrows - row0);
    double out[8];
    rhs_rows<HAS_UDEF>(vel, udef, chi, pold, nbr, row0, nv, fac, sw, lane, out);
    rows_store1(tmp, row0, nv, sw, lane, out);
#pragma unroll
    for (int i = 0; i < 8; i++) out[i] = 0.0;
    rows_store1(pres, row0, nv, sw, lane, out);
  }
}

int pressure_rhs_inputs(cup2d_sim *s, bool has_udef) {
  // pold <- pres is a pointer swap; the right-hand side then reads pold (main.cpp:7016-7021)
  swap_fields(s, CUP2D_PRES, CUP2D_POLD);
  if (s->nranks > 1) {
    int rc;
    if ((rc = halo_exchange_ptr(s, s->f[CUP2D_VEL], 2, CUP2D_VEL))) return rc;
    if (has_udef && (rc = halo_exchange_ptr(s, s->f[CUP2D_TMPV], 2, CUP2D_TMPV))) return rc;
    if ((rc = halo_exchange_ptr(s, s->f[CUP2D_POLD], 1, CUP2D_POLD))) return rc;
  }
  return CUP2D_OK;
}

int launch_pressure_rhs(cup2d_sim *s, double dt, bool has_udef) {
  int rc = pressure_rhs_inputs(s, has_udef);
  if (rc) return rc;
  const int nrows = (int)s->nloc * 8;
  const int grid = min((nrows + NT - 1) / NT, s->num_sms * 8);
  const double fac = 0.5 * s->h / dt; // main.cpp:6119
  ProfScope prof(s, KC_RHS);
  if (has_udef)
    pressure_rhs_kernel<true><<<grid, NT, 0, s->stream>>>(s->f[CUP2D_VEL], s->f[CUP2D_TMPV], s->f[CUP2D_CHI],
                                                          s->f[CUP2D_POLD], s->f[CUP2D_TMP], s->f[CUP2D_PRES],
                                                          reinterpret_cast<const int4 *>(s->d_nbr), nrows, fac);
  else // no bodies: chi * div(udef) is identically zero (main.cpp:6980-6983 leaves tmpV = 0)
    pressure_rhs_kernel<false><<<grid, NT, 0, s->stream>>>(s->f[CUP2D_VEL], s->f[CUP2D_TMPV], s->f[CUP2D_CHI],
                                                           s->f[CUP2D_POLD], s->f[CUP2D_TMP], s->f[CUP2D_PRES],
                                                           reinterpret_cast<const int4 *>(s->d_nbr), nrows, fac);
  s->launches++;
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

// own row + the rows above/below + W/E ghosts of  P = (x - avg) + pold  (Neumann ghost = own value)
__device__ __forceinline__ void rows_P(const double *__restrict__ x, const double *__restrict__ pold,
                                       double avg, int row0, int nvalid, const int4 nb, int y,
                                       double *sw, int lane, double (&c)[8], double (&up)[8],
                                       double (&dn)[8], double &gW, double &gE) {
  double t[8];
  // x part
  rows_load1(x, row0, nvalid, sw, lane, c);
  const bool act = lane < nvalid;
  const bool hasN = y < 7 || nb.w >= 0, hasS = y > 0 || nb.z >= 0;
  if (act) {
    if (y < 7) rows_peek1(sw, lane + 1, up);
    else if (nb.w >= 0) grow_load1(x, nb.w, 0, up);
    if (y > 0) rows_peek1(sw, lane - 1, dn);
    else if (nb.z >= 0) grow_load1(x, nb.z, 7, dn);
    gW = nb.x >= 0 ? x[(size_t)nb.x * 64 + y * 8 + 7] : 0.0;
    gE = nb.y >= 0 ? x[(size_t)nb.y * 64 + y * 8] : 0.0;
  }
  // pold part
  rows_load1(pold, row0, nvalid, sw, lane, t);
  if (act) {
#pragma unroll
    for (int i = 0; i < 8; i++) c[i] = (c[i] - avg) + t[i];
    if (hasN) {
      if (y < 7) rows_peek1(sw, lane + 1, t);
      else grow_load1(pold, nb.w, 0, t);
#pragma unroll
      for (int i = 0; i < 8; i++) up[i] = (up[i] - avg) + t[i];
    } else {
#pragma unroll
      for (int i = 0; i < 8; i++) up[i] = c[i];
    }
    if (hasS) {
      if (y > 0) rows_peek1(sw, lane - 1, t);
      else grow_load1(pold, nb.z, 7, t);
#pragma unroll
      for (int i = 0; i < 8; i++) dn[i] = (dn[i] - avg) + t[i];
    } else {
#pragma unroll
      for (int i = 0; i < 8; i++) dn[i] = c[i];
    }
    gW = nb.x >= 0 ? (gW - avg) + pold[(size_t)nb.x * 64 + y * 8 + 7] : c[0];
    gE = nb.y >= 0 ? (gE - avg) + pold[(size_t)nb.y * 64 + y * 8] : c[7];
  }
}

// pres = (x - avg) + pold ; vel += (-0.5 dt h) * grad(pres) / h^2        (main.cpp:7120-7187)
// x = Poisson solution (lives in a Krylov buffer), avg = its volume-weighted mean.  The reference's
// second mean (of the already mean-free field, main.cpp:7149-7166) is rounding noise and is dropped.
__global__ void __launch_bounds__(NT)
pressure_correct_kernel(const double *x0, const double *x1, const double *x2, const double *__restrict__ pold,
                        double *__restrict__ pres, double *__restrict__ vel,
                        const int4 *__restrict__ nbr, int nrows, const KrylovState *__restrict__ st,
                        double inv_ncells, double pfac_ih2_arg, const StepFactors *__restrict__ sf) {
  __shared__ __align__(16) double s_scr[WPB * ROWS_SCRATCH];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double *sw = s_scr + warp * ROWS_SCRATCH;
  // the best iterate is in the x buffer the device-side Krylov state names (no host copy of the state is needed)
  const int opt = st->opt;
  const double *__restrict__ x = opt == 0 ? x0 : (opt == 1 ? x1 : x2);
  const double avg = st->xsum * inv_ncells;
  const double pfac_ih2 = sf ? sf->corr_fac : pfac_ih2_arg;
  for (int row0 = (blockIdx.x * WPB + warp) * 32; row0 < nrows; row0 += gridDim.x * WPB * 32) {
    const int nv = min(32, nrows - row0);
    const int row = row0 + lane, slot = row >> 3, y = row & 7;
    const int4 nb = lane < nv ? nbr[slot] : make_int4(-1, -1, -1, -1);
    double c[8], up[8], dn[8], gW = 0, gE = 0;
    rows_P(x, pold, avg, row0, nv, nb, y, sw, lane, c, up, dn, gW, gE);
    rows_store1(pres, row0, nv, sw, lane, c);
    double2 v[8];
    rows_load2(vel, row0, nv, sw, lane, v);
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const double e = i < 7 ? c[i + 1] : gE, w = i > 0 ? c[i - 1] : gW;
      v[i].x = fma(pfac_ih2, e - w, v[i].x);
      v[i].y = fma(pfac_ih2, up[i] - dn[i], v[i].y);
    }
    rows_store2(vel, row0, nv, sw, lane, v);
  }
}

// pold_halo_current: the halo slots of pold are still those the right-hand-side kernel's refresh brought (inside one step
// nothing writes pold in between), so only the solution's halo is pulled
int launch_pressure_correct(cup2d_sim *s, double dt, const StepFactors *dev, bool pold_halo_current) {
  if (s->nranks > 1) {
    int rc;
    if ((rc = halo_exchange_xopt(s))) return rc;
    if (!pold_halo_current && (rc = halo_exchange_ptr(s, s->f[CUP2D_POLD], 1, CUP2D_POLD))) return rc;
  }
  const int nrows = (int)s->nloc * 8;
  const int grid = min((nrows + NT - 1) / NT, s->num_sms * 8);
  const double pfac = -0.5 * dt * s->h; // main.cpp:6028
  const double ih2 = 1.0 / s->h / s->h; // main.cpp:7182
  ProfScope prof(s, KC_CORRECT);
  pressure_correct_kernel<<<grid, NT, 0, s->stream>>>(
      s->kx[0], s->kx[1], s->kx[2], s->f[CUP2D_POLD], s->f[CUP2D_PRES], s->f[CUP2D_VEL], reinterpret_cast<const int4 *>(s->d_nbr),
      nrows, s->d_state, 1.0 / ((double)s->nglobal * 64.0), pfac * ih2, dev);
  s->launches++;
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

} // namespace cup2d
