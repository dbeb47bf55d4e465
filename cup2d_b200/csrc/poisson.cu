// Pressure-Poisson solve: block-Jacobi preconditioned BiCGSTAB, matrix-free, device-resident control.
//
// Restates BiCGSTABSolver::main (cuda.cu:403-548) — same recurrence, same operation order, same
// 1e-21 guards (cuda.cu:315-326), same breakdown/restart rule (cuda.cu:452-477), same L-inf stopping
// rule with best-iterate tracking (cuda.cu:525-541) — but
//   * A is applied matrix-free from the block neighbour table (the COO of main.cpp:7074-7107 on a
//     uniform level is the undivided 5-point Laplacian with Neumann walls), instead of cusparseSpMV;
//   * the preconditioner P_inv = -(A_loc)^-1 (main.cpp:6451-6488; cublasDgemm at cuda.cu:484,503) is
//     applied by fast diagonalisation: A_loc = T (x) I + I (x) T, T = tridiag(-1,2,-1) = Q L Q^T with
//     Q[j][k] = sqrt(2/9) sin((j+1)(k+1)pi/9), so z = -(Q(x)Q) diag(1/(l_i+l_j)) (Q(x)Q)^T v:
//     four 8x8 transforms per block (32 FMA/cell) instead of a 64x64 product (64 FMA/cell);
//   * the ~25 launches + 4 host syncs per iteration of the reference become 5 fused kernels and no
//     host sync: dots are reduced deterministically on the device, the scalar recurrences
//     (set_alpha/beta/omega/rho, cuda.cu:303-330) run in the last CTA of the producing kernel, the
//     x_opt snapshot (cuda.cu:537) is a rotation among three x buffers, and convergence is a device
//     flag that turns the remaining launches into no-ops.
// (On one rank with a uniform grid the five kernels become three, 120 B/cell: see k_p_spmv below.)
// Traffic per iteration: 23 doubles/cell = 184 B/cell (SURVEY.md §8(d) budgets 25 = 200 B): the half-step update
// x' = x + alpha z of cuda.cu:498 is deferred into the final kernel, which applies x'' = (x + alpha z_p) + omega z_r
// in the reference's order (bitwise the same iterate), so the middle kernel neither reads nor writes x or z_p.
// Memory access: warp-cooperative coalesced rows through padded shared memory (rows.cuh).
#include "rhs.cuh"
#include "sim.h"
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <type_traits>

namespace cup2d {

constexpr int NT = 256;
constexpr int WPB = NT / 32;
constexpr double EPS21 = 1e-21;    // cuda.cu:409
#ifndef SPMV_CTAS
#define SPMV_CTAS 3 // resident CTAs/SM of the SpMV kernels (80 registers); 4 is a measurement variant (make variant EXTRA=-DSPMV_CTAS=4)
#endif
#ifndef PRECOND_CTAS
#define PRECOND_CTAS 3 // resident CTAs/SM of the two preconditioner kernels (3: 73-78 regs; 4 (64 regs) measured 2 % slower)
#endif

// Fast diagonalisation constants.  S[j][k] = sin((j+1)(k+1) pi/9) (DST-I of length 8) has only four distinct
// magnitudes, so one transform is an even/odd split + two 4x4 products with zeros: 38 FP64 operations instead of
// 64, and four constants that live in uniform registers (the dense 64-entry table needed one LDC per FMA and spilled).
//   Q = sqrt(2/9) S,  Q^2 = I;   z = -(Q(x)Q) diag(1/(l_m+l_k)) (Q(x)Q) v = (S(x)S) [cIL .* ((S(x)S) v)]
__constant__ double cS[4];   // sin(pi/9), sin(2pi/9), sin(3pi/9), sin(4pi/9)
__constant__ double cIL[64]; // -(2/9)^2 / (lambda_m + lambda_k)

static int upload_consts() {
  double S[4], IL[64], lam[8];
  const double pi = 3.14159265358979323846;
  for (int k = 0; k < 4; k++) S[k] = std::sin((k + 1) * pi / 9.0);
  for (int k = 0; k < 8; k++) lam[k] = 2.0 - 2.0 * std::cos((k + 1) * pi / 9.0);
  for (int m = 0; m < 8; m++)
    for (int k = 0; k < 8; k++) IL[m * 8 + k] = -(4.0 / 81.0) / (lam[m] + lam[k]);
  CUP2D_CUDA(cudaMemcpyToSymbol(cS, S, sizeof S));
  CUP2D_CUDA(cudaMemcpyToSymbol(cIL, IL, sizeof IL));
  return CUP2D_OK;
}
static PerDeviceOnce g_consts;

// X[k] = sum_j x[j] sin((j+1)(k+1) pi/9).  sin((9-j')k' pi/9) = (-1)^(k'+1) sin(j'k' pi/9): odd modes see the
// symmetric part u of the input, even modes the antisymmetric part w.
__host__ __device__ __forceinline__ void dst8(const double (&x)[8], double (&X)[8], double a, double b, double c,
                                              double d) {
  const double u1 = x[0] + x[7], u2 = x[1] + x[6], u3 = x[2] + x[5], u4 = x[3] + x[4];
  const double w1 = x[0] - x[7], w2 = x[1] - x[6], w3 = x[2] - x[5], w4 = x[3] - x[4];
  X[0] = fma(d, u4, fma(c, u3, fma(b, u2, a * u1)));
  X[2] = c * ((u1 + u2) - u4);
  X[4] = fma(b, u4, fma(-c, u3, fma(-a, u2, d * u1)));
  X[6] = fma(-a, u4, fma(c, u3, fma(-d, u2, b * u1)));
  X[1] = fma(a, w4, fma(c, w3, fma(d, w2, b * w1)));
  X[3] = fma(-b, w4, fma(-c, w3, fma(a, w2, d * w1)));
  X[5] = c * ((w1 - w2) + w4);
  X[7] = fma(-d, w4, fma(c, w3, fma(-b, w2, a * w1)));
}

// z_blk = P_inv v_blk for the block whose row `y` this lane holds (8 lanes = one block).
// sw: per-warp scratch (>= 4*72 doubles).  All 32 lanes must call.
__device__ __forceinline__ void precond_row(double (&v)[8], double *sw, int lane) {
  const int y = lane & 7, bl = lane >> 3;
  double *sb = sw + bl * 72;
  const double sa = cS[0], sb_ = cS[1], sc = cS[2], sd = cS[3];
  double a[8], b[8];
  dst8(v, a, sa, sb_, sc, sd); // along x: lane = row y, a[k] = x-mode k
  __syncwarp();
#pragma unroll
  for (int k = 0; k < 8; k++) sb[y * 9 + k] = a[k];
  __syncwarp();
#pragma unroll
  for (int yy = 0; yy < 8; yy++) b[yy] = sb[yy * 9 + y]; // lane now owns x-mode kx = y, b[yy] over rows
  dst8(b, a, sa, sb_, sc, sd);                            // along y: a[m] = y-mode m
#pragma unroll
  for (int m = 0; m < 8; m++) a[m] *= cIL[m * 8 + y];
  dst8(a, b, sa, sb_, sc, sd); // back along y
  __syncwarp();
#pragma unroll
  for (int yy = 0; yy < 8; yy++) sb[yy * 9 + y] = b[yy];
  __syncwarp();
#pragma unroll
  for (int k = 0; k < 8; k++) a[k] = sb[y * 9 + k];
  dst8(a, v, sa, sb_, sc, sd); // back along x
}

__device__ __forceinline__ void set_gate(NoGate &, unsigned, const Comm &) {}
__device__ __forceinline__ void set_gate(HaloGate &g, unsigned src_mask, const Comm &comm) {
  g.mask = src_mask;
  g.comm = comm;
  g.target = ld_relaxed_sys(comm.mb[comm.rank] + MB_PEPOCH); // this rank's own producer has run: every rank is at this epoch
}
__device__ __forceinline__ int next_buf(int cur, int opt) { return cur != opt ? 3 - cur - opt : (cur + 1) % 3; }

// decisions taken at the top of the reference loop (cuda.cu:440-477), given rho' = rhat.r and |r|^2
__device__ void prepare_iteration(KrylovState *st, double rho_new, double nr2) {
  st->rho_curr = rho_new;
  st->nr2 = nr2;
  const bool breakdown = rho_new * rho_new < 1e-16 * nr2 * st->nrh2;                      // 452-454
  st->beta = (st->rho_curr / (st->rho_prev + EPS21)) * (st->alpha / (st->omega + EPS21)); // set_beta
  st->restart_now = 0;
  if (breakdown && st->max_restarts > 0) { // 457-477
    st->restarts++;
    if (st->restarts >= st->max_restarts) {
      st->done = 1;
      return;
    }
    st->restart_now = 1; // K1: rhat = r, p = r (p = nu = 0 then p = beta*0 + r)
    st->rho_curr = nr2;  // nrm2(rhat)^2 with rhat = r
    st->nrh2 = nr2;
    st->rho_prev = 1.0;  // breakdown_update, cuda.cu:308-314
    st->alpha = 1.0;
    st->omega = 1.0;
    st->beta = (st->rho_curr / (st->rho_prev + EPS21)) * (st->alpha / (st->omega + EPS21));
  }
}

// ---- halo rows of the Krylov operands, pushed by their producer (multi-rank contexts) --------------------------------
// z = M p and z_r = M r are consumed by the next kernel's stencil, which needs the face-neighbour blocks other ranks
// own.  Instead of a separate halo kernel between producer and consumer (launch + all-rank handshake + NVLink round
// trip on the critical path, twice per iteration), the producer writes every row of a block that some peer holds as a
// halo slot straight into that slot (plain remote stores: fire and forget) and its last CTA raises this rank's PUSHED
// flag in those peers' mailboxes; the consumer waits for the flags only in the lanes that touch a halo slot
// (rows.cuh: HaloGate).  Write-after-read safety: a peer pushes the next version of a slot only after the all-reduce of
// the consuming SpMV, which completes on no rank before every rank has finished that SpMV.
struct PushView {
  const int *first;        // [nloc]: first entry of the block's destinations, -1 = none
  const int2 *ent;         // (peer rank, halo slot on the peer) ..., (-1,-1)
  double *peer[MAX_RANKS]; // the vector's base address on every peer
  unsigned dst_mask;       // peers that hold halo slots of this rank's blocks
};
__device__ __forceinline__ void push_rows(const PushView &pv, int slot, int y, const double (&v)[8]) {
  const int pf = pv.first[slot];
  if (pf < 0) return;
  for (int e = pf;; e++) {
    const int2 d = pv.ent[e];
    if (d.x < 0) break;
    double2 *dst = reinterpret_cast<double2 *>(pv.peer[d.x] + (size_t)d.y * 64 + y * 8);
#pragma unroll
    for (int k = 0; k < 4; k++) dst[k] = make_double2(v[2 * k], v[2 * k + 1]);
  }
  // no fence here: push_finish orders these stores before the flag for the whole CTA (CTA barrier, then ONE system-scope
  // fence by the thread that takes part in the release chain — fences are cumulative over what the barrier made visible
  // to that thread, the same pattern a cooperative grid barrier relies on).  A fence per pushing lane stalled every
  // perimeter warp for an NVLink round trip.
}
// end of a pushing kernel: the CTA that finishes last publishes the new push epoch to the destination ranks
__device__ __forceinline__ void push_finish(const PushView &pv, const Comm &comm, unsigned int *counter) {
  __shared__ bool s_push_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    s_push_last = atomicAdd(counter, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!s_push_last) return;
  unsigned long long *mine = comm.mb[comm.rank];
  const unsigned long long e = ld_relaxed_sys(mine + MB_PEPOCH) + 1;
  if ((int)threadIdx.x < comm.nranks && ((pv.dst_mask >> threadIdx.x) & 1u)) {
    __threadfence_system();
    st_release_sys(comm.mb[threadIdx.x] + MB_PUSHED + comm.rank, e);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    *counter = 0;
    st_relaxed_sys(mine + MB_PEPOCH, e);
  }
}

// Krylov state of a new solve, written on the device from by-value arguments (a host-to-device copy of a staging
// struct would be read when the copy executes, i.e. possibly after the host has prepared the next solve)
__global__ void k_state_init(KrylovState *st, double tol_abs, double tol_rel, int max_restarts, int max_iter) {
  KrylovState z = KrylovState{};
  z.alpha = z.omega = z.rho_prev = z.rho_curr = 1.0; // cuda.cu:409
  z.tol_abs = tol_abs;
  z.tol_rel = tol_rel;
  z.max_restarts = max_restarts;
  z.max_iter = max_iter;
  *st = z;
}

// end-of-iteration logic of the reference loop (cuda.cu:525-541, 438), run by one thread with the global sums
__device__ void end_of_iteration(KrylovState *st, const double *tsum, double m, int nxt) {
  st->iter++;
  st->err = m;
  st->cur = nxt;
  if (m < st->err_opt) { // cuda.cu:535-541
    st->err_opt = m;
    st->opt = nxt;
    st->xsum = tsum[2];
    if (m <= st->tol_abs || m / st->err_init <= st->tol_rel) {
      st->done = 1;
      return;
    }
  }
  st->rho_prev = st->rho_curr; // set_rho
  if (st->iter >= st->max_iter) { // cuda.cu:438
    st->done = 1;
    return;
  }
  prepare_iteration(st, tsum[0], tsum[1]);
}
// a solve captured as the body of a graph WHILE node keeps iterating while its condition is non-zero
__device__ __forceinline__ void set_loop_condition(unsigned long long handle, const KrylovState *st) {
#ifndef CUP2D_FULL_EMU
  if (handle) cudaGraphSetConditional((cudaGraphConditionalHandle)handle, st->done ? 0u : 1u);
#endif
}

#define CHUNK_LOOP()                                                                              \
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;                                     \
  double *sw = s_scr + warp * SCR1;                                                               \
  for (int row0 = (blockIdx.x * WPB + warp) * 32; row0 < nrows; row0 += gridDim.x * WPB * 32)

// state of a solve after its start kernel, from the global |r|^2, sum(x0) and |r|_inf (cuda.cu:428-430)
__device__ void start_of_solve(KrylovState *st, const double *t, double m, unsigned long long loop_handle) {
  st->err = st->err_init = st->err_opt = m;
  st->xsum = t[1];
  st->nrh2 = t[0];
  st->iter = 0;
  if (st->max_iter <= 0) st->done = 1;
  prepare_iteration(st, t[0], t[0]);
  set_loop_condition(loop_handle, st);
}

// ---- K0: r = b - A x0 ; rhat = r ; x[0] = x0 ; err0, |r|^2, sum(x0) -----------------
// p = nu = 0 is not stored: the first p-update of a solve (iter 0) takes p = r, which is beta*(0 - omega*0) + r.
template <bool IRR>
__global__ void __launch_bounds__(NT)
k_init(const double *__restrict__ b, const double *__restrict__ x0, double *__restrict__ x,
       double *__restrict__ r, double *__restrict__ rhat, const int4 *__restrict__ nbr, int nrows, KrylovState *st,
       double *partials, unsigned int *counter, Comm comm, IrrView irr, unsigned long long loop_handle) {
  __shared__ __align__(16) double s_scr[WPB * SCR1];
  double sums[2] = {0, 0}; // |r|^2, sum x0
  double mx = 0;
  CHUNK_LOOP() {
    const int nv = min(32, nrows - row0);
    double xx[8], ax[8], bb[8];
    double2 cx0[4], cb[4];
    chunk_ld(x0, row0, nv, lane, cx0);
    chunk_ld(b, row0, nv, lane, cb);
    rows_lap_c(cx0, x0, row0, nv, nbr, sw, lane, xx, ax, IRR ? irr : IrrView());
    chunk_to_rows(sw, lane, cb, bb);
#pragma unroll
    for (int i = 0; i < 8; i++) {
      bb[i] -= ax[i];
      sums[0] = fma(bb[i], bb[i], sums[0]);
      sums[1] += xx[i];
      mx = fmax(mx, fabs(bb[i]));
    }
    rows_store1(r, row0, nv, sw, lane, bb);
    rows_store1(rhat, row0, nv, sw, lane, bb);
    rows_store1(x, row0, nv, sw, lane, xx);
  }
  grid_reduce<2, NT>(sums, mx, partials, counter, comm,
                     [=](const double *t, double m) { start_of_solve(st, t, m, loop_handle); });
}

// ---- K0 of a time step: b = fac*(div vel) - fac*chi*(div udef) - lap(pold) ; r = rhat = b ; x[0] = 0 ; err0, |r|^2 -------
// k_init with x0 = 0 fused into the right-hand-side kernel: A*0 = +0 (for general rows too), so r = b - A*0 is b bit for
// bit, and neither b nor x0 makes a round trip through tmp / pres.  Launched on k_init's grid with its row partition and
// per-lane summation order, so |r|^2, |r|_inf and sum(x0) = +0 are bitwise what k_init returns for b and x0 = 0.
template <bool HAS_UDEF>
__global__ void __launch_bounds__(NT)
pressure_rhs_start_kernel(const double *__restrict__ vel, const double *__restrict__ udef, const double *__restrict__ chi,
                          const double *__restrict__ pold, double *__restrict__ x, double *__restrict__ r,
                          double *__restrict__ rhat, const int4 *__restrict__ nbr, int nrows,
                          const StepFactors *__restrict__ sf, KrylovState *st, double *partials, unsigned int *counter,
                          Comm comm, unsigned long long loop_handle) {
  __shared__ __align__(16) double s_scr[WPB * ROWS_SCRATCH];
  const double fac = sf->rhs_fac;
  double sums[2] = {0, 0}; // |r|^2, sum x0 (= +0)
  double mx = 0;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double *sw = s_scr + warp * ROWS_SCRATCH;
  for (int row0 = (blockIdx.x * WPB + warp) * 32; row0 < nrows; row0 += gridDim.x * WPB * 32) {
    const int nv = min(32, nrows - row0);
    double bb[8];
    rhs_rows<HAS_UDEF>(vel, udef, chi, pold, nbr, row0, nv, fac, sw, lane, bb);
#pragma unroll
    for (int i = 0; i < 8; i++) {
      sums[0] = fma(bb[i], bb[i], sums[0]);
      mx = fmax(mx, fabs(bb[i]));
    }
    double2 cb[4];
    rows_to_chunk(sw, lane, bb, cb);
    chunk_st(r, row0, nv, lane, cb);
    chunk_st(rhat, row0, nv, lane, cb);
    const double2 zero[4] = {};
    chunk_st(x, row0, nv, lane, zero);
  }
  grid_reduce<2, NT>(sums, mx, partials, counter, comm, [=](const double *t, double m) {
    start_of_solve(st, t, m, loop_handle);
    st->x0_zero = 1;
  });
}

// ---- K1: p = r + beta (p - omega nu) ; z = M p    (cuda.cu:478-486) -------------------------------
template <bool MULTI>
__global__ void __launch_bounds__(NT, PRECOND_CTAS)
k_pupdate(const double *__restrict__ r, double *__restrict__ rhat, double *__restrict__ p,
          const double *__restrict__ nu, double *__restrict__ z, int nrows,
          const KrylovState *__restrict__ st, PushView pv, Comm comm, unsigned int *counter) {
  __shared__ __align__(16) double s_scr[WPB * SCR1];
  if (st->done) return;
  const double beta = st->beta, nomega = -st->omega;
  const bool restart = st->restart_now != 0, first = st->iter == 0;
  CHUNK_LOOP() {
    const int nv = min(32, nrows - row0);
    // element-wise part in chunk layout (coalesced, no shared memory)
    double2 cp[4], cr[4];
    chunk_ld(r, row0, nv, lane, cr);
    if (restart || first) { // p = r: p = nu = 0 at the start of a solve and after a restart (k_init stores neither)
      if (restart) chunk_st(rhat, row0, nv, lane, cr);
#pragma unroll
      for (int j = 0; j < 4; j++) cp[j] = cr[j];
    } else {
      double2 cn[4];
      chunk_ld(p, row0, nv, lane, cp);
      chunk_ld(nu, row0, nv, lane, cn);
#pragma unroll
      for (int j = 0; j < 4; j++) {
        cp[j].x = fma(beta, fma(nomega, cn[j].x, cp[j].x), cr[j].x);
        cp[j].y = fma(beta, fma(nomega, cn[j].y, cp[j].y), cr[j].y);
      }
    }
    chunk_st(p, row0, nv, lane, cp);
    // block preconditioner in row layout
    double pp[8];
    chunk_to_rows(sw, lane, cp, pp);
    precond_row(pp, sw, lane);
    rows_store1(z, row0, nv, sw, lane, pp);
    if (MULTI && lane < nv) push_rows(pv, (row0 + lane) >> 3, lane & 7, pp);
  }
  if (MULTI) push_finish(pv, comm, counter);
}

// ---- K2 / K4: y = A z with one or two dots against `d` and y -------------------------------------
//   MODE 0 (K2): nu = A z ; rhat.nu             -> alpha = rho/(rhat.nu + eps)   (cuda.cu:487-496)
//   MODE 1 (K4): t  = A z ; t.r, t.t            -> omega = t.r/(t.t + eps)       (cuda.cu:506-518)
//   MULTI: the halo rows of z were pushed by the peers' producing kernels; lanes that touch them wait for the flags
template <int MODE, bool IRR, bool MULTI>
__global__ void __launch_bounds__(NT, SPMV_CTAS)
k_spmv(const double *__restrict__ z, const double *__restrict__ d, double *__restrict__ yout,
       const int4 *__restrict__ nbr, int nrows, KrylovState *st, double *partials,
       unsigned int *counter, Comm comm, IrrView irr, unsigned src_mask) {
  constexpr bool COOP = CUP2D_ROWS_COOP && !MULTI; // see the call below
  constexpr int SCRW = COOP ? SCR_COOP : SCR1;
  __shared__ __align__(16) double s_scr[WPB * SCRW];
  if (st->done) return;
  typename std::conditional<MULTI, HaloGate, NoGate>::type gate;
  if (MULTI) {
    gate.nloc = nrows >> 3;
    set_gate(gate, src_mask, comm);
    if (IRR) { // general rows may name any halo slot: every CTA waits before it starts
      if (threadIdx.x == 0) gate.wait();
      __syncthreads();
    }
  }
  double sums[2] = {0, 0};
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double *sw = s_scr + warp * SCRW;
  for (int row0 = (blockIdx.x * WPB + warp) * 32; row0 < nrows; row0 += gridDim.x * WPB * 32) {
    const int nv = min(32, nrows - row0);
    // uniform grids: both global loads are issued before any shared-memory work (memory-level parallelism); with general
    // rows the extra live registers cost more than that
    constexpr bool HOIST = !IRR;
    double2 cz[4], ca[4], cd[4];
    chunk_ld(z, row0, nv, lane, cz);
    if (HOIST) chunk_ld(d, row0, nv, lane, cd);
    double zz[8], az[8];
    // one GPU: the cooperative form (rows.cuh).  Several ranks keep the plain form; the cooperative form handles halo
    // slots too (emulated 2-rank tests) but has not been timed or run on more than one GPU
    if (COOP) rows_lap_coop(cz, z, row0, nv, nbr, sw, lane, zz, az, IRR ? irr : IrrView(), gate);
    else rows_lap_c(cz, z, row0, nv, nbr, sw, lane, zz, az, IRR ? irr : IrrView(), gate);
    // back to chunk layout: the dots and the store are element-wise
    if (!HOIST) chunk_ld(d, row0, nv, lane, cd);
    rows_to_chunk(sw, lane, az, ca);
#pragma unroll
    for (int j = 0; j < 4; j++) {
      sums[0] = fma(ca[j].x, cd[j].x, sums[0]);
      sums[0] = fma(ca[j].y, cd[j].y, sums[0]);
      if (MODE == 1) {
        sums[1] = fma(ca[j].x, ca[j].x, sums[1]);
        sums[1] = fma(ca[j].y, ca[j].y, sums[1]);
      }
    }
    chunk_st(yout, row0, nv, lane, ca);
  }
  grid_reduce<2, NT>(sums, 0.0, partials, counter, comm, [=](const double *t, double) {
    if (MODE == 0) {
      st->rhat_nu = t[0];
      st->alpha = st->rho_curr / (t[0] + EPS21); // set_alpha
      st->restart_now = 0;
    } else {
      st->tr = t[0];
      st->tt = t[1];
      st->omega = t[0] / (t[1] + EPS21); // set_omega
    }
  });
}

// ---- K3: r -= alpha nu ; z_r = M r     (cuda.cu:499-505; the x half-step of cuda.cu:498 happens in K5) ----------
template <bool MULTI>
__global__ void __launch_bounds__(NT, PRECOND_CTAS)
k_r_update(double *__restrict__ r, const double *__restrict__ nu, double *__restrict__ zr, int nrows,
           const KrylovState *__restrict__ st, PushView pv, Comm comm, unsigned int *counter) {
  __shared__ __align__(16) double s_scr[WPB * SCR1];
  if (st->done) return;
  const double alpha = st->alpha;
  CHUNK_LOOP() {
    const int nv = min(32, nrows - row0);
    // element-wise part in chunk layout (coalesced, no shared memory)
    double2 cr[4], cn[4];
    chunk_ld(r, row0, nv, lane, cr);
    chunk_ld(nu, row0, nv, lane, cn);
#pragma unroll
    for (int j = 0; j < 4; j++) {
      cr[j].x = fma(-alpha, cn[j].x, cr[j].x);
      cr[j].y = fma(-alpha, cn[j].y, cr[j].y);
    }
    chunk_st(r, row0, nv, lane, cr);
    // block preconditioner in row layout
    double rr[8];
    chunk_to_rows(sw, lane, cr, rr);
    precond_row(rr, sw, lane);
    rows_store1(zr, row0, nv, sw, lane, rr);
    if (MULTI && lane < nv) push_rows(pv, (row0 + lane) >> 3, lane & 7, rr);
  }
  if (MULTI) push_finish(pv, comm, counter);
}

// ---- K5: x = (x + alpha z_p) + omega z_r ; r -= omega t ; err, rhat.r, |r|^2, sum(x) ; end-of-iteration logic ----
// The new iterate goes to the x buffer that holds neither the current nor the best iterate (x_opt snapshot of
// cuda.cu:537 without a copy).
__global__ void __launch_bounds__(NT)
k_final(double *x0, double *x1, double *x2, const double *__restrict__ zp, const double *__restrict__ zr,
        double *__restrict__ r, const double *__restrict__ t, const double *__restrict__ rhat, int nrows,
        KrylovState *st, double *partials, unsigned int *counter, Comm comm, unsigned long long loop_handle) {
  if (st->done) return;
  const double alpha = st->alpha, omega = st->omega;
  const int cur = st->cur, nxt = next_buf(st->cur, st->opt);
  const double *xc = cur == 0 ? x0 : (cur == 1 ? x1 : x2);
  double *xn = nxt == 0 ? x0 : (nxt == 1 ? x1 : x2);
  double sums[3] = {0, 0, 0}; // rhat.r, r.r, sum x
  double mx = 0;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int row0 = (blockIdx.x * WPB + warp) * 32; row0 < nrows; row0 += gridDim.x * WPB * 32) {
    const int nv = min(32, nrows - row0);
    // purely element-wise: chunk layout only, no shared memory
    double2 cx[4], cz[4], cy[4], cr[4], ct[4], ch[4];
    chunk_ld(xc, row0, nv, lane, cx);
    chunk_ld(zp, row0, nv, lane, cz);
    chunk_ld(zr, row0, nv, lane, cy);
    chunk_ld(r, row0, nv, lane, cr);
    chunk_ld(t, row0, nv, lane, ct);
    chunk_ld(rhat, row0, nv, lane, ch);
#pragma unroll
    for (int j = 0; j < 4; j++) {
      cx[j].x = fma(omega, cy[j].x, fma(alpha, cz[j].x, cx[j].x)); // cuda.cu:498 then 520
      cx[j].y = fma(omega, cy[j].y, fma(alpha, cz[j].y, cx[j].y));
      cr[j].x = fma(-omega, ct[j].x, cr[j].x); // cuda.cu:524
      cr[j].y = fma(-omega, ct[j].y, cr[j].y);
      sums[0] = fma(ch[j].x, cr[j].x, sums[0]);
      sums[0] = fma(ch[j].y, cr[j].y, sums[0]);
      sums[1] = fma(cr[j].x, cr[j].x, sums[1]);
      sums[1] = fma(cr[j].y, cr[j].y, sums[1]);
      sums[2] += cx[j].x + cx[j].y;
      mx = fmax(mx, fmax(fabs(cr[j].x), fabs(cr[j].y)));
    }
    chunk_st(xn, row0, nv, lane, cx);
    chunk_st(r, row0, nv, lane, cr);
  }
  grid_reduce<3, NT>(sums, mx, partials, counter, comm, [=](const double *tsum, double m) {
    end_of_iteration(st, tsum, m, nxt);
    set_loop_condition(loop_handle, st);
  });
}

// ==== single-rank uniform grids: the same iteration in three kernels that recompute z = M p and z_r = M r ================
// M is block-local (about 19 FP64 operations per cell), so recomputing it is cheaper than writing z and reading it back:
// the iteration moves 15 doubles per cell instead of 23.  What stands in the way is the SpMV after each preconditioner: it
// needs z on the face-neighbour blocks, and z there depends on the whole neighbour block.  So the kernels work on the
// advect stage's tiles (4x4 blocks + their 16 ring blocks) and precondition the ring blocks themselves:
//   k_p_spmv  (KA): p' = r + beta (p - omega nu) ; z = M p' on tile + ring ; nu' = A z ; rhat.nu' -> alpha      r p nu rhat | p' nu'
//   k_r_spmv  (KB): r' = r - alpha nu' ; z_r = M r' on tile + ring ; t = A z_r ; t.r', t.t -> omega               r nu'       | r'
//   k_x_final (KC): z_r = M r' on tile + ring ; t = A z_r ; z_p = M p' ; x = (x + alpha z_p) + omega z_r ;
//                   r = r' - omega t ; rhat.r, |r|^2, sum x, |r|_inf                                            x p' r' rhat | x r
// KC reads r' of the ring blocks too, mostly from L2.  Every element-wise value is computed by the same expression from the
// same operands as in the five-kernel path above; only the partition of the dot products differs.  KA reads p and nu of
// ring blocks, so it must not write them in place: (p, nu) alternate between (kp, knu) and (kz, kzr) by the parity of the
// iteration count, which one captured iteration body of the graph WHILE node serves for every pass (iteration 0 reads
// neither: p = r).  r stays in kr and r' in kt: KB reads r of ring blocks and writes r' to kt, KC reads r' of ring blocks
// and writes r to kr, so neither writes a vector that another of its CTAs reads.
#ifndef KTILE_CTAS
#define KTILE_CTAS 2 // resident CTAs/SM k_p_spmv and k_x_final are register-bounded for (128 registers; at 3 (80) both spill)
#endif
constexpr int PST = 34; // tile plane row stride in doubles: 16-byte rows, conflict-free 128-bit row reads of a warp

__device__ __forceinline__ int pair_in(const KrylovState *st) { return st->iter & 1; }

// chunk layout of the warp's four blocks (any slots; -1 = absent): c[j] = piece `lane` of block sl[j] (as chunk_ld for four
// consecutive blocks, so chunk_to_rows / rows_to_chunk apply unchanged)
__device__ __forceinline__ void blocks_ld(const double *__restrict__ f, const int (&sl)[4], int lane, double2 (&c)[4]) {
#pragma unroll
  for (int j = 0; j < 4; j++)
    c[j] = sl[j] >= 0 ? reinterpret_cast<const double2 *>(f + (size_t)sl[j] * 64)[lane] : make_double2(0.0, 0.0);
}
__device__ __forceinline__ void blocks_st(double *__restrict__ f, const int (&sl)[4], int lane, const double2 (&c)[4]) {
#pragma unroll
  for (int j = 0; j < 4; j++)
    if (sl[j] >= 0) reinterpret_cast<double2 *>(f + (size_t)sl[j] * 64)[lane] = c[j];
}

// A load that stays in flight while the tile is computed: 16-byte cp.async (SASS LDGSTS) of each lane's pieces of the
// warp's four blocks into a per-warp stage in shared memory (128 double2, [block][lane]), no registers held meanwhile.  A
// lane reads back only what it copied itself, so cp.async.wait_all is all the data needs; the caller rewrites a stage
// only after a CTA barrier that follows the stage's last read.
__device__ __forceinline__ void stage_ld16(void *smem_dst, const void *gmem_src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void stage_wait() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ void blocks_stage(double2 *stg, const double *f, const int (&sl)[4], int lane) {
#pragma unroll
  for (int j = 0; j < 4; j++)
    if (sl[j] >= 0) stage_ld16(stg + j * 32 + lane, f + (size_t)sl[j] * 64 + 2 * lane);
}
// after stage_wait(): the chunk layout blocks_ld would have loaded
__device__ __forceinline__ void blocks_unstage(const double2 *stg, const int (&sl)[4], int lane, double2 (&c)[4]) {
#pragma unroll
  for (int j = 0; j < 4; j++) c[j] = sl[j] >= 0 ? stg[j * 32 + lane] : make_double2(0.0, 0.0);
}

// Shared memory of a tile: z of the 16 interior blocks (plane rows 1..32), row 7 of the S ring blocks (plane row 0),
// row 0 of the N ring blocks (plane row 33), column 7 of the W and column 0 of the E ring blocks.
struct __align__(16) TileSmem {
  double plane[34 * PST];
  double wcol[32], ecol[32];
};

// Warp w holds the blocks tiles[4w .. 4w+3] in row layout (lane = block lane>>3, row lane&7): warps 0-3 the interior block
// rows, warps 4-7 the W, E, S, N ring blocks.  v: the vector to precondition; on return the interior warps hold
// out = A M v of their rows in chunk layout (zero for absent blocks), and M v of the interior blocks stays in the plane
// until the next call's first CTA barrier; warps 4-7 return right after the plane is complete (out unset).  All threads
// call.  Walls: ghost = own cell.
__device__ __forceinline__ void tile_precond_lap(double (&v)[8], TileSmem &ts, double *sw, int lane, int warp,
                                                 const int *__restrict__ tslots, double2 (&out)[4]) {
  precond_row(v, sw, lane);
  const int bx = lane >> 3, y = lane & 7;
  __syncthreads(); // the previous tile's reads of the plane are done
  if (warp < 4) {
    double2 *p = reinterpret_cast<double2 *>(ts.plane + (warp * 8 + y + 1) * PST + bx * 8);
#pragma unroll
    for (int k = 0; k < 4; k++) p[k] = make_double2(v[2 * k], v[2 * k + 1]);
  } else if (warp == 4) {
    ts.wcol[bx * 8 + y] = v[7];
  } else if (warp == 5) {
    ts.ecol[bx * 8 + y] = v[0];
  } else if ((warp == 6 && y == 7) || (warp == 7 && y == 0)) {
    double2 *p = reinterpret_cast<double2 *>(ts.plane + (warp == 6 ? 0 : 33) * PST + bx * 8);
#pragma unroll
    for (int k = 0; k < 4; k++) p[k] = make_double2(v[2 * k], v[2 * k + 1]);
  }
  __syncthreads();
  if (warp >= 4) return;
  const int by = warp, R = by * 8 + y;
  double o[8];
  if (tslots[by * 4 + bx] < 0) {
#pragma unroll
    for (int i = 0; i < 8; i++) o[i] = 0.0;
  } else {
    const bool hN = y < 7 || tslots[by < 3 ? (by + 1) * 4 + bx : 28 + bx] >= 0;
    const bool hS = y > 0 || tslots[by > 0 ? (by - 1) * 4 + bx : 24 + bx] >= 0;
    const bool hW = tslots[bx > 0 ? by * 4 + bx - 1 : 16 + by] >= 0;
    const bool hE = tslots[bx < 3 ? by * 4 + bx + 1 : 20 + by] >= 0;
    const double *pl = ts.plane + (R + 1) * PST + bx * 8;
    const double2 *pu = reinterpret_cast<const double2 *>(pl + PST), *pd = reinterpret_cast<const double2 *>(pl - PST);
    const double gW = hW ? (bx > 0 ? pl[-1] : ts.wcol[R]) : v[0];
    const double gE = hE ? (bx < 3 ? pl[8] : ts.ecol[R]) : v[7];
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const int i = 2 * k;
      const double2 u = hN ? pu[k] : make_double2(v[i], v[i + 1]), d = hS ? pd[k] : make_double2(v[i], v[i + 1]);
      const double w0 = i > 0 ? v[i - 1] : gW, e1 = i + 1 < 7 ? v[i + 2] : gE;
      o[i] = (((d.x + w0) + v[i + 1]) + u.x) - 4.0 * v[i]; // summation order S,W,E,N then -4C (rows_lap_coop)
      o[i + 1] = (((d.y + v[i]) + e1) + u.y) - 4.0 * v[i + 1];
    }
  }
  rows_to_chunk(sw, lane, o, out);
}

#define TILE_LOOP()                                                                               \
  __shared__ __align__(16) double s_scr[WPB * SCR1];                                              \
  __shared__ TileSmem s_tile;                                                                     \
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;                                     \
  double *sw = s_scr + warp * SCR1;                                                               \
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x)

// ---- KA: p' = r + beta (p - omega nu) ; nu' = A M p' ; rhat.nu' -> alpha   (cuda.cu:478-496) ----------------------------
__global__ void __launch_bounds__(NT, KTILE_CTAS)
k_p_spmv(const double *__restrict__ r, double *__restrict__ rhat, double *p0, double *p1, double *nu0, double *nu1,
         const int *__restrict__ tiles, int ntiles, KrylovState *st, double *partials, unsigned int *counter, Comm comm) {
  if (st->done) return;
  const double beta = st->beta, nomega = -st->omega;
  const bool restart = st->restart_now != 0, first = st->iter == 0;
  const int in = pair_in(st);
  const double *__restrict__ p = in ? p1 : p0;
  const double *__restrict__ nu = in ? nu1 : nu0;
  double *__restrict__ pn = in ? p0 : p1;
  double *__restrict__ nun = in ? nu0 : nu1;
  double sums[2] = {0, 0};
  // r^ of the interior blocks is needed only after the preconditioner: it is copied into a stage when the tile starts, so
  // its load overlaps the preconditioner and the stencil.  Two stages, alternating by tile: a copy is issued only after the
  // CTA barriers of the tile that read the stage last.  Iteration 0 and a restart read no r^: it equals r bit for bit (the
  // start kernel stored r^ = r; a restart stores it here).
  const bool rhat_is_r = restart || first;
  __shared__ __align__(16) double2 s_rhat[2 * 4 * 128];
  int par = 0;
  TILE_LOOP() {
    const int *ts = tiles + (size_t)tile * TILE_SLOTS;
    int sl[4];
#pragma unroll
    for (int j = 0; j < 4; j++) sl[j] = ts[4 * warp + j];
    double2 *stg = s_rhat + (par * 4 + (warp & 3)) * 128;
    if (warp < 4 && !rhat_is_r) blocks_stage(stg, rhat, sl, lane);
    double2 cp[4], cr[4], ch[4];
    blocks_ld(r, sl, lane, cr);
    if (rhat_is_r) { // p = r, as in k_pupdate
#pragma unroll
      for (int j = 0; j < 4; j++) cp[j] = ch[j] = cr[j];
      if (restart && warp < 4) blocks_st(rhat, sl, lane, cr);
    } else {
      double2 cn[4];
      blocks_ld(p, sl, lane, cp);
      blocks_ld(nu, sl, lane, cn);
#pragma unroll
      for (int j = 0; j < 4; j++) {
        cp[j].x = fma(beta, fma(nomega, cn[j].x, cp[j].x), cr[j].x);
        cp[j].y = fma(beta, fma(nomega, cn[j].y, cp[j].y), cr[j].y);
      }
    }
    if (warp < 4) blocks_st(pn, sl, lane, cp);
    double v[8];
    chunk_to_rows(sw, lane, cp, v);
    double2 ca[4];
    tile_precond_lap(v, s_tile, sw, lane, warp, ts, ca);
    if (warp < 4) {
      if (!rhat_is_r) { // held in registers across the preconditioner it would cost spills
        stage_wait();
        blocks_unstage(stg, sl, lane, ch);
      }
#pragma unroll
      for (int j = 0; j < 4; j++) {
        sums[0] = fma(ca[j].x, ch[j].x, sums[0]);
        sums[0] = fma(ca[j].y, ch[j].y, sums[0]);
      }
      blocks_st(nun, sl, lane, ca);
    }
    par ^= 1;
  }
  grid_reduce<2, NT>(sums, 0.0, partials, counter, comm, [=](const double *t, double) {
    st->rhat_nu = t[0];
    st->alpha = st->rho_curr / (t[0] + EPS21); // set_alpha
    st->restart_now = 0;
  });
}

#ifndef KR_CTAS
// k_r_spmv holds fewer values than the other two: bounded for 3 CTAs/SM it needs 80 registers and spills 48 bytes, and is
// still faster than at 2 (more warps to cover its loads).  It launches one wave of its own, so its dot products are
// partitioned over other CTAs than k_p_spmv's.
#define KR_CTAS 3
#endif
// ---- KB: r' = r - alpha nu' ; t = A M r' ; t.r', t.t -> omega   (cuda.cu:499-518) -------------------------------------
// Stores r' (not t): k_x_final recomputes t on its tile, which costs less than writing t and reading it back.
__global__ void __launch_bounds__(NT, KR_CTAS)
k_r_spmv(const double *__restrict__ r, const double *nu0, const double *nu1, double *__restrict__ rp,
         const int *__restrict__ tiles, int ntiles, KrylovState *st, double *partials, unsigned int *counter, Comm comm) {
  if (st->done) return;
  const double alpha = st->alpha;
  const double *__restrict__ nu = pair_in(st) ? nu0 : nu1; // what k_p_spmv of this iteration wrote
  double sums[2] = {0, 0};
  TILE_LOOP() {
    const int *ts = tiles + (size_t)tile * TILE_SLOTS;
    int sl[4];
#pragma unroll
    for (int j = 0; j < 4; j++) sl[j] = ts[4 * warp + j];
    double2 cr[4], cn[4];
    blocks_ld(r, sl, lane, cr);
    blocks_ld(nu, sl, lane, cn);
#pragma unroll
    for (int j = 0; j < 4; j++) {
      cr[j].x = fma(-alpha, cn[j].x, cr[j].x);
      cr[j].y = fma(-alpha, cn[j].y, cr[j].y);
    }
    if (warp < 4) blocks_st(rp, sl, lane, cr);
    double v[8];
    chunk_to_rows(sw, lane, cr, v);
    double2 ca[4];
    tile_precond_lap(v, s_tile, sw, lane, warp, ts, ca);
    if (warp < 4) {
#pragma unroll
      for (int j = 0; j < 4; j++) {
        sums[0] = fma(ca[j].x, cr[j].x, sums[0]);
        sums[0] = fma(ca[j].y, cr[j].y, sums[0]);
        sums[1] = fma(ca[j].x, ca[j].x, sums[1]);
        sums[1] = fma(ca[j].y, ca[j].y, sums[1]);
      }
    }
  }
  grid_reduce<2, NT>(sums, 0.0, partials, counter, comm, [=](const double *tsum, double) {
    st->tr = tsum[0];
    st->tt = tsum[1];
    st->omega = tsum[0] / (tsum[1] + EPS21); // set_omega
  });
}

// ---- KC: t = A M r' ; x = (x + alpha M p') + omega M r' ; r = r' - omega t ; rhat.r, |r|^2, sum x, |r|_inf --------------
// t is recomputed on the tile from the r' that k_r_spmv stored.  Warps 0-3 then hold t of the interior block rows and form
// r; warps 4-7, done with their ring blocks, form x of interior block row warp-4 from z_p = M p' and from z_r, which they
// read from the plane (rows 1..32, chunk layout).  The plane is overwritten only after the next tile's first CTA barrier,
// which every warp reaches after it has finished this tile.  When the tile starts, warps 0-3 copy r^ into a stage (as
// k_p_spmv does) and keep r' in registers, and warps 4-7 keep p'; x is loaded after the stencil: held across the tile
// with the others it would cost spills.  Iteration 0 of a solve that started from x0 = +0 (a time step's) loads no x.
__global__ void __launch_bounds__(NT, KTILE_CTAS)
k_x_final(double *x0, double *x1, double *x2, const double *p0, const double *p1, double *__restrict__ r,
          const double *__restrict__ rp, const double *__restrict__ rhat, const int *__restrict__ tiles, int ntiles,
          KrylovState *st, double *partials, unsigned int *counter, Comm comm, unsigned long long loop_handle) {
  if (st->done) return;
  const double alpha = st->alpha, omega = st->omega;
  const int cur = st->cur, nxt = next_buf(st->cur, st->opt);
  const double *xc = cur == 0 ? x0 : (cur == 1 ? x1 : x2);
  double *xn = nxt == 0 ? x0 : (nxt == 1 ? x1 : x2);
  const double *__restrict__ p = pair_in(st) ? p0 : p1; // what k_p_spmv of this iteration wrote
  const bool x_zero = st->x0_zero && st->iter == 0;
  double sums[3] = {0, 0, 0}; // rhat.r, r.r, sum x
  double mx = 0;
  __shared__ __align__(16) double2 s_rhat[2 * 4 * 128]; // two stages, alternating by tile (see k_p_spmv)
  int par = 0;
  TILE_LOOP() {
    const int *ts = tiles + (size_t)tile * TILE_SLOTS;
    int sl[4], il[4]; // the warp's blocks; the interior blocks of block row warp & 3
#pragma unroll
    for (int j = 0; j < 4; j++) {
      sl[j] = ts[4 * warp + j];
      il[j] = ts[4 * (warp & 3) + j];
    }
    double2 *stg = s_rhat + (par * 4 + (warp & 3)) * 128;
    if (warp < 4) blocks_stage(stg, rhat, sl, lane);
    double2 cr[4], ca[4]; // ca: r' (warps 0-3) or p' (warps 4-7) of block row warp & 3
    blocks_ld(rp, sl, lane, cr);
    if (warp < 4) {
#pragma unroll
      for (int j = 0; j < 4; j++) ca[j] = cr[j];
    } else {
      blocks_ld(p, il, lane, ca);
    }
    double v[8];
    chunk_to_rows(sw, lane, cr, v);
    double2 ct[4];
    tile_precond_lap(v, s_tile, sw, lane, warp, ts, ct);
    if (warp < 4) {
      double2 ch[4];
      stage_wait();
      blocks_unstage(stg, sl, lane, ch);
#pragma unroll
      for (int j = 0; j < 4; j++) {
        ca[j].x = fma(-omega, ct[j].x, ca[j].x); // cuda.cu:524
        ca[j].y = fma(-omega, ct[j].y, ca[j].y);
        sums[0] = fma(ch[j].x, ca[j].x, sums[0]);
        sums[0] = fma(ch[j].y, ca[j].y, sums[0]);
        sums[1] = fma(ca[j].x, ca[j].x, sums[1]);
        sums[1] = fma(ca[j].y, ca[j].y, sums[1]);
        mx = fmax(mx, fmax(fabs(ca[j].x), fabs(ca[j].y)));
      }
      blocks_st(r, sl, lane, ca);
    } else {
      double2 cx[4];
      if (x_zero) {
#pragma unroll
        for (int j = 0; j < 4; j++) cx[j] = make_double2(0.0, 0.0);
      } else {
        blocks_ld(xc, il, lane, cx);
      }
      chunk_to_rows(sw, lane, ca, v);
      precond_row(v, sw, lane);
      rows_to_chunk(sw, lane, v, ca); // z_p
      const double2 *zr = reinterpret_cast<const double2 *>(s_tile.plane + ((warp - 4) * 8 + (lane >> 2) + 1) * PST) + (lane & 3);
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const double2 z = zr[4 * j]; // z_r of block j, piece `lane`
        cx[j].x = fma(omega, z.x, fma(alpha, ca[j].x, cx[j].x)); // cuda.cu:498 then 520
        cx[j].y = fma(omega, z.y, fma(alpha, ca[j].y, cx[j].y));
        sums[2] += cx[j].x + cx[j].y;
      }
      blocks_st(xn, il, lane, cx);
    }
    par ^= 1;
  }
  grid_reduce<3, NT>(sums, mx, partials, counter, comm, [=](const double *tsum, double m) {
    end_of_iteration(st, tsum, m, nxt);
    set_loop_condition(loop_handle, st);
  });
}

static inline int red_grid(const cup2d_sim *s, int nrows) {
  int g = (nrows + NT - 1) / NT;
  int cap = s->num_sms * 8;
  if (cap > RED_MAX_CTAS) cap = RED_MAX_CTAS;
  return g < cap ? g : cap;
}

static PushView make_push(const cup2d_sim *s, int peer_index) {
  PushView pv;
  pv.first = s->d_push_first;
  pv.ent = s->d_push_ent;
  for (int r = 0; r < MAX_RANKS; r++) pv.peer[r] = r < s->nranks ? (double *)s->peer_base[r][peer_index] : nullptr;
  pv.dst_mask = s->dst_mask;
  return pv;
}

// Start of a solve: Krylov state, r = b - A x0 (b = tmp, x0 = pres)
int poisson_begin(cup2d_sim *s, double tol_abs, double tol_rel, int max_restarts, int max_iter) {
  int rc = g_consts.run(s->device, upload_consts);
  if (rc) return rc;
  const int nrows = (int)s->nloc * 8;
  const int grid = red_grid(s, nrows);
  const int4 *nbr = reinterpret_cast<const int4 *>(s->d_nbr);
  const bool has_irr = s->n_irr_rows > 0; // general rows present: kernels with the CSR override compiled in
  k_state_init<<<1, 1, 0, s->stream>>>(s->d_state, tol_abs, tol_rel, max_restarts, max_iter);
  if (s->nranks > 1 && (rc = halo_exchange_ptr(s, s->f[CUP2D_PRES], 1, CUP2D_PRES))) return rc;
  {
    ProfScope prof(s, KC_KINIT);
    if (has_irr)
      k_init<true><<<grid, NT, 0, s->stream>>>(s->f[CUP2D_TMP], s->f[CUP2D_PRES], s->kx[0], s->kr, s->krhat, nbr,
                                               nrows, s->d_state, s->d_partials, s->d_counter,
                                               s->comm, irr_view(s), s->cond_handle);
    else
      k_init<false><<<grid, NT, 0, s->stream>>>(s->f[CUP2D_TMP], s->f[CUP2D_PRES], s->kx[0], s->kr, s->krhat, nbr,
                                                nrows, s->d_state, s->d_partials, s->d_counter,
                                                s->comm, irr_view(s), s->cond_handle);
  }
  s->launches += 2;
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

// Start of a time step's solve: Krylov state, then b from the step's right-hand side, r = rhat = b and x = 0 in one kernel
// (x0 = 0: no halo of it is needed).  pres is neither read nor written: the correction writes it.
int poisson_begin_rhs(cup2d_sim *s, double tol_abs, double tol_rel, int max_restarts, int max_iter, const StepRhs &rhs) {
  int rc = g_consts.run(s->device, upload_consts);
  if (rc) return rc;
  const int nrows = (int)s->nloc * 8;
  const int grid = red_grid(s, nrows);
  const int4 *nbr = reinterpret_cast<const int4 *>(s->d_nbr);
  k_state_init<<<1, 1, 0, s->stream>>>(s->d_state, tol_abs, tol_rel, max_restarts, max_iter);
  if ((rc = pressure_rhs_inputs(s, rhs.has_udef))) return rc;
  {
    ProfScope prof(s, KC_RHS_START);
    if (rhs.has_udef)
      pressure_rhs_start_kernel<true><<<grid, NT, 0, s->stream>>>(
          s->f[CUP2D_VEL], s->f[CUP2D_TMPV], s->f[CUP2D_CHI], s->f[CUP2D_POLD], s->kx[0], s->kr, s->krhat, nbr, nrows, rhs.dev,
          s->d_state, s->d_partials, s->d_counter, s->comm, s->cond_handle);
    else // no bodies: chi * div(udef) is identically zero (main.cpp:6980-6983 leaves tmpV = 0)
      pressure_rhs_start_kernel<false><<<grid, NT, 0, s->stream>>>(
          s->f[CUP2D_VEL], s->f[CUP2D_TMPV], s->f[CUP2D_CHI], s->f[CUP2D_POLD], s->kx[0], s->kr, s->krhat, nbr, nrows, rhs.dev,
          s->d_state, s->d_partials, s->d_counter, s->comm, s->cond_handle);
  }
  s->launches += 2;
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

// n BiCGSTAB iterations, no host involvement (a converged solve turns them into no-ops): 3 kernels each on a single-rank
// uniform grid; 5 with several ranks, general rows or no tiles (Poisson-only contexts)
int poisson_iterations(cup2d_sim *s, int n, cudaStream_t stream) {
  const int nrows = (int)s->nloc * 8;
  const int grid = red_grid(s, nrows);
  const int4 *nbr = reinterpret_cast<const int4 *>(s->d_nbr);
  const bool has_irr = s->n_irr_rows > 0;
  const bool multi = s->nranks > 1;
  if (!multi && !has_irr && !s->poisson_only) {
    // one wave of tile CTAs: the tiles in flight then form one compact region of the Hilbert order, whose ring blocks
    // are mostly read from L2
    const int tgrid = std::min(grid, s->num_sms * KTILE_CTAS), rgrid = std::min(grid, s->num_sms * KR_CTAS);
    for (int k = 0; k < n; k++) {
      {
        ProfScope prof(s, KC_P_SPMV);
        k_p_spmv<<<tgrid, NT, 0, stream>>>(s->kr, s->krhat, s->kp, s->kz, s->knu, s->kzr, s->d_tiles, s->ntiles, s->d_state,
                                           s->d_partials, s->d_counter, s->comm);
      }
      {
        ProfScope prof(s, KC_R_SPMV);
        k_r_spmv<<<rgrid, NT, 0, stream>>>(s->kr, s->knu, s->kzr, s->kt, s->d_tiles, s->ntiles, s->d_state, s->d_partials,
                                           s->d_counter, s->comm);
      }
      {
        ProfScope prof(s, KC_X_FINAL);
        k_x_final<<<tgrid, NT, 0, stream>>>(s->kx[0], s->kx[1], s->kx[2], s->kp, s->kz, s->kr, s->kt, s->krhat, s->d_tiles,
                                            s->ntiles, s->d_state, s->d_partials, s->d_counter, s->comm, s->cond_handle);
      }
      s->launches += 3;
    }
    CUP2D_CUDA(cudaGetLastError());
    return CUP2D_OK;
  }
  const PushView pz = make_push(s, CUP2D_NFIELDS), pzr = make_push(s, CUP2D_NFIELDS + 4);
  const IrrView irr = irr_view(s);
  for (int k = 0; k < n; k++) {
    {
      ProfScope prof(s, KC_PUPDATE);
      if (multi)
        k_pupdate<true><<<grid, NT, 0, stream>>>(s->kr, s->krhat, s->kp, s->knu, s->kz, nrows, s->d_state, pz, s->comm, s->d_counter);
      else
        k_pupdate<false><<<grid, NT, 0, stream>>>(s->kr, s->krhat, s->kp, s->knu, s->kz, nrows, s->d_state, pz, s->comm, s->d_counter);
    }
    {
      ProfScope prof(s, KC_SPMV_NU);
      if (has_irr && multi)
        k_spmv<0, true, true><<<grid, NT, 0, stream>>>(s->kz, s->krhat, s->knu, nbr, nrows, s->d_state, s->d_partials, s->d_counter, s->comm, irr, s->src_mask);
      else if (has_irr)
        k_spmv<0, true, false><<<grid, NT, 0, stream>>>(s->kz, s->krhat, s->knu, nbr, nrows, s->d_state, s->d_partials, s->d_counter, s->comm, irr, s->src_mask);
      else if (multi)
        k_spmv<0, false, true><<<grid, NT, 0, stream>>>(s->kz, s->krhat, s->knu, nbr, nrows, s->d_state, s->d_partials, s->d_counter, s->comm, irr, s->src_mask);
      else
        k_spmv<0, false, false><<<grid, NT, 0, stream>>>(s->kz, s->krhat, s->knu, nbr, nrows, s->d_state, s->d_partials, s->d_counter, s->comm, irr, s->src_mask);
    }
    {
      ProfScope prof(s, KC_XRUPDATE);
      if (multi)
        k_r_update<true><<<grid, NT, 0, stream>>>(s->kr, s->knu, s->kzr, nrows, s->d_state, pzr, s->comm, s->d_counter);
      else
        k_r_update<false><<<grid, NT, 0, stream>>>(s->kr, s->knu, s->kzr, nrows, s->d_state, pzr, s->comm, s->d_counter);
    }
    {
      ProfScope prof(s, KC_SPMV_T);
      if (has_irr && multi)
        k_spmv<1, true, true><<<grid, NT, 0, stream>>>(s->kzr, s->kr, s->kt, nbr, nrows, s->d_state, s->d_partials, s->d_counter, s->comm, irr, s->src_mask);
      else if (has_irr)
        k_spmv<1, true, false><<<grid, NT, 0, stream>>>(s->kzr, s->kr, s->kt, nbr, nrows, s->d_state, s->d_partials, s->d_counter, s->comm, irr, s->src_mask);
      else if (multi)
        k_spmv<1, false, true><<<grid, NT, 0, stream>>>(s->kzr, s->kr, s->kt, nbr, nrows, s->d_state, s->d_partials, s->d_counter, s->comm, irr, s->src_mask);
      else
        k_spmv<1, false, false><<<grid, NT, 0, stream>>>(s->kzr, s->kr, s->kt, nbr, nrows, s->d_state, s->d_partials, s->d_counter, s->comm, irr, s->src_mask);
    }
    {
      ProfScope prof(s, KC_FINAL);
      k_final<<<grid, NT, 0, stream>>>(s->kx[0], s->kx[1], s->kx[2], s->kz, s->kzr, s->kr, s->kt, s->krhat, nrows, s->d_state,
                                       s->d_partials, s->d_counter, s->comm, s->cond_handle);
    }
    s->launches += 5;
  }
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

// state of the last solve -> host (synchronises the stream); a cross-GPU wait that was given up surfaces here
int poisson_result(cup2d_sim *s, int *iters, double *err) {
  KrylovState *h = s->h_state;
  CUP2D_CUDA(cudaMemcpyAsync(h, s->d_state, sizeof *h, cudaMemcpyDeviceToHost, s->stream));
  CUP2D_CUDA(cudaStreamSynchronize(s->stream));
  if (iters) *iters = h->iter;
  if (err) *err = h->err_opt;
  return comm_check(s);
}

int poisson_solve(cup2d_sim *s, double tol_abs, double tol_rel, int max_restarts, int max_iter, int *iters, double *err) {
  int rc = poisson_begin(s, tol_abs, tol_rel, max_restarts, max_iter);
  if (rc) return rc;
  // fixed work (tolerances 0: the reference's first ten steps, main.cpp:7028-7030): everything is queued at once;
  // tolerance-driven: the host looks at the device's `done` flag every 8 iterations
  const int check_every = (tol_abs > 0 || tol_rel > 0) ? 8 : (max_iter > 0 ? max_iter : 1);
  int launched = 0;
  bool done = max_iter <= 0;
  while (!done) {
    const int batch = max_iter - launched < check_every ? max_iter - launched : check_every;
    if ((rc = poisson_iterations(s, batch, s->stream))) return rc;
    launched += batch;
    if ((rc = poisson_result(s, nullptr, nullptr))) return rc;
    done = s->h_state->done || launched >= max_iter;
  }
  return poisson_result(s, iters, err);
}

} // namespace cup2d
