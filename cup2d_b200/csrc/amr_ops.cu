// Stencil operators on multi-level (block-AMR) meshes — FIRST, CORRECTNESS-ORIENTED DEVICE PATH (SURVEY §8(f) rank 2).
//
// STATUS: checked on the GPU by tests/test_gpu_amr.py and on the CPU by the host emulation (tests/host_emu/).  See DESIGN.md
// 7.1 for the plan this is step 0 of.
//
// Shape (deliberately the simplest thing that can be compared with the reference, not the fast design):
//   1. lab = T . field : the ghost-stencil tables of the host plan (csrc/amr_plan.cpp) applied as a CSR gather into a
//      lab buffer in global memory (one lab per block: 14x14x2 for the advect stencil, 10x10x{2,1} for the +-1 stencils);
//   2. one thread per cell evaluates the operator from its block's lab, in the reference's own expression order
//      (KernelAdvectDiffuse main.cpp:5441-5503 with weno5_plus/minus main.cpp:162-208 in division form; pressure_rhs
//      main.cpp:6105-6139; pressure_rhs1 main.cpp:6209-6230; pressureCorrectionKernel main.cpp:6021-6043);
//   3. flux correction per coarse face (fillcases, main.cpp:1763-1849): the coarse block's own face flux plus the
//      pairwise sums of the two fine blocks' face fluxes, all recomputed from the labs, added to the coarse cells next to
//      the face — x faces first, then y faces, and for vector fields the second pass over the upper part of the face
//      that the reference's fillcase1 performs (DESIGN.md 7.1, property 3).  The pressure-gradient update is not
//      corrected (property 4).
#include "sim.h"
#include <algorithm>
#include <cmath>
#include <map>
#include <string>
#include <vector>

#include "amr.h"

namespace cup2d {

constexpr int LABN[4] = {14, 10, 10, 16}, LABD[4] = {2, 2, 1, 1}, LABG[4] = {3, 1, 1, 4}; // kind 3: chi lab of GradChiOnTmp

__global__ void amr_gather_kernel(Csr t, const double *__restrict__ field, double *__restrict__ lab, int dim) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < t.nrows; r += (int64_t)gridDim.x * blockDim.x) {
    double acc = 0.0;
    for (int64_t e = t.rowptr[r]; e < t.rowptr[r + 1]; e++)
      acc += t.w[e] * field[(int64_t)t.src_block[e] * 64 * dim + t.src_cc[e]];
    lab[r] = acc;
  }
}

// ---- WENO5 in the reference's own form (main.cpp:162-208) -----------------------------------------------------------
__device__ __forceinline__ void betas(double um2, double um1, double u, double up1, double up2, double &b1, double &b2,
                                      double &b3) {
  const double a1 = (um2 + u) - 2 * um1, c1 = (um2 + 3 * u) - 4 * um1;
  const double a2 = (um1 + up1) - 2 * u, c2 = um1 - up1;
  const double a3 = (u + up2) - 2 * up1, c3 = (3 * u + up2) - 4 * up1;
  b1 = 13.0 / 12.0 * (a1 * a1) + 0.25 * (c1 * c1);
  b2 = 13.0 / 12.0 * (a2 * a2) + 0.25 * (c2 * c2);
  b3 = 13.0 / 12.0 * (a3 * a3) + 0.25 * (c3 * c3);
}
__device__ __forceinline__ double weno_plus(double um2, double um1, double u, double up1, double up2) {
  const double e = 1e-6;
  double b1, b2, b3;
  betas(um2, um1, u, up1, up2, b1, b2, b3);
  const double w1 = 0.1 / ((b1 + e) * (b1 + e)), w2 = 0.6 / ((b2 + e) * (b2 + e)), w3 = 0.3 / ((b3 + e) * (b3 + e));
  const double aux = 1.0 / ((w1 + w3) + w2);
  const double f1 = (11.0 / 6.0) * u + ((1.0 / 3.0) * um2 - (7.0 / 6.0) * um1);
  const double f2 = (5.0 / 6.0) * u + ((-1.0 / 6.0) * um1 + (1.0 / 3.0) * up1);
  const double f3 = (1.0 / 3.0) * u + ((+5.0 / 6.0) * up1 - (1.0 / 6.0) * up2);
  return ((w1 * aux) * f1 + (w3 * aux) * f3) + (w2 * aux) * f2;
}
__device__ __forceinline__ double weno_minus(double um2, double um1, double u, double up1, double up2) {
  const double e = 1e-6;
  double b1, b2, b3;
  betas(um2, um1, u, up1, up2, b1, b2, b3);
  const double w1 = 0.3 / ((b1 + e) * (b1 + e)), w2 = 0.6 / ((b2 + e) * (b2 + e)), w3 = 0.1 / ((b3 + e) * (b3 + e));
  const double aux = 1.0 / ((w1 + w3) + w2);
  const double f1 = (1.0 / 3.0) * u + ((-1.0 / 6.0) * um2 + (5.0 / 6.0) * um1);
  const double f2 = (5.0 / 6.0) * u + ((1.0 / 3.0) * um1 - (1.0 / 6.0) * up1);
  const double f3 = (11.0 / 6.0) * u + ((-7.0 / 6.0) * up1 + (1.0 / 3.0) * up2);
  return ((w1 * aux) * f1 + (w3 * aux) * f3) + (w2 * aux) * f2;
}
__device__ __forceinline__ double derivative(double U, double um3, double um2, double um1, double u, double up1, double up2,
                                             double up3) {
  if (U > 0) return weno_plus(um2, um1, u, up1, up2) - weno_plus(um3, um2, um1, u, up1);
  return weno_minus(um1, u, up1, up2, up3) - weno_minus(um2, um1, u, up1, up2);
}

// lab accessors: L0 = 14x14x2 (ghost 3), L1 = 10x10x2 (ghost 1), L2 = 10x10 (ghost 1); (ix, iy) block-relative
__device__ __forceinline__ double L0(const double *lab, int64_t k, int ix, int iy, int c) {
  return lab[((k * 14 + (iy + 3)) * 14 + (ix + 3)) * 2 + c];
}
__device__ __forceinline__ double L1(const double *lab, int64_t k, int ix, int iy, int c) {
  return lab[((k * 10 + (iy + 1)) * 10 + (ix + 1)) * 2 + c];
}
__device__ __forceinline__ double L2(const double *lab, int64_t k, int ix, int iy) {
  return lab[(k * 10 + (iy + 1)) * 10 + (ix + 1)];
}

template <class DT>
__global__ void amr_advect_kernel(const double *__restrict__ lab, double *__restrict__ out, const double *__restrict__ hb,
                                  int64_t ncells, double nu, DT dt_arg) {
  const double dt = dt_arg.get();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < ncells; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t k = i >> 6;
    const int ix = (int)(i & 7), iy = (int)((i >> 3) & 7);
    const double h = hb[k], dfac = nu * dt, afac = -dt * h;
    auto U = [&](int dx, int dy) { return L0(lab, k, ix + dx, iy + dy, 0); };
    auto V = [&](int dx, int dy) { return L0(lab, k, ix + dx, iy + dy, 1); };
    const double u = U(0, 0), v = V(0, 0);
    const double dudx = derivative(u, U(-3, 0), U(-2, 0), U(-1, 0), u, U(1, 0), U(2, 0), U(3, 0));
    const double dudy = derivative(v, U(0, -3), U(0, -2), U(0, -1), u, U(0, 1), U(0, 2), U(0, 3));
    const double dvdx = derivative(u, V(-3, 0), V(-2, 0), V(-1, 0), v, V(1, 0), V(2, 0), V(3, 0));
    const double dvdy = derivative(v, V(0, -3), V(0, -2), V(0, -1), v, V(0, 1), V(0, 2), V(0, 3));
    out[2 * i] = afac * (u * dudx + v * dudy) + dfac * ((((U(1, 0) + U(-1, 0)) + U(0, 1)) + U(0, -1)) - 4 * u);
    out[2 * i + 1] = afac * (u * dvdx + v * dvdy) + dfac * ((((V(1, 0) + V(-1, 0)) + V(0, 1)) + V(0, -1)) - 4 * v);
  }
}

template <class DT>
__global__ void amr_div_kernel(const double *__restrict__ labv, const double *__restrict__ labu,
                               const double *__restrict__ chi, double *__restrict__ tmp, const double *__restrict__ hb,
                               int64_t ncells, DT dt_arg) {
  const double dt = dt_arg.get();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < ncells; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t k = i >> 6;
    const int ix = (int)(i & 7), iy = (int)((i >> 3) & 7);
    const double fac = 0.5 * hb[k] / dt;
    const double dv = ((L1(labv, k, ix + 1, iy, 0) - L1(labv, k, ix - 1, iy, 0)) + L1(labv, k, ix, iy + 1, 1)) - L1(labv, k, ix, iy - 1, 1);
    const double du = ((L1(labu, k, ix + 1, iy, 0) - L1(labu, k, ix - 1, iy, 0)) + L1(labu, k, ix, iy + 1, 1)) - L1(labu, k, ix, iy - 1, 1);
    tmp[i] = fac * dv - fac * chi[i] * du;
  }
}

__global__ void amr_lap_kernel(const double *__restrict__ labp, double *__restrict__ tmp, int64_t ncells) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < ncells; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t k = i >> 6;
    const int ix = (int)(i & 7), iy = (int)((i >> 3) & 7);
    tmp[i] -= (((L2(labp, k, ix - 1, iy) + L2(labp, k, ix + 1, iy)) + L2(labp, k, ix, iy - 1)) + L2(labp, k, ix, iy + 1)) -
              4 * L2(labp, k, ix, iy);
  }
}

template <class DT>
__global__ void amr_gradp_kernel(const double *__restrict__ labp, double *__restrict__ tmpv, const double *__restrict__ hb,
                                 int64_t ncells, DT dt_arg) {
  const double dt = dt_arg.get();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < ncells; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t k = i >> 6;
    const int ix = (int)(i & 7), iy = (int)((i >> 3) & 7);
    const double pfac = -0.5 * dt * hb[k];
    tmpv[2 * i] = pfac * (L2(labp, k, ix + 1, iy) - L2(labp, k, ix - 1, iy));
    tmpv[2 * i + 1] = pfac * (L2(labp, k, ix, iy + 1) - L2(labp, k, ix, iy - 1));
  }
}

// ---- the glue of a time step on a multi-level mesh (per-block cell size) --------------------------------------------
__global__ void amr_block_absmax_kernel(const double *__restrict__ vel, double *__restrict__ out, int64_t nb) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < nb; k += (int64_t)gridDim.x * blockDim.x) {
    double m = 0.0;
    for (int j = 0; j < 128; j++) m = fmax(m, fabs(vel[k * 128 + j]));
    out[k] = m;
  }
}
// adapt()'s tagging field (main.cpp:4676-4678).  KernelVorticity (3343-3366): tmp = (0.5/h) ((u_S - u_N) + v_E - v_W)
__global__ void amr_vorticity_kernel(const double *__restrict__ labv, double *__restrict__ tmp, const double *__restrict__ hb,
                                     int64_t ncells) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < ncells; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t k = i >> 6;
    const int ix = (int)(i & 7), iy = (int)((i >> 3) & 7);
    const double i2h = 0.5 / hb[k];
    tmp[i] = i2h * (((L1(labv, k, ix, iy - 1, 0) - L1(labv, k, ix, iy + 1, 0)) + L1(labv, k, ix + 1, iy, 1)) - L1(labv, k, ix - 1, iy, 1));
  }
}
// GradChiOnTmp (4631-4656): a block whose chi lab is positive anywhere within `offset` cells of it (4 on the finest level,
// 2 elsewhere; the clamp to [0,1] of 4645-4646 does not change the sign) gets 2 Rtol in its four centre cells; then the
// per-block L-inf that adapt() thresholds (4693-4697).  One thread per block.
__global__ void amr_tag_block_kernel(const double *__restrict__ labchi, double *__restrict__ tmp, const double *__restrict__ hb,
                                     double h_finest, double rtol, double *__restrict__ linf, int64_t nb) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < nb; k += (int64_t)gridDim.x * blockDim.x) {
    const int offset = hb[k] == h_finest ? 4 : 2;
    bool fire = false;
    for (int y = -offset; y < CUP2D_BS + offset && !fire; y++)
      for (int x = -offset; x < CUP2D_BS + offset; x++)
        if (labchi[(k * 16 + (y + 4)) * 16 + (x + 4)] > 0.0) {
          fire = true;
          break;
        }
    double *t = tmp + k * 64;
    if (fire) t[4 * 8 + 3] = t[3 * 8 + 3] = t[4 * 8 + 4] = t[3 * 8 + 4] = 2 * rtol;
    double m = 0.0;
    for (int j = 0; j < 64; j++) m = fmax(m, fabs(t[j]));
    linf[k] = m;
  }
}
// V = Vold + c * tmpV / h^2   (main.cpp:6618-6626, 6634-6642, 7180-7187 with Vold = V)
__global__ void amr_axpy_h2_kernel(double *__restrict__ v, const double *__restrict__ vold, const double *__restrict__ tmpv,
                                   const double *__restrict__ hb, int64_t n, double c) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const double h = hb[i >> 7], ih2 = c / (h * h);
    v[i] = vold[i] + tmpv[i] * ih2;
  }
}
// per block: sum(P * h^2) and 64 h^2 (main.cpp:7126-7135, 7150-7158); the host adds the blocks up in order
__global__ void amr_block_wsum_kernel(const double *__restrict__ p, const double *__restrict__ hb, double *__restrict__ out,
                                      int64_t nb) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < nb; k += (int64_t)gridDim.x * blockDim.x) {
    const double vv = hb[k] * hb[k];
    double a = 0.0, w = 0.0;
    for (int j = 0; j < 64; j++) {
      a += p[k * 64 + j] * vv;
      w += vv;
    }
    out[2 * k] = a;
    out[2 * k + 1] = w;
  }
}
// p[i] = (src ? src[i] : p[i]) + (add ? add[i] : 0) - shift
template <class S>
__global__ void amr_shift_kernel(double *__restrict__ p, const double *__restrict__ src, const double *__restrict__ add,
                                 int64_t n, S shift_arg) {
  const double shift = shift_arg.get();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    double v = src ? src[i] : p[i];
    if (add) v += add[i] - shift; else v += -shift;
    p[i] = v;
  }
}

// ---- face fluxes (what the kernels store in BlockCase::d[face]) -----------------------------------------------------
// position t along the face (0..7), face 0 = x-, 1 = x+, 2 = y-, 3 = y+; inner cell and the ghost behind the face
__device__ __forceinline__ void face_cells(int face, int t, int &ix, int &iy, int &gx, int &gy) {
  if (face < 2) {
    ix = face == 0 ? 0 : 7, iy = t, gx = face == 0 ? -1 : 8, gy = t;
  } else {
    ix = t, iy = face == 2 ? 0 : 7, gx = t, gy = face == 2 ? -1 : 8;
  }
}
// MODE 0: advect (dim 2, main.cpp:5515-5569)   1: pressure_rhs (dim 1, 6152-6205)   2: pressure_rhs1 (dim 1, 6243-6283)
template <int MODE>
__device__ __forceinline__ double face_flux(const double *labA, const double *labB, const double *chi, const double *hb,
                                            int64_t k, int face, int t, int comp, double nu, double dt) {
  int ix, iy, gx, gy;
  face_cells(face, t, ix, iy, gx, gy);
  if (MODE == 0) return (nu * dt) * (L0(labA, k, ix, iy, comp) - L0(labA, k, gx, gy, comp));
  if (MODE == 2) return L2(labA, k, gx, gy) - L2(labA, k, ix, iy);
  const double fac = 0.5 * hb[k] / dt;
  const int c = face < 2 ? 0 : 1;
  const double sv = L1(labA, k, gx, gy, c) + L1(labA, k, ix, iy, c), su = L1(labB, k, gx, gy, c) + L1(labB, k, ix, iy, c);
  const double x = chi[k * 64 + iy * 8 + ix];
  return (face & 1) == 0 ? fac * sv - (fac * x) * su : -fac * sv + (fac * x) * su;
}

// one thread per (coarse face, position t, comp): coarse cell += [own flux + (fine a + fine b)], twice where the reference does
template <int MODE, class DT>
__global__ void amr_fluxcorr_kernel(const CoarseFace *__restrict__ cf, int ncf, const double *labA, const double *labB,
                                    const double *chi, const double *hb, double *__restrict__ result, double nu,
                                    DT dt_arg) {
  constexpr int DIM = MODE == 0 ? 2 : 1;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ncf * 8 * DIM) return;
  const double dt = dt_arg.get();
  const int comp = i % DIM, t = (i / DIM) % 8;
  const CoarseFace f = cf[i / (8 * DIM)];
  double acc = face_flux<MODE>(labA, labB, chi, hb, f.coarse, f.face, t, comp, nu, dt);
  const int fb = f.fine[t >> 2];
  if (fb >= 0) { // the fine block abutting this half: its face is the opposite one; positions 2(t%4), 2(t%4)+1
    const int ff = f.face ^ 1, t2 = 2 * (t & 3);
    acc += face_flux<MODE>(labA, labB, chi, hb, fb, ff, t2, comp, nu, dt) + face_flux<MODE>(labA, labB, chi, hb, fb, ff, t2 + 1, comp, nu, dt);
  }
  int ix, iy, gx, gy;
  face_cells(f.face, t, ix, iy, gx, gy);
  double *dst = result + ((int64_t)f.coarse * 64 + iy * 8 + ix) * DIM + comp;
  double v = *dst + acc;
  // fillcase1 runs once per fine block and clears only entries [0, 8] of the 16 of a vector face in its first pass
  if (DIM == 2 && f.fine[0] >= 0 && f.fine[1] >= 0 && 2 * t + comp >= 9) v += acc;
  *dst = v;
}

static int grid_for(int64_t n) { return (int)std::min<int64_t>((n + 255) / 256, AMR_GRID_SMS * 16); }

static int upload_csr(cup2d_amr *a, int which) {
  const int64_t nnz = cup2d_amr_plan_stencil(a->plan, which, nullptr, nullptr, nullptr, nullptr);
  if (nnz < 0) return CUP2D_EINVAL;
  const int64_t per_block = LABN[which] * LABN[which] * LABD[which];
  const int64_t nrows = a->nb * per_block;
  std::vector<int64_t> rp(a->nglobal * per_block + 1);
  std::vector<int32_t> sb(nnz), sc(nnz);
  std::vector<double> w(nnz);
  cup2d_amr_plan_stencil(a->plan, which, rp.data(), sb.data(), sc.data(), w.data());
  // the rows of the context's blocks (contiguous: rows are in block order), sources renumbered to slots
  const int64_t r0 = a->gbegin * per_block, e0 = rp[r0], e1 = rp[r0 + nrows];
  for (int64_t e = e0; e < e1; e++) {
    sb[e] = a->slot(sb[e]);
    if (sb[e] < 0) {
      set_error("distributed context: a lab source lies outside the halo set");
      return CUP2D_EINVAL;
    }
  }
  rp.erase(rp.begin() + r0 + nrows + 1, rp.end());
  rp.erase(rp.begin(), rp.begin() + r0);
  for (auto &r : rp) r -= e0;
  auto keep = [&](auto &v) {
    v.erase(v.begin() + e1, v.end());
    v.erase(v.begin(), v.begin() + e0);
  };
  keep(sb);
  keep(sc);
  keep(w);
  Csr &c = a->csr[which];
  c.nrows = nrows;
  CUP2D_CUDA(upload(&c.rowptr, rp));
  CUP2D_CUDA(upload(&c.src_block, sb));
  CUP2D_CUDA(upload(&c.src_cc, sc));
  CUP2D_CUDA(upload(&c.w, w));
  CUP2D_CUDA(cudaMalloc(&a->lab[which], nrows * sizeof(double)));
  return CUP2D_OK;
}

// The full tables (every lab cell of every block) serve the baseline kernels only; they are built the first time one of
// those runs, so that a context driven through the fast kernels (compact tables: ghost rows of irregular blocks) never pays
// for them — they grow with the mesh, the compact ones with its level interfaces.
static int gather(cup2d_amr *a, int which, const double *field, double *&lab) {
  int rc;
  if (a->dist) {
    set_error("this operator runs on the table-gather baseline kernels, which a distributed context does not have");
    return CUP2D_ESTATE;
  }
  if (!a->csr[which].rowptr && (rc = upload_csr(a, which))) return rc;
  if (!lab) CUP2D_CUDA(cudaMalloc(&lab, a->csr[which].nrows * sizeof(double)));
  amr_gather_kernel<<<grid_for(a->csr[which].nrows), 256, 0, a->stream>>>(a->csr[which], field, lab, LABD[which]);
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

template <int MODE>
static int fluxcorr(cup2d_amr *a, const double *labA, const double *labB, double *result, double dt, const double *ddt = nullptr) {
  constexpr int DIM = MODE == 0 ? 2 : 1;
  for (int dir = 0; dir < 2; dir++) { // x faces, then y faces (fillcases order)
    const int n = a->ncf[dir] * 8 * DIM;
    if (n == 0) continue;
    with_scalar(dt, ddt, [&](auto d) {
      amr_fluxcorr_kernel<MODE><<<(n + 127) / 128, 128, 0, a->stream>>>(a->d_cf[dir], a->ncf[dir], labA, labB, a->f[CUP2D_CHI],
                                                                        a->d_h, result, a->nu, d);
      return 0;
    });
  }
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

// The cell size of every block the context holds (own blocks and halo slots, nslots in all), the smallest cell of the whole
// mesh (the time step's), the (i, j) of the own blocks, the per-block partials
static int block_sizes(cup2d_amr *a, const int32_t *level_ij, int64_t nslots) {
  std::vector<double> h(nslots, a->h0);
  a->hmin = a->h0;
  for (int64_t g = 0; g < a->nglobal; g++) {
    const double hg = a->h0 / (double)(1 << level_ij[3 * g]);
    a->hmin = std::min(a->hmin, hg);
    if (a->slot(g) >= 0) h[a->slot(g)] = hg;
  }
  const int32_t *own = level_ij + 3 * a->gbegin;
  a->h_ij.resize(2 * a->nb);
  for (int64_t k = 0; k < a->nb; k++) a->h_ij[2 * k] = own[3 * k + 1], a->h_ij[2 * k + 1] = own[3 * k + 2];
  a->h_part.resize(2 * a->nb);
  if (cudaMalloc(&a->d_part, 2 * a->nb * sizeof(double)) != cudaSuccess || upload(&a->d_h, h) != cudaSuccess) return CUP2D_ECUDA;
  return CUP2D_OK;
}

// The coarse faces of the context's blocks: the plan's (fine block, face, coarse block, face, half) records grouped by
// (coarse block, face), the fine side by slot (on a distributed context it may be a halo slot)
static int coarse_faces(cup2d_amr *a) {
  const std::vector<int32_t> rec = plan_faces(a);
  const int64_t b0 = a->gbegin, b1 = a->gbegin + a->nb;
  std::map<std::pair<int, int>, CoarseFace> byface;
  for (size_t r = 0; r < rec.size(); r += 5) {
    const int fine = rec[r], kc = rec[r + 2], fc = rec[r + 3], half = rec[r + 4];
    if (kc < b0 || kc >= b1) continue;
    auto it = byface.find({kc, fc});
    if (it == byface.end()) it = byface.emplace(std::make_pair(kc, fc), CoarseFace{(int)(kc - b0), fc, {-1, -1}}).first;
    if ((it->second.fine[half] = a->slot(fine)) < 0) return CUP2D_EINVAL;
  }
  std::vector<CoarseFace> lists[2];
  for (auto &e : byface) lists[e.second.face < 2 ? 0 : 1].push_back(e.second);
  for (int d = 0; d < 2; d++) {
    a->ncf[d] = (int)lists[d].size();
    if (!lists[d].empty()) CUP2D_CUDA(upload(&a->d_cf[d], lists[d]));
  }
  return CUP2D_OK;
}

} // namespace cup2d

using namespace cup2d;

#ifndef CUP2D_AMR_EMU
// the executable graphs of enqueued steps (an in-flight launch completes before its graph is freed)
static void amr_drop_graphs(cup2d_amr *a) {
  for (auto &g : a->graphs) {
    if (g.exec) cudaGraphExecDestroy((cudaGraphExec_t)g.exec);
    if (g.graph) cudaGraphDestroy((cudaGraph_t)g.graph);
  }
  a->graphs.clear();
}
#endif

#define CHECK_AMR(a)                                                                              \
  if (!(a)) {                                                                                     \
    cup2d::set_error("null cup2d_amr handle");                                                    \
    return CUP2D_EINVAL;                                                                          \
  }

extern "C" {

int cup2d_amr_create(int64_t nblocks, const int32_t *level_ij, int32_t bpdx, int32_t bpdy, double h0, double nu,
                     int32_t device, cup2d_amr **out) {
  if (!out || !level_ij || nblocks <= 0 || !(h0 > 0)) {
    set_error("cup2d_amr_create: bad arguments");
    return CUP2D_EINVAL;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    set_error("cup2d_amr_create: no CUDA device visible; this library has no CPU fallback");
    return CUP2D_ENOGPU;
  }
  if (device < 0 || device >= ndev) {
    set_error("cup2d_amr_create: bad device ordinal");
    return CUP2D_EINVAL;
  }
  cup2d_amr_plan *plan = nullptr;
  int rc = cup2d_amr_plan_create(nblocks, level_ij, bpdx, bpdy, &plan);
  if (rc) return rc;
  cup2d_amr *a = new cup2d_amr;
  a->plan = plan;
  a->nb = a->nglobal = nblocks;
  a->device = device;
  a->h0 = h0;
  a->nu = nu;
  auto fail = [&](int code) {
    cup2d_amr_destroy(a);
    return code;
  };
  if (cudaSetDevice(device) != cudaSuccess || cudaStreamCreate(&a->stream) != cudaSuccess) {
    set_error("cup2d_amr_create: cannot initialise the device");
    return fail(CUP2D_ECUDA);
  }
  for (int f = 0; f < CUP2D_NFIELDS; f++) {
    const size_t bytes = (size_t)nblocks * 64 * dim_of(f) * sizeof(double);
    if (cudaMalloc(&a->f[f], bytes) != cudaSuccess || cudaMemset(a->f[f], 0, bytes) != cudaSuccess) {
      set_error("cup2d_amr_create: out of device memory");
      return fail(CUP2D_ECUDA);
    }
  }
  // the baseline kernels' flux correction reads the coarse faces too: they are built here, not with the fast tables
  if ((rc = block_sizes(a, level_ij, nblocks)) || (rc = coarse_faces(a))) return fail(rc);
  *out = a;
  return CUP2D_OK;
}

void cup2d_amr_destroy(cup2d_amr *a) {
  if (!a) return;
  cudaSetDevice(a->device);
  if (!a->dist)
    for (auto p : a->f) cudaFree(p); // a distributed context borrows the field arrays (and the stream) of its Poisson context
  for (auto &c : a->csr) {
    cudaFree(c.rowptr); cudaFree(c.src_block); cudaFree(c.src_cc); cudaFree(c.w);
  }
  for (auto p : a->lab) cudaFree(p);
  cudaFree(a->lab_udef); cudaFree(a->d_h); cudaFree(a->d_cf[0]); cudaFree(a->d_cf[1]); cudaFree(a->d_part);
  cudaFree(a->d_nbr4); cudaFree(a->d_nbr8); cudaFree(a->d_irr_of); cudaFree(a->d_faceflux); cudaFree(a->d_vsum);
  a->free_shapes();
  auto free_ghosts = [](cup2d::GhostDev &g) {
    cudaFree(g.grow); cudaFree(g.rowptr); cudaFree(g.dst); cudaFree(g.sb); cudaFree(g.sc); cudaFree(g.w);
  };
  for (auto &g : a->gt) free_ghosts(g);
  for (auto &g : a->gt_src) free_ghosts(g);
#ifndef CUP2D_AMR_EMU
  amr_drop_graphs(a);
  if (a->ev_fork) cudaEventDestroy((cudaEvent_t)a->ev_fork);
  if (a->ev_join) cudaEventDestroy((cudaEvent_t)a->ev_join);
  if (a->poisson) cup2d_destroy(a->poisson);
#endif
  cudaFree(a->d_rec);
  if (a->stream && !a->dist) cudaStreamDestroy(a->stream);
  if (a->plan) cup2d_amr_plan_destroy(a->plan);
  delete a;
}

int cup2d_amr_field_upload(cup2d_amr *a, int field, const double *host) {
  CHECK_AMR(a);
  if (field < 0 || field >= CUP2D_NFIELDS || !host) return CUP2D_EINVAL;
  CUP2D_CUDA(cudaSetDevice(a->device));
  CUP2D_CUDA(cudaMemcpyAsync(a->f[field], host, (size_t)a->nb * 64 * dim_of(field) * sizeof(double), cudaMemcpyHostToDevice, a->stream));
  CUP2D_CUDA(cudaStreamSynchronize(a->stream));
  return CUP2D_OK;
}

int cup2d_amr_field_download(cup2d_amr *a, int field, double *host) {
  CHECK_AMR(a);
  if (field < 0 || field >= CUP2D_NFIELDS || !host) return CUP2D_EINVAL;
  CUP2D_CUDA(cudaSetDevice(a->device));
  CUP2D_CUDA(cudaMemcpyAsync(host, a->f[field], (size_t)a->nb * 64 * dim_of(field) * sizeof(double), cudaMemcpyDeviceToHost, a->stream));
  CUP2D_CUDA(cudaStreamSynchronize(a->stream));
  return CUP2D_OK;
}

} // extern "C"

// the dt-dependent operators, dt by value (ddt = nullptr: the blocking calls) or from the device record of an enqueued step
static int advect_rhs(cup2d_amr *a, double dt, const double *ddt) {
  if (a->fast) return amr_advect_rhs_fast(a, dt, ddt);
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc = gather(a, 0, a->f[CUP2D_VEL], a->lab[0]);
  if (rc) return rc;
  with_scalar(dt, ddt, [&](auto d) {
    amr_advect_kernel<<<grid_for(a->nb * 64), 256, 0, a->stream>>>(a->lab[0], a->f[CUP2D_TMPV], a->d_h, a->nb * 64, a->nu, d);
    return 0;
  });
  CUP2D_CUDA(cudaGetLastError());
  return fluxcorr<0>(a, a->lab[0], nullptr, a->f[CUP2D_TMPV], dt, ddt);
}

static int pressure_rhs(cup2d_amr *a, double dt, int with_laplacian, const double *ddt) {
  if (a->fast) return amr_pressure_rhs_fast(a, dt, with_laplacian, ddt);
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc = gather(a, 1, a->f[CUP2D_VEL], a->lab[1]);
  if (rc || (rc = gather(a, 1, a->f[CUP2D_TMPV], a->lab_udef))) return rc;
  with_scalar(dt, ddt, [&](auto d) {
    amr_div_kernel<<<grid_for(a->nb * 64), 256, 0, a->stream>>>(a->lab[1], a->lab_udef, a->f[CUP2D_CHI], a->f[CUP2D_TMP], a->d_h,
                                                               a->nb * 64, d);
    return 0;
  });
  CUP2D_CUDA(cudaGetLastError());
  if ((rc = fluxcorr<1>(a, a->lab[1], a->lab_udef, a->f[CUP2D_TMP], dt, ddt))) return rc;
  if (!with_laplacian) return CUP2D_OK;
  if ((rc = gather(a, 2, a->f[CUP2D_POLD], a->lab[2]))) return rc;
  amr_lap_kernel<<<grid_for(a->nb * 64), 256, 0, a->stream>>>(a->lab[2], a->f[CUP2D_TMP], a->nb * 64);
  CUP2D_CUDA(cudaGetLastError());
  return fluxcorr<2>(a, a->lab[2], nullptr, a->f[CUP2D_TMP], dt);
}

static int pressure_gradient(cup2d_amr *a, double dt, const double *ddt) {
  if (a->fast) return amr_pressure_gradient_fast(a, dt, ddt);
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc = gather(a, 2, a->f[CUP2D_PRES], a->lab[2]);
  if (rc) return rc;
  with_scalar(dt, ddt, [&](auto d) {
    amr_gradp_kernel<<<grid_for(a->nb * 64), 256, 0, a->stream>>>(a->lab[2], a->f[CUP2D_TMPV], a->d_h, a->nb * 64, d);
    return 0;
  });
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

extern "C" {

/* tmpV = KernelAdvectDiffuse(vel), flux-corrected (main.cpp:6611-6617) */
int cup2d_amr_advect_diffuse_rhs(cup2d_amr *a, double dt) {
  CHECK_AMR(a);
  return advect_rhs(a, dt, nullptr);
}

/* tmp = pressure_rhs(vel, u_def = tmpV, chi), flux-corrected (main.cpp:7007-7013); with_laplacian: then
 * tmp -= lap(pold), flux-corrected (main.cpp:7022-7027) */
int cup2d_amr_pressure_rhs(cup2d_amr *a, double dt, int with_laplacian) {
  CHECK_AMR(a);
  return pressure_rhs(a, dt, with_laplacian, nullptr);
}

/* tmpV = pressureCorrectionKernel(pres) (main.cpp:7174-7179; not flux-corrected in the reference either) */
int cup2d_amr_pressure_gradient(cup2d_amr *a, double dt) {
  CHECK_AMR(a);
  return pressure_gradient(a, dt, nullptr);
}

static int block_partials(cup2d_amr *a, int n_per_block) {
  CUP2D_CUDA(cudaMemcpyAsync(a->h_part.data(), a->d_part, (size_t)a->nb * n_per_block * sizeof(double), cudaMemcpyDeviceToHost,
                             a->stream));
  CUP2D_CUDA(cudaStreamSynchronize(a->stream));
  return CUP2D_OK;
}

/* adapt()'s per-block L-inf (main.cpp:4676-4697) on a multi-level mesh: vorticity of vel through the +-1 lab, the chi rule
 * of GradChiOnTmp through the {-4,-4,5,5,tensorial} chi lab; leaves the tagging field in tmp like the reference does.
 * level_max = sim.levelMax (the finest level is level_max - 1).  Fast contexts (distributed ones included) run the fused
 * kernel of amr_fast.cu on the compact tables; baseline-mode contexts gather both labs through the full per-cell tables
 * (built on first use).  Both give the same bits. */
int amr_adapt_tags_enqueue(cup2d_amr *a, double rtol, int level_max) {
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc;
  if ((rc = amr_dist_refresh(a, CUP2D_VEL)) || (rc = amr_dist_refresh(a, CUP2D_CHI))) return rc;
  const double h_finest = a->h0 / (double)(1 << (level_max - 1));
  if (a->fast) return amr_tags_fast(a, rtol, h_finest);
  if ((rc = gather(a, 1, a->f[CUP2D_VEL], a->lab[1])) || (rc = gather(a, 3, a->f[CUP2D_CHI], a->lab[3]))) return rc;
  amr_vorticity_kernel<<<grid_for(a->nb * 64), 256, 0, a->stream>>>(a->lab[1], a->f[CUP2D_TMP], a->d_h, a->nb * 64);
  amr_tag_block_kernel<<<grid_for(a->nb), 256, 0, a->stream>>>(a->lab[3], a->f[CUP2D_TMP], a->d_h, h_finest, rtol, a->d_part, a->nb);
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

int cup2d_amr_adapt_tags(cup2d_amr *a, double rtol, int level_max, double *block_linf_out) {
  CHECK_AMR(a);
  if (!block_linf_out || level_max < 1 || level_max > 30) {
    set_error("cup2d_amr_adapt_tags: bad arguments");
    return CUP2D_EINVAL;
  }
  int rc;
  if ((rc = amr_adapt_tags_enqueue(a, rtol, level_max)) || (rc = block_partials(a, 1))) return rc;
  memcpy(block_linf_out, a->h_part.data(), (size_t)a->nb * sizeof(double));
  return CUP2D_OK;
}

#ifndef CUP2D_AMR_EMU
// distributed contexts: two sums and one maximum over all ranks, by the one-warp peer all-reduce of the Krylov kernels
__global__ void amr_allreduce_kernel(double *v, Comm comm) {
  double tot[2] = {v[0], v[1]}, mx = v[2];
  peer_allreduce<2>(comm, tot, mx, threadIdx.x & 31);
  if (threadIdx.x == 0) v[0] = tot[0], v[1] = tot[1], v[2] = mx;
}
static int dist_allreduce(cup2d_amr *a, double &s0, double &s1, double &mx) {
  if (!a->dist || a->nranks == 1) return CUP2D_OK;
  cup2d_sim *ps = a->poisson;
  if (!ps->peers_attached) { // e.g. between a regrid onto new arrays and the re-attach
    set_error("distributed context: all-reduce before cup2d_amr_peer_attach");
    return CUP2D_ESTATE;
  }
  ps->h_scal[0] = s0, ps->h_scal[1] = s1, ps->h_scal[2] = mx;
  CUP2D_CUDA(cudaMemcpyAsync(ps->d_scal, ps->h_scal, 3 * sizeof(double), cudaMemcpyHostToDevice, a->stream));
  amr_allreduce_kernel<<<1, 32, 0, a->stream>>>(ps->d_scal, ps->comm);
  CUP2D_CUDA(cudaGetLastError());
  CUP2D_CUDA(cudaMemcpyAsync(ps->h_scal, ps->d_scal, 3 * sizeof(double), cudaMemcpyDeviceToHost, a->stream));
  CUP2D_CUDA(cudaStreamSynchronize(a->stream));
  s0 = ps->h_scal[0], s1 = ps->h_scal[1], mx = ps->h_scal[2];
  return CUP2D_OK;
}
int amr_dist_refresh(cup2d_amr *a, int field) { return a->dist ? cup2d_halo_exchange(a->poisson, field) : CUP2D_OK; }
int amr_dist_sum(cup2d_amr *a, double *v, int n) {
  for (int k = 0; k < n; k += 2) {
    double s0 = v[k], s1 = k + 1 < n ? v[k + 1] : 0.0, mx = 0.0;
    const int rc = dist_allreduce(a, s0, s1, mx);
    if (rc) return rc;
    v[k] = s0;
    if (k + 1 < n) v[k + 1] = s1;
  }
  return CUP2D_OK;
}

// v[0..n) summed over all ranks by one warp, seven values per peer all-reduce; v[n] = 0, or 1 if the ranks disagree on n.
// n goes round first (its sum and its maximum): every rank sees the same pair, so either all ranks add the values or all
// of them skip them, and a call made with different arguments on different ranks fails everywhere instead of mixing values.
constexpr int AMR_VSUM_CHUNK = 7;
__global__ void __launch_bounds__(32) amr_allreduce_vec_kernel(double *v, int n, Comm comm) {
  const int lane = threadIdx.x & 31;
  double cnt[1] = {(double)n}, cmax = (double)n;
  peer_allreduce<1>(comm, cnt, cmax, lane);
  if (cnt[0] != comm.nranks * cmax) {
    if (lane == 0) v[n] = 1.0;
    return;
  }
  for (int k0 = 0; k0 < n; k0 += AMR_VSUM_CHUNK) {
    double t[AMR_VSUM_CHUNK], m = 0.0;
#pragma unroll
    for (int q = 0; q < AMR_VSUM_CHUNK; q++) t[q] = k0 + q < n ? v[k0 + q] : 0.0;
    __syncwarp();
    peer_allreduce<AMR_VSUM_CHUNK>(comm, t, m, lane);
    if (lane == 0)
      for (int q = 0; q < AMR_VSUM_CHUNK && k0 + q < n; q++) v[k0 + q] = t[q];
    __syncwarp();
  }
  if (lane == 0) v[n] = 0.0;
}
int amr_dist_sum_vec(cup2d_amr *a, double *v, int n) {
  if (!a->dist || a->nranks == 1) return CUP2D_OK;
  if (!a->poisson->peers_attached) {
    set_error("distributed context: all-reduce before cup2d_amr_peer_attach");
    return CUP2D_ESTATE;
  }
  const size_t bytes = ((size_t)n + 1) * sizeof(double);
  if (bytes > a->vsum_cap) {
    cudaFree(a->d_vsum);
    a->d_vsum = nullptr, a->vsum_cap = 0;
    CUP2D_CUDA(cudaMalloc(&a->d_vsum, bytes));
    a->vsum_cap = bytes;
  }
  std::vector<double> h(n + 1);
  CUP2D_CUDA(cudaMemcpyAsync(a->d_vsum, v, (size_t)n * sizeof(double), cudaMemcpyHostToDevice, a->stream));
  amr_allreduce_vec_kernel<<<1, 32, 0, a->stream>>>(a->d_vsum, n, a->poisson->comm);
  CUP2D_CUDA(cudaGetLastError());
  CUP2D_CUDA(cudaMemcpyAsync(h.data(), a->d_vsum, bytes, cudaMemcpyDeviceToHost, a->stream));
  CUP2D_CUDA(cudaStreamSynchronize(a->stream));
  int rc = comm_check(a->poisson);
  if (rc) return rc;
  if (h[n] != 0.0) {
    set_error("distributed context: the ranks summed different numbers of values (the same call with different arguments)");
    return CUP2D_ECOMM;
  }
  std::copy(h.begin(), h.begin() + n, v);
  return CUP2D_OK;
}
#else
static int dist_allreduce(cup2d_amr *, double &, double &, double &) { return CUP2D_OK; }
int amr_dist_refresh(cup2d_amr *, int) { return CUP2D_OK; }
int amr_dist_sum(cup2d_amr *, double *, int) { return CUP2D_OK; }
int amr_dist_sum_vec(cup2d_amr *, double *, int) { return CUP2D_OK; }
#endif

/* main.cpp:6579-6595 with h = the smallest cell size of the mesh */
int cup2d_amr_compute_dt(cup2d_amr *a, double cfl, double *umax_out, double *dt_out) {
  CHECK_AMR(a);
  CUP2D_CUDA(cudaSetDevice(a->device));
  amr_block_absmax_kernel<<<grid_for(a->nb), 256, 0, a->stream>>>(a->f[CUP2D_VEL], a->d_part, a->nb);
  CUP2D_CUDA(cudaGetLastError());
  int rc = block_partials(a, 1);
  if (rc) return rc;
  double umax = 0, z0 = 0, z1 = 0;
  for (int64_t k = 0; k < a->nb; k++) umax = std::max(umax, a->h_part[k]);
  if ((rc = dist_allreduce(a, z0, z1, umax))) return rc;
  const double h = a->hmin;
  const double dt_diff = 0.25 * h * h / (a->nu + 0.25 * h * umax), dt_adv = h / (umax + 1e-8);
  if (umax_out) *umax_out = umax;
  if (dt_out) *dt_out = std::min(dt_diff, cfl * dt_adv);
  return CUP2D_OK;
}

} // extern "C"

static int rk2(cup2d_amr *a, double dt, const double *ddt) {
  CUP2D_CUDA(cudaSetDevice(a->device));
  const int64_t n = a->nb * 128;
  CUP2D_CUDA(cudaMemcpyAsync(a->f[CUP2D_VOLD], a->f[CUP2D_VEL], n * sizeof(double), cudaMemcpyDeviceToDevice, a->stream));
  for (int stage = 0; stage < 2; stage++) {
    int rc = advect_rhs(a, dt, ddt);
    if (rc) return rc;
    amr_axpy_h2_kernel<<<grid_for(n), 256, 0, a->stream>>>(a->f[CUP2D_VEL], a->f[CUP2D_VOLD], a->f[CUP2D_TMPV], a->d_h, n,
                                                          stage == 0 ? 0.5 : 1.0);
    CUP2D_CUDA(cudaGetLastError());
  }
  return CUP2D_OK;
}

static int poisson_rhs(cup2d_amr *a, double dt, const double *ddt) {
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc = pressure_rhs(a, dt, 0, ddt);
  if (rc) return rc;
  const size_t bytes = (size_t)a->nb * 64 * sizeof(double);
  CUP2D_CUDA(cudaMemcpyAsync(a->f[CUP2D_POLD], a->f[CUP2D_PRES], bytes, cudaMemcpyDeviceToDevice, a->stream));
  CUP2D_CUDA(cudaMemsetAsync(a->f[CUP2D_PRES], 0, bytes, a->stream));
  if (a->fast) return cup2d_amr_laplacian_fast(a, dt);
  if ((rc = gather(a, 2, a->f[CUP2D_POLD], a->lab[2]))) return rc;
  amr_lap_kernel<<<grid_for(a->nb * 64), 256, 0, a->stream>>>(a->lab[2], a->f[CUP2D_TMP], a->nb * 64);
  CUP2D_CUDA(cudaGetLastError());
  return fluxcorr<2>(a, a->lab[2], nullptr, a->f[CUP2D_TMP], dt);
}

extern "C" {

/* main.cpp:6607-6642: vold = vel; vel = vold + 0.5 K(vel)/h^2; vel = vold + K(vel)/h^2 (K flux-corrected) */
int cup2d_amr_advect_diffuse_rk2(cup2d_amr *a, double dt) {
  CHECK_AMR(a);
  return rk2(a, dt, nullptr);
}

/* main.cpp:7007-7027 as one call: tmp = pressure_rhs(vel, u_def = tmpV, chi); pold = pres; pres = 0; tmp -= lap(pold) */
int cup2d_amr_poisson_rhs(cup2d_amr *a, double dt) {
  CHECK_AMR(a);
  return poisson_rhs(a, dt, nullptr);
}

static int weighted_mean(cup2d_amr *a, const double *p, double *mean) {
  amr_block_wsum_kernel<<<grid_for(a->nb), 256, 0, a->stream>>>(p, a->d_h, a->d_part, a->nb);
  CUP2D_CUDA(cudaGetLastError());
  int rc = block_partials(a, 2);
  if (rc) return rc;
  double s = 0, w = 0, m0 = 0;
  for (int64_t k = 0; k < a->nb; k++) s += a->h_part[2 * k], w += a->h_part[2 * k + 1];
  if ((rc = dist_allreduce(a, s, w, m0))) return rc;
  *mean = s / w;
  return CUP2D_OK;
}

/* main.cpp:7120-7187 with the solution x of the Poisson solve in `pres`: pres = x - mean_h2(x); pres += pold - mean_h2(pres);
 * tmpV = pressureCorrectionKernel(pres); vel += tmpV / h^2 */
int cup2d_amr_pressure_correct(cup2d_amr *a, double dt) {
  CHECK_AMR(a);
  CUP2D_CUDA(cudaSetDevice(a->device));
  const int64_t n = a->nb * 64;
  double avg = 0;
  int rc = weighted_mean(a, a->f[CUP2D_PRES], &avg);
  if (rc) return rc;
  amr_shift_kernel<<<grid_for(n), 256, 0, a->stream>>>(a->f[CUP2D_PRES], nullptr, nullptr, n, ByValue{avg});
  if ((rc = weighted_mean(a, a->f[CUP2D_PRES], &avg))) return rc;
  amr_shift_kernel<<<grid_for(n), 256, 0, a->stream>>>(a->f[CUP2D_PRES], nullptr, a->f[CUP2D_POLD], n, ByValue{avg});
  CUP2D_CUDA(cudaGetLastError());
  if ((rc = cup2d_amr_pressure_gradient(a, dt))) return rc;
  amr_axpy_h2_kernel<<<grid_for(2 * n), 256, 0, a->stream>>>(a->f[CUP2D_VEL], a->f[CUP2D_VEL], a->f[CUP2D_TMPV], a->d_h, 2 * n, 1.0);
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

#ifndef CUP2D_AMR_EMU
/* Several GPUs, second form: the mesh is DISTRIBUTED — rank r holds the blocks rank_begin[r] .. rank_begin[r+1] of the list
 * (all ranks pass the same whole list) plus halo slots for every remote block its tables name, and computes only its own
 * blocks.  The field arrays are those of the distributed Poisson context (cup2d_poisson_create_general_ranks), so a halo
 * refresh is the whole-block peer pull of the uniform path (csrc/halo.cu) and the solve runs in place; the face fluxes of
 * fillcases travel the same way, stored per block in a field that is free at that point; dt and the pressure means are
 * all-reduced by the in-kernel peer all-reduce.  Fast kernels only.  Then cup2d_amr_peer_export / _attach; field upload and
 * download move this rank's blocks. */
// rank_begin[0..nranks] must be strictly increasing from 0 to nblocks (every rank owns blocks), and a field must keep
// its cell indices in 31 bits: checked before anything indexes by these ranges
static bool valid_partition(int64_t nblocks, int32_t nranks, const int64_t *rank_begin) {
  if (!rank_begin || nranks < 1 || nranks > MAX_RANKS || nblocks <= 0 || nblocks * 64 >= (1LL << 31)) return false;
  if (rank_begin[0] != 0 || rank_begin[nranks] != nblocks) return false;
  for (int r = 0; r < nranks; r++)
    if (rank_begin[r + 1] <= rank_begin[r]) return false;
  return true;
}

// The Poisson rows (cup2d_amr_plan_poisson) of the blocks [b0, b1) of the plan's list, as cup2d_poisson_create_general_ranks
// takes them: the blocks' face neighbours, their general rows numbered from the range's first cell, columns global.
// [0, nglobal) gives the plan's arrays unchanged.
struct PoissonRows {
  std::vector<int32_t> nbr, rows, rowptr, col;
  std::vector<double> val;
};
static int poisson_rows(cup2d_amr *a, int64_t b0, int64_t b1, PoissonRows &q) {
  int64_t nnz = 0;
  const int64_t nr = cup2d_amr_plan_poisson(a->plan, nullptr, &nnz, nullptr, nullptr, nullptr, nullptr);
  if (nr < 0) return (int)nr;
  q.nbr.resize(4 * a->nglobal), q.rows.resize(nr), q.rowptr.resize(nr + 1), q.col.resize(nnz), q.val.resize(nnz);
  cup2d_amr_plan_poisson(a->plan, q.nbr.data(), &nnz, q.rows.data(), q.rowptr.data(), q.col.data(), q.val.data());
  const int64_t k0 = std::lower_bound(q.rows.begin(), q.rows.end(), (int32_t)(64 * b0)) - q.rows.begin();
  const int64_t k1 = std::lower_bound(q.rows.begin(), q.rows.end(), (int32_t)(64 * b1)) - q.rows.begin();
  const int32_t e0 = q.rowptr[k0], e1 = q.rowptr[k1];
  auto keep = [](auto &v, int64_t i0, int64_t i1) {
    v.erase(v.begin() + i1, v.end());
    v.erase(v.begin(), v.begin() + i0);
  };
  keep(q.nbr, 4 * b0, 4 * b1), keep(q.rows, k0, k1), keep(q.rowptr, k0, k1 + 1), keep(q.col, e0, e1), keep(q.val, e0, e1);
  for (auto &r : q.rows) r -= (int32_t)(64 * b0);
  for (auto &e : q.rowptr) e -= e0;
  return CUP2D_OK;
}

int cup2d_amr_create_ranks(int64_t nblocks, const int32_t *level_ij, int32_t bpdx, int32_t bpdy, double h0, double nu, int32_t rank,
                           int32_t nranks, const int64_t *rank_begin, int32_t device, cup2d_amr **out) {
  if (!out || !level_ij || !(h0 > 0) || rank < 0 || rank >= nranks || !valid_partition(nblocks, nranks, rank_begin)) {
    set_error("cup2d_amr_create_ranks: bad arguments (rank_begin must increase strictly from 0 to nblocks, 1..8 ranks, fewer than 2^31 cells)");
    return CUP2D_EINVAL;
  }
  cup2d_amr_plan *plan = nullptr;
  int rc = cup2d_amr_plan_create(nblocks, level_ij, bpdx, bpdy, &plan);
  if (rc) return rc;
  cup2d_amr *a = new cup2d_amr;
  a->plan = plan;
  a->device = device;
  a->h0 = h0;
  a->nu = nu;
  a->dist = a->fast = true;
  a->rank = rank;
  a->nranks = nranks;
  a->rank_begin.assign(rank_begin, rank_begin + nranks + 1);
  auto fail = [&](int code) {
    cup2d_amr_destroy(a);
    return code;
  };
  const int64_t b0 = rank_begin[rank], b1 = rank_begin[rank + 1], nloc = b1 - b0;
  a->nb = nloc;
  a->gbegin = b0;
  a->nglobal = nblocks;
  // every remote block the stencil tables of this rank name: face neighbours, sources of its ghost rows, fine sides of its
  // coarse faces (the Poisson rows add theirs inside the constructor below)
  std::vector<int32_t> extra, n8;
  if ((rc = plan_neighbours(a, n8))) return fail(rc);
  for (int64_t k = b0; k < b1; k++)
    for (int j = 0; j < 8; j++)
      if (n8[8 * k + j] >= 0) extra.push_back(n8[8 * k + j]);
  const std::vector<int32_t> irr = plan_irregular(a);
  for (int which : {0, 1, 2, 3, 6}) { // 3: the chi lab of the tagging rule and of the forces, 6: the forces' velocity lab
    PlanGhosts g;
    if ((rc = plan_ghosts(a, which, g))) return fail(rc);
    for (size_t row = 0; row < g.dst.size(); row++) {
      const int32_t blk = irr[g.dst[row] / GHOST_NCELL[which]];
      if (blk < b0 || blk >= b1) continue;
      for (int64_t e = g.rowptr[row]; e < g.rowptr[row + 1]; e++) extra.push_back(g.sb[e]);
    }
  }
  const std::vector<int32_t> rec = plan_faces(a);
  for (size_t r = 0; r < rec.size(); r += 5)
    if (rec[r + 2] >= b0 && rec[r + 2] < b1) extra.push_back(rec[r]);
  PoissonRows q; // this rank's rows of the Poisson matrix (as cup2d_amr_set_ranks)
  if ((rc = poisson_rows(a, b0, b1, q))) return fail(rc);
  if ((rc = poisson_create_general_ranks_ex(nblocks, rank, nranks, rank_begin, q.nbr.data(), (int64_t)q.rows.size(), q.rows.data(),
                                            q.rowptr.data(), q.col.data(), q.val.data(), (int64_t)extra.size(), extra.data(),
                                            device, &a->poisson)))
    return fail(rc);
  cup2d_sim *ps = a->poisson;
  a->stream = ps->stream;
  for (int f = 0; f < CUP2D_NFIELDS; f++) a->f[f] = ps->f[f];
  a->slot_of.assign(nblocks, -1);
  for (int64_t k = 0; k < nloc; k++) a->slot_of[b0 + k] = (int32_t)k;
  for (int64_t k = 0; k < ps->nhalo; k++) a->slot_of[ps->halo_gid[k]] = (int32_t)(nloc + k);
  if ((rc = block_sizes(a, level_ij, ps->nslots)) || (rc = coarse_faces(a)) || (rc = amr_fast_build(a))) return fail(rc);
  *out = a;
  return CUP2D_OK;
}

/* Several GPUs, first form: every rank holds the whole mesh and computes the stencil operators redundantly (bitwise the same
 * everywhere), the Poisson solve — the part that dominates a step — is distributed over the ranks by block ranges
 * (cup2d_poisson_create_general_ranks) and its result all-gathered over NVLink.  rank_begin[nranks+1] partitions the block
 * list.  Then cup2d_amr_peer_export / cup2d_amr_peer_attach like the cup2d_peer_* pair. */
int cup2d_amr_set_ranks(cup2d_amr *a, int32_t rank, int32_t nranks, const int64_t *rank_begin) {
  CHECK_AMR(a);
  if (a->poisson || rank < 0 || rank >= nranks || !valid_partition(a->nb, nranks, rank_begin)) {
    set_error("cup2d_amr_set_ranks: bad arguments (rank_begin must increase strictly from 0 to the block count) or called after the first solve");
    return CUP2D_EINVAL;
  }
  CUP2D_CUDA(cudaSetDevice(a->device));
  PoissonRows q;
  int rc = poisson_rows(a, rank_begin[rank], rank_begin[rank + 1], q);
  if (rc || (rc = cup2d_poisson_create_general_ranks(a->nb, rank, nranks, rank_begin, q.nbr.data(), (int64_t)q.rows.size(), q.rows.data(),
                                                     q.rowptr.data(), q.col.data(), q.val.data(), a->device, &a->poisson)))
    return rc;
  a->rank = rank;
  a->nranks = nranks;
  a->rank_begin.assign(rank_begin, rank_begin + nranks + 1);
  return CUP2D_OK;
}
int cup2d_amr_peer_export(cup2d_amr *a, void *blob) {
  CHECK_AMR(a);
  if (!a->poisson) {
    set_error("cup2d_amr_peer_export: call cup2d_amr_set_ranks first");
    return CUP2D_ESTATE;
  }
  return cup2d_peer_export(a->poisson, blob);
}
int cup2d_amr_peer_attach(cup2d_amr *a, const void *all_blobs) {
  CHECK_AMR(a);
  if (!a->poisson) {
    set_error("cup2d_amr_peer_attach: call cup2d_amr_set_ranks first");
    return CUP2D_ESTATE;
  }
  amr_drop_graphs(a); // their halo pulls and all-reduces hold the peer pointers of the previous attach
  return cup2d_peer_attach(a->poisson, all_blobs);
}

static int poisson_solve_distributed(cup2d_amr *a, double tol_abs, double tol_rel, int max_restarts, int max_iter, int *iters,
                                     double *err) {
  const int64_t b0 = a->rank_begin[a->rank], nloc = a->rank_begin[a->rank + 1] - b0;
  const size_t bytes = (size_t)nloc * 64 * sizeof(double);
  CUP2D_CUDA(cudaStreamSynchronize(a->stream));
  cudaStream_t ps = (cudaStream_t)cup2d_stream(a->poisson);
  // this rank's rows of the right-hand side and of the initial guess (every rank computed the whole of both)
  CUP2D_CUDA(cudaMemcpyAsync(cup2d_field_device_ptr(a->poisson, CUP2D_TMP), a->f[CUP2D_TMP] + b0 * 64, bytes, cudaMemcpyDeviceToDevice, ps));
  CUP2D_CUDA(cudaMemcpyAsync(cup2d_field_device_ptr(a->poisson, CUP2D_PRES), a->f[CUP2D_PRES] + b0 * 64, bytes, cudaMemcpyDeviceToDevice, ps));
  int rc = cup2d_poisson_solve(a->poisson, tol_abs, tol_rel, max_restarts, max_iter, iters, err);
  // all-gather of the solution: a halo refresh is a barrier (every rank's pressure is final when it returns), then every
  // rank copies the others' rows straight out of their arrays over NVLink; a second barrier before anyone overwrites them
  if (rc || (rc = cup2d_halo_exchange(a->poisson, CUP2D_PRES))) return rc;
  for (int r = 0; r < a->nranks; r++) {
    const double *src = static_cast<const double *>(cup2d_peer_field_ptr(a->poisson, r, CUP2D_PRES));
    if (!src) {
      set_error("cup2d_amr_poisson_solve: peers not attached");
      return CUP2D_ESTATE;
    }
    CUP2D_CUDA(cudaMemcpyAsync(a->f[CUP2D_PRES] + a->rank_begin[r] * 64, src, (size_t)(a->rank_begin[r + 1] - a->rank_begin[r]) * 64 * sizeof(double),
                               cudaMemcpyDeviceToDevice, ps));
  }
  if ((rc = cup2d_halo_exchange(a->poisson, CUP2D_PRES))) return rc;
  CUP2D_CUDA(cudaStreamSynchronize(ps));
  return CUP2D_OK;
}

/* the Poisson solve of the step: b = tmp, x0 = pres -> pres, on the general-rows solver (csrc/poisson.cu) with the
 * rows of cup2d_amr_plan_poisson; same stopping parameters as cup2d_poisson_solve */
// the general-rows Poisson context over the blocks of the mesh, created on first use
static int ensure_poisson(cup2d_amr *a) {
  if (a->poisson) return CUP2D_OK;
  PoissonRows q;
  const int rc = poisson_rows(a, 0, a->nb, q);
  if (rc) return rc;
  return cup2d_poisson_create_general(a->nb, q.nbr.data(), (int64_t)q.rows.size(), q.rows.data(), q.rowptr.data(), q.col.data(),
                                      q.val.data(), a->device, &a->poisson);
}

int cup2d_amr_poisson_solve(cup2d_amr *a, double tol_abs, double tol_rel, int max_restarts, int max_iter, int *iters,
                            double *err) {
  CHECK_AMR(a);
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc;
  if ((rc = ensure_poisson(a))) return rc;
  if (a->dist) { // the fields ARE the Poisson context's: b = tmp and x0 = pres are in place, so is the result
    CUP2D_CUDA(cudaSetDevice(a->device));
    return cup2d_poisson_solve(a->poisson, tol_abs, tol_rel, max_restarts, max_iter, iters, err);
  }
  if (a->nranks > 1) return poisson_solve_distributed(a, tol_abs, tol_rel, max_restarts, max_iter, iters, err);
  const size_t bytes = (size_t)a->nb * 64 * sizeof(double);
  CUP2D_CUDA(cudaStreamSynchronize(a->stream));
  cudaStream_t ps = (cudaStream_t)cup2d_stream(a->poisson);
  CUP2D_CUDA(cudaMemcpyAsync(cup2d_field_device_ptr(a->poisson, CUP2D_TMP), a->f[CUP2D_TMP], bytes, cudaMemcpyDeviceToDevice, ps));
  CUP2D_CUDA(cudaMemcpyAsync(cup2d_field_device_ptr(a->poisson, CUP2D_PRES), a->f[CUP2D_PRES], bytes, cudaMemcpyDeviceToDevice, ps));
  if ((rc = cup2d_poisson_solve(a->poisson, tol_abs, tol_rel, max_restarts, max_iter, iters, err))) return rc;
  CUP2D_CUDA(cudaMemcpyAsync(a->f[CUP2D_PRES], cup2d_field_device_ptr(a->poisson, CUP2D_PRES), bytes, cudaMemcpyDeviceToDevice, ps));
  CUP2D_CUDA(cudaStreamSynchronize(ps));
  return CUP2D_OK;
}

/* one time step without bodies (main.cpp:6576-7187 minus the OUT-of-scope parts) on a multi-level mesh */
int cup2d_amr_step(cup2d_amr *a, double cfl, double dt_in, double tol_abs, double tol_rel, int max_restarts, int max_iter,
                   double *dt_out, int *iters, double *err) {
  CHECK_AMR(a);
  double dt = dt_in, umax = 0;
  int rc;
  if (!(dt > 0) && (rc = cup2d_amr_compute_dt(a, cfl, &umax, &dt))) return rc;
  if ((rc = cup2d_amr_advect_diffuse_rk2(a, dt))) return rc;
  CUP2D_CUDA(cudaMemsetAsync(a->f[CUP2D_TMPV], 0, (size_t)a->nb * 128 * sizeof(double), a->stream)); // no bodies: u_def = 0
  if ((rc = cup2d_amr_poisson_rhs(a, dt))) return rc;
  if ((rc = cup2d_amr_poisson_solve(a, tol_abs, tol_rel, max_restarts, max_iter, iters, err))) return rc;
  if ((rc = cup2d_amr_pressure_correct(a, dt))) return rc;
  if (dt_out) *dt_out = dt;
  return CUP2D_OK;
}

} // extern "C"

// ---- time steps enqueued without host synchronisation (cup2d_amr_step_enqueue / _pressure_enqueue) --------------------
// The blocking calls above wait on the host for dt (per-block maxima), for the two pressure means (per-block sums) and for
// the Krylov solve.  Here dt lives in the device record a->d_rec and every dt-dependent kernel reads it from there
// (OnDevice), the means are reduced on the device into the same record, and the solve is enqueued on the Poisson context's
// stream, joined to this one by events: nothing in the body depends on a host value that changes from step to step, so it
// is captured once per argument set into a CUDA graph and replayed with one cudaGraphLaunch.  A distributed context
// (cup2d_amr_create_ranks) runs the same body on its Poisson context's stream and arrays: the solve in place, the halo
// refreshes as stream-ordered peer pulls, dt's maximum and the means all-reduced by warp 0 of the one-CTA reductions.
namespace cup2d {

constexpr int AMR_RED_NT = 1024; // one CTA reduces the per-block partials of the whole mesh

// dt given by value: written by a kernel ahead of the graph launch, so that the graph does not hold it
__global__ void amr_set_dt_kernel(double *rec, double dt) { rec[AMR_REC_DT] = dt; }

// the dt rule of cup2d_amr_compute_dt: the largest per-block maximum (a maximum is exact in any order), on a distributed
// context all-reduced over the ranks by warp 0 (peer_allreduce returns at once on one rank), then main.cpp:6593-6595 in the
// host code's operation order with explicit round-to-nearest operations (no FMA contraction): bitwise the host's dt
__global__ void __launch_bounds__(AMR_RED_NT) amr_dt_kernel(const double *__restrict__ part, int64_t nb, double h, double nu,
                                                            double cfl, double *rec, Comm comm) {
  __shared__ double sm[AMR_RED_NT];
  double m = 0.0;
  for (int64_t k = threadIdx.x; k < nb; k += AMR_RED_NT) m = fmax(m, part[k]);
  sm[threadIdx.x] = m;
  __syncthreads();
  for (int s = AMR_RED_NT / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) sm[threadIdx.x] = fmax(sm[threadIdx.x], sm[threadIdx.x + s]);
    __syncthreads();
  }
  if (threadIdx.x >= 32) return;
  double umax = sm[0], none[1] = {0.0};
  peer_allreduce<1>(comm, none, umax, threadIdx.x);
  if (threadIdx.x == 0) {
    const double dt_diff = __ddiv_rn(__dmul_rn(__dmul_rn(0.25, h), h), __dadd_rn(nu, __dmul_rn(__dmul_rn(0.25, h), umax)));
    const double dt_adv = __ddiv_rn(h, __dadd_rn(umax, 1e-8));
    const double c = __dmul_rn(cfl, dt_adv);
    rec[AMR_REC_DT] = c < dt_diff ? c : dt_diff; // std::min(dt_diff, c)
  }
}

// sum(P h^2) / sum(h^2) over the per-block pairs of amr_block_wsum_kernel in a FIXED order, so that a step gives the same bits
// every time: thread t adds the blocks t, t + NT, t + 2 NT, ... in block order, then the NT partial sums are combined by a
// binary tree (s[t] += s[t + m] for m = NT/2, ..., 1).  On a distributed context warp 0 then all-reduces the rank's pair
// (sum P h^2, sum h^2), the ranks' pairs added in rank order, so every rank divides the same bits (one rank: no-op).  The
// blocking path adds the blocks in one serial chain on the host; the two orders agree to rounding.
__global__ void __launch_bounds__(AMR_RED_NT) amr_wmean_kernel(const double *__restrict__ part, int64_t nb, double *mean,
                                                               Comm comm) {
  __shared__ double ss[AMR_RED_NT];
  __shared__ double sw[AMR_RED_NT];
  const double2 *p2 = reinterpret_cast<const double2 *>(part);
  double s = 0.0, w = 0.0;
  for (int64_t k0 = threadIdx.x; k0 < nb; k0 += 4 * AMR_RED_NT) { // four loads in flight per thread, added in block order
    double2 v[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const int64_t k = k0 + (int64_t)u * AMR_RED_NT;
      v[u] = k < nb ? p2[k] : double2{0.0, 0.0};
    }
#pragma unroll
    for (int u = 0; u < 4; u++) s += v[u].x, w += v[u].y;
  }
  ss[threadIdx.x] = s;
  sw[threadIdx.x] = w;
  __syncthreads();
  for (int m = AMR_RED_NT / 2; m > 0; m >>= 1) {
    if ((int)threadIdx.x < m) ss[threadIdx.x] += ss[threadIdx.x + m], sw[threadIdx.x] += sw[threadIdx.x + m];
    __syncthreads();
  }
  if (threadIdx.x >= 32) return;
  double sum[2] = {ss[0], sw[0]}, none = 0.0;
  peer_allreduce<2>(comm, sum, none, threadIdx.x);
  if (threadIdx.x == 0) *mean = sum[0] / sum[1];
}

// dst = the Krylov iterate the solve returns (KrylovState::opt, chosen on the device)
__global__ void amr_take_x_kernel(double *__restrict__ dst, const double *x0, const double *x1, const double *x2,
                                  const KrylovState *__restrict__ st, int64_t n) {
  const int o = st->opt;
  const double *__restrict__ src = o == 0 ? x0 : o == 1 ? x1 : x2;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) dst[i] = src[i];
}

} // namespace cup2d

// cup2d_amr_pressure_correct with dt and both means from the device record
static int pressure_correct_enqueued(cup2d_amr *a) {
  const int64_t n = a->nb * 64;
  for (int pass = 0; pass < 2; pass++) { // pres -= mean_h2(pres); then pres += pold - mean_h2(pres)
    double *mean = a->d_rec + AMR_REC_MEAN0 + pass;
    amr_block_wsum_kernel<<<grid_for(a->nb), 256, 0, a->stream>>>(a->f[CUP2D_PRES], a->d_h, a->d_part, a->nb);
    amr_wmean_kernel<<<1, AMR_RED_NT, 0, a->stream>>>(a->d_part, a->nb, mean, a->poisson->comm);
    amr_shift_kernel<<<grid_for(n), 256, 0, a->stream>>>(a->f[CUP2D_PRES], nullptr, pass ? a->f[CUP2D_POLD] : nullptr, n,
                                                         OnDevice{mean});
    CUP2D_CUDA(cudaGetLastError());
  }
  int rc = pressure_gradient(a, 0.0, a->d_rec + AMR_REC_DT);
  if (rc) return rc;
  amr_axpy_h2_kernel<<<grid_for(2 * n), 256, 0, a->stream>>>(a->f[CUP2D_VEL], a->f[CUP2D_VEL], a->f[CUP2D_TMPV], a->d_h, 2 * n, 1.0);
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

// the body of an enqueued step (pressure_only = false: cup2d_amr_step without bodies) or pressure section
static int enqueue_body(cup2d_amr *a, bool pressure_only, bool dev_dt, double cfl, double tol_abs, double tol_rel,
                        int max_restarts, int max_iter, bool capturing) {
  const double *ddt = a->d_rec + AMR_REC_DT;
  const int64_t n = a->nb * 64;
  int rc;
  if (!pressure_only) {
    if (dev_dt) {
      amr_block_absmax_kernel<<<grid_for(a->nb), 256, 0, a->stream>>>(a->f[CUP2D_VEL], a->d_part, a->nb);
      amr_dt_kernel<<<1, AMR_RED_NT, 0, a->stream>>>(a->d_part, a->nb, a->hmin, a->nu, cfl, a->d_rec, a->poisson->comm);
      CUP2D_CUDA(cudaGetLastError());
    }
    if ((rc = rk2(a, 0.0, ddt))) return rc;
    CUP2D_CUDA(cudaMemsetAsync(a->f[CUP2D_TMPV], 0, (size_t)n * 2 * sizeof(double), a->stream)); // no bodies: u_def = 0
  }
  if ((rc = poisson_rhs(a, 0.0, ddt))) return rc;
  cup2d_sim *ps = a->poisson;
  if (a->dist) { // stream and fields are the Poisson context's: b = tmp and x0 = pres in place, as the blocking solve
    if ((rc = poisson_enqueue(ps, tol_abs, tol_rel, max_restarts, max_iter, capturing))) return rc;
    // this rank's blocks; the pressure gradient refreshes the halo slots of pres itself
    amr_take_x_kernel<<<grid_for(n), 256, 0, a->stream>>>(a->f[CUP2D_PRES], ps->kx[0], ps->kx[1], ps->kx[2], ps->d_state, n);
    CUP2D_CUDA(cudaGetLastError());
    return pressure_correct_enqueued(a);
  }
  // b = tmp, x0 = pres into the Poisson context, on its stream after this one's work (the event also pulls that stream
  // into a capture of this one); the iterate comes back after the solve's last kernel
  CUP2D_CUDA(cudaEventRecord((cudaEvent_t)a->ev_fork, a->stream));
  CUP2D_CUDA(cudaStreamWaitEvent(ps->stream, (cudaEvent_t)a->ev_fork, 0));
  CUP2D_CUDA(cudaMemcpyAsync(ps->f[CUP2D_TMP], a->f[CUP2D_TMP], n * sizeof(double), cudaMemcpyDeviceToDevice, ps->stream));
  CUP2D_CUDA(cudaMemcpyAsync(ps->f[CUP2D_PRES], a->f[CUP2D_PRES], n * sizeof(double), cudaMemcpyDeviceToDevice, ps->stream));
  if ((rc = poisson_enqueue(ps, tol_abs, tol_rel, max_restarts, max_iter, capturing))) return rc;
  CUP2D_CUDA(cudaEventRecord((cudaEvent_t)a->ev_join, ps->stream));
  CUP2D_CUDA(cudaStreamWaitEvent(a->stream, (cudaEvent_t)a->ev_join, 0));
  amr_take_x_kernel<<<grid_for(n), 256, 0, a->stream>>>(a->f[CUP2D_PRES], ps->kx[0], ps->kx[1], ps->kx[2], ps->d_state, n);
  CUP2D_CUDA(cudaGetLastError());
  return pressure_correct_enqueued(a);
}

static int amr_enqueue(cup2d_amr *a, const char *who, bool pressure_only, double cfl, double dt_in, double tol_abs,
                       double tol_rel, int max_restarts, int max_iter) {
  CHECK_AMR(a);
  if (!a->dist && !a->rank_begin.empty()) {
    set_error(std::string(who) + ": contexts of cup2d_amr_set_ranks have the blocking calls only");
    return CUP2D_ESTATE;
  }
  // a distributed context's kernels pull halos and all-reduce through the peer mapping, and a graph keeps its pointers:
  // nothing before the attach (a fresh context, or one whose regrid moved it onto new arrays)
  if (a->dist && a->nranks > 1 && !a->poisson->peers_attached) {
    set_error(std::string(who) + ": distributed context before cup2d_amr_peer_attach");
    return CUP2D_ESTATE;
  }
  const bool dev_dt = !(dt_in > 0);
  if (std::isnan(dt_in) || std::isinf(dt_in) || (pressure_only && dev_dt) || (dev_dt && !(cfl > 0 && std::isfinite(cfl))) ||
      !(tol_abs >= 0) || !(tol_rel >= 0) || max_restarts < 0 || max_iter < 0) {
    set_error(std::string(who) + ": bad arguments");
    return CUP2D_EINVAL;
  }
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc;
  if ((rc = ensure_poisson(a))) return rc;
  if (!a->d_rec) CUP2D_CUDA(cudaMalloc(&a->d_rec, AMR_REC_N * sizeof(double)));
  if (!a->dist && !a->ev_fork) {
    cudaEvent_t f, j;
    CUP2D_CUDA(cudaEventCreateWithFlags(&f, cudaEventDisableTiming));
    a->ev_fork = f;
    CUP2D_CUDA(cudaEventCreateWithFlags(&j, cudaEventDisableTiming));
    a->ev_join = j;
  }
  if (!dev_dt) amr_set_dt_kernel<<<1, 1, 0, a->stream>>>(a->d_rec, dt_in);
  CUP2D_CUDA(cudaGetLastError());
  a->step_pending = true;
  // the first enqueue of each form on a mesh runs directly: the lazily built tables, labs and Poisson context, the kernels'
  // attributes and constants are set up in it (no allocation or synchronous copy may happen inside a capture)
  const unsigned form = 1u << (2 * (a->fast ? 1 : 0) + (pressure_only ? 1 : 0));
  bool graph = a->use_graph && (a->warmed & form);
#ifdef CUP2D_FULL_EMU
  graph = false;
#endif
  if (!graph) {
    if ((rc = enqueue_body(a, pressure_only, dev_dt, cfl, tol_abs, tol_rel, max_restarts, max_iter, false))) return rc;
    a->warmed |= form;
    return CUP2D_OK;
  }
#ifndef CUP2D_FULL_EMU
  auto bits = [](double v) { unsigned long long u; memcpy(&u, &v, 8); return u; };
  const std::vector<unsigned long long> key = {(unsigned long long)a->fast, (unsigned long long)pressure_only, (unsigned long long)dev_dt,
                                               bits(cfl), bits(tol_abs), bits(tol_rel), (unsigned long long)max_restarts,
                                               (unsigned long long)max_iter};
  cup2d_amr::StepGraph *hit = nullptr;
  for (auto &g : a->graphs)
    if (g.key == key) hit = &g;
  if (!hit) {
    if (a->graphs.size() >= 32) { // a caller cycling through many argument sets: drop the oldest
      cudaGraphExecDestroy((cudaGraphExec_t)a->graphs.front().exec);
      cudaGraphDestroy((cudaGraph_t)a->graphs.front().graph);
      a->graphs.erase(a->graphs.begin());
    }
    CUP2D_CUDA(cudaStreamBeginCapture(a->stream, cudaStreamCaptureModeRelaxed));
    rc = enqueue_body(a, pressure_only, dev_dt, cfl, tol_abs, tol_rel, max_restarts, max_iter, true);
    cudaGraph_t g = nullptr;
    const cudaError_t e = cudaStreamEndCapture(a->stream, &g);
    if (rc || e != cudaSuccess) {
      if (g) cudaGraphDestroy(g);
      if (rc) return rc;
      CUP2D_CUDA(e);
    }
    cudaGraphExec_t x = nullptr;
    if (cudaGraphInstantiate(&x, g, 0) != cudaSuccess) {
      cudaGraphDestroy(g);
      set_error(std::string(who) + ": cudaGraphInstantiate failed");
      return CUP2D_ECUDA;
    }
    cup2d_amr::StepGraph sg;
    sg.key = key;
    sg.exec = x;
    sg.graph = g;
    a->graphs.push_back(sg);
    hit = &a->graphs.back();
  }
  CUP2D_CUDA(cudaGraphLaunch((cudaGraphExec_t)hit->exec, a->stream));
#endif
  return CUP2D_OK;
}

extern "C" {

/* cup2d_amr_step without bodies and without host synchronisation (include/cup2d_b200.h) */
int cup2d_amr_step_enqueue(cup2d_amr *a, double cfl, double dt_in, double tol_abs, double tol_rel, int max_restarts,
                           int max_iter) {
  return amr_enqueue(a, "cup2d_amr_step_enqueue", false, cfl, dt_in, tol_abs, tol_rel, max_restarts, max_iter);
}

/* the pressure section alone: poisson_rhs (u_def = tmpV, chi as they stand), solve, pressure_correct, enqueued */
int cup2d_amr_pressure_enqueue(cup2d_amr *a, double dt, double tol_abs, double tol_rel, int max_restarts, int max_iter) {
  return amr_enqueue(a, "cup2d_amr_pressure_enqueue", true, 0.0, dt, tol_abs, tol_rel, max_restarts, max_iter);
}

int cup2d_amr_step_result(cup2d_amr *a, double *dt_out, int *iters_out, double *err_out) {
  CHECK_AMR(a);
  if (!a->step_pending) {
    set_error("cup2d_amr_step_result: no step or pressure section has been enqueued since the last result");
    return CUP2D_ESTATE;
  }
  CUP2D_CUDA(cudaSetDevice(a->device));
  double dt = 0;
  CUP2D_CUDA(cudaMemcpyAsync(&dt, a->d_rec + AMR_REC_DT, sizeof dt, cudaMemcpyDeviceToHost, a->stream));
  CUP2D_CUDA(cudaStreamSynchronize(a->stream)); // (the stream waited for the solve on the Poisson context's stream)
  a->step_pending = false;
  const int rc = poisson_result(a->poisson, iters_out, err_out);
  if (dt_out) *dt_out = dt;
  return rc;
}

int cup2d_amr_set_graph(cup2d_amr *a, int on) {
  CHECK_AMR(a);
  if (!a->dist && !a->rank_begin.empty()) {
    set_error("cup2d_amr_set_graph: contexts of cup2d_amr_set_ranks have the blocking calls only");
    return CUP2D_ESTATE;
  }
  a->use_graph = on != 0;
  return CUP2D_OK;
}
#endif

int cup2d_amr_sync(cup2d_amr *a) {
  CHECK_AMR(a);
  CUP2D_CUDA(cudaSetDevice(a->device));
  CUP2D_CUDA(cudaStreamSynchronize(a->stream));
  return CUP2D_OK;
}

} // extern "C"
