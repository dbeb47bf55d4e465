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
#include <map>
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

__global__ void amr_advect_kernel(const double *__restrict__ lab, double *__restrict__ out, const double *__restrict__ hb,
                                  int64_t ncells, double nu, double dt) {
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

__global__ void amr_div_kernel(const double *__restrict__ labv, const double *__restrict__ labu,
                               const double *__restrict__ chi, double *__restrict__ tmp, const double *__restrict__ hb,
                               int64_t ncells, double dt) {
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

__global__ void amr_gradp_kernel(const double *__restrict__ labp, double *__restrict__ tmpv, const double *__restrict__ hb,
                                 int64_t ncells, double dt) {
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
__global__ void amr_shift_kernel(double *__restrict__ p, const double *__restrict__ src, const double *__restrict__ add,
                                 int64_t n, double shift) {
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
template <int MODE>
__global__ void amr_fluxcorr_kernel(const CoarseFace *__restrict__ cf, int ncf, const double *labA, const double *labB,
                                    const double *chi, const double *hb, double *__restrict__ result, double nu,
                                    double dt) {
  constexpr int DIM = MODE == 0 ? 2 : 1;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ncf * 8 * DIM) return;
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
  int64_t nnz = cup2d_amr_plan_stencil(a->plan, which, nullptr, nullptr, nullptr, nullptr);
  if (nnz < 0) return CUP2D_EINVAL;
  const int64_t per_block = LABN[which] * LABN[which] * LABD[which];
  const int64_t nrows = a->nb * per_block;
  std::vector<int64_t> rp((a->dist ? a->nglobal : a->nb) * per_block + 1);
  std::vector<int32_t> sb(nnz), sc(nnz);
  std::vector<double> w(nnz);
  cup2d_amr_plan_stencil(a->plan, which, rp.data(), sb.data(), sc.data(), w.data());
  if (a->dist) { // the rows of this rank's blocks (contiguous: rows are in block order), sources renumbered to local slots
    const int64_t r0 = a->gbegin * per_block, e0 = rp[r0], e1 = rp[r0 + nrows];
    for (int64_t e = e0; e < e1; e++) {
      sb[e] = a->slot_of[sb[e]];
      if (sb[e] < 0) {
        set_error("distributed context: a lab source lies outside the halo set");
        return CUP2D_EINVAL;
      }
    }
    std::vector<int64_t> rpl(nrows + 1);
    for (int64_t r = 0; r <= nrows; r++) rpl[r] = rp[r0 + r] - e0;
    rp.swap(rpl);
    auto keep = [&](auto &v) {
      v.erase(v.begin() + e1, v.end());
      v.erase(v.begin(), v.begin() + e0);
    };
    keep(sb);
    keep(sc);
    keep(w);
    nnz = e1 - e0;
  }
  Csr &c = a->csr[which];
  c.nrows = nrows;
  CUP2D_CUDA(cudaMalloc(&c.rowptr, (nrows + 1) * sizeof(int64_t)));
  CUP2D_CUDA(cudaMalloc(&c.src_block, std::max<int64_t>(nnz, 1) * sizeof(int)));
  CUP2D_CUDA(cudaMalloc(&c.src_cc, std::max<int64_t>(nnz, 1) * sizeof(int)));
  CUP2D_CUDA(cudaMalloc(&c.w, std::max<int64_t>(nnz, 1) * sizeof(double)));
  CUP2D_CUDA(cudaMemcpy(c.rowptr, rp.data(), (nrows + 1) * sizeof(int64_t), cudaMemcpyHostToDevice));
  CUP2D_CUDA(cudaMemcpy(c.src_block, sb.data(), nnz * sizeof(int), cudaMemcpyHostToDevice));
  CUP2D_CUDA(cudaMemcpy(c.src_cc, sc.data(), nnz * sizeof(int), cudaMemcpyHostToDevice));
  CUP2D_CUDA(cudaMemcpy(c.w, w.data(), nnz * sizeof(double), cudaMemcpyHostToDevice));
  CUP2D_CUDA(cudaMalloc(&a->lab[which], nrows * sizeof(double)));
  return CUP2D_OK;
}

// The full tables (every lab cell of every block) serve the baseline kernels only; they are built the first time one of
// those runs, so that a context driven through the fast kernels (compact tables: ghost rows of irregular blocks) never pays
// for them — they grow with the mesh, the compact ones with its level interfaces.
static int gather(cup2d_amr *a, int which, const double *field, double *&lab) {
  int rc;
  if (a->dist && which != 1 && which != 3) { // (1 and 3: the labs of the tagging field, whose sources are in the halo set)
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
static int fluxcorr(cup2d_amr *a, const double *labA, const double *labB, double *result, double dt) {
  constexpr int DIM = MODE == 0 ? 2 : 1;
  for (int dir = 0; dir < 2; dir++) { // x faces, then y faces (fillcases order)
    const int n = a->ncf[dir] * 8 * DIM;
    if (n == 0) continue;
    amr_fluxcorr_kernel<MODE><<<(n + 127) / 128, 128, 0, a->stream>>>(a->d_cf[dir], a->ncf[dir], labA, labB, a->f[CUP2D_CHI],
                                                                      a->d_h, result, a->nu, dt);
  }
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

} // namespace cup2d

using namespace cup2d;

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
  a->nb = nblocks;
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
  std::vector<double> h(nblocks);
  for (int64_t k = 0; k < nblocks; k++) h[k] = h0 / (double)(1 << level_ij[3 * k]);
  a->h_ij.resize(2 * nblocks);
  for (int64_t k = 0; k < nblocks; k++) a->h_ij[2 * k] = level_ij[3 * k + 1], a->h_ij[2 * k + 1] = level_ij[3 * k + 2];
  a->hmin = *std::min_element(h.begin(), h.end());
  a->h_part.resize(2 * nblocks);
  if (cudaMalloc(&a->d_part, 2 * nblocks * sizeof(double)) != cudaSuccess) return fail(CUP2D_ECUDA);
  if (cudaMalloc(&a->d_h, nblocks * sizeof(double)) != cudaSuccess ||
      cudaMemcpy(a->d_h, h.data(), nblocks * sizeof(double), cudaMemcpyHostToDevice) != cudaSuccess)
    return fail(CUP2D_ECUDA);
  // coarse faces: group the plan's (fine block, face, coarse block, face, half) records by (coarse block, face)
  const int64_t nf = cup2d_amr_plan_faces(plan, nullptr);
  std::vector<int32_t> rec(5 * std::max<int64_t>(nf, 1));
  cup2d_amr_plan_faces(plan, rec.data());
  std::map<std::pair<int, int>, CoarseFace> byface;
  for (int64_t r = 0; r < nf; r++) {
    const int fine = rec[5 * r], kc = rec[5 * r + 2], fc = rec[5 * r + 3], half = rec[5 * r + 4];
    auto it = byface.find({kc, fc});
    if (it == byface.end()) it = byface.emplace(std::make_pair(kc, fc), CoarseFace{kc, fc, {-1, -1}}).first;
    it->second.fine[half] = fine;
  }
  std::vector<CoarseFace> lists[2];
  for (auto &e : byface) lists[e.second.face < 2 ? 0 : 1].push_back(e.second);
  for (int d = 0; d < 2; d++) {
    a->ncf[d] = (int)lists[d].size();
    if (lists[d].empty()) continue;
    if (cudaMalloc(&a->d_cf[d], lists[d].size() * sizeof(CoarseFace)) != cudaSuccess ||
        cudaMemcpy(a->d_cf[d], lists[d].data(), lists[d].size() * sizeof(CoarseFace), cudaMemcpyHostToDevice) != cudaSuccess)
      return fail(CUP2D_ECUDA);
  }
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
  cudaFree(a->d_nbr4); cudaFree(a->d_nbr8); cudaFree(a->d_irr_of); cudaFree(a->d_faceflux);
  a->free_shapes();
  for (auto &g : a->gt) {
    cudaFree(g.grow); cudaFree(g.rowptr); cudaFree(g.dst); cudaFree(g.sb); cudaFree(g.sc); cudaFree(g.w);
  }
#ifndef CUP2D_AMR_EMU
  if (a->poisson) cup2d_destroy(a->poisson);
#endif
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

/* tmpV = KernelAdvectDiffuse(vel), flux-corrected (main.cpp:6611-6617) */
int cup2d_amr_advect_diffuse_rhs(cup2d_amr *a, double dt) {
  CHECK_AMR(a);
  if (a->fast) return cup2d_amr_advect_diffuse_rhs_fast(a, dt);
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc = gather(a, 0, a->f[CUP2D_VEL], a->lab[0]);
  if (rc) return rc;
  amr_advect_kernel<<<grid_for(a->nb * 64), 256, 0, a->stream>>>(a->lab[0], a->f[CUP2D_TMPV], a->d_h, a->nb * 64, a->nu, dt);
  CUP2D_CUDA(cudaGetLastError());
  return fluxcorr<0>(a, a->lab[0], nullptr, a->f[CUP2D_TMPV], dt);
}

/* tmp = pressure_rhs(vel, u_def = tmpV, chi), flux-corrected (main.cpp:7007-7013); with_laplacian: then
 * tmp -= lap(pold), flux-corrected (main.cpp:7022-7027) */
int cup2d_amr_pressure_rhs(cup2d_amr *a, double dt, int with_laplacian) {
  CHECK_AMR(a);
  if (a->fast) return cup2d_amr_pressure_rhs_fast(a, dt, with_laplacian);
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc = gather(a, 1, a->f[CUP2D_VEL], a->lab[1]);
  if (rc || (rc = gather(a, 1, a->f[CUP2D_TMPV], a->lab_udef))) return rc;
  amr_div_kernel<<<grid_for(a->nb * 64), 256, 0, a->stream>>>(a->lab[1], a->lab_udef, a->f[CUP2D_CHI], a->f[CUP2D_TMP], a->d_h,
                                                             a->nb * 64, dt);
  CUP2D_CUDA(cudaGetLastError());
  if ((rc = fluxcorr<1>(a, a->lab[1], a->lab_udef, a->f[CUP2D_TMP], dt))) return rc;
  if (!with_laplacian) return CUP2D_OK;
  if ((rc = gather(a, 2, a->f[CUP2D_POLD], a->lab[2]))) return rc;
  amr_lap_kernel<<<grid_for(a->nb * 64), 256, 0, a->stream>>>(a->lab[2], a->f[CUP2D_TMP], a->nb * 64);
  CUP2D_CUDA(cudaGetLastError());
  return fluxcorr<2>(a, a->lab[2], nullptr, a->f[CUP2D_TMP], dt);
}

/* tmpV = pressureCorrectionKernel(pres) (main.cpp:7174-7179; not flux-corrected in the reference either) */
int cup2d_amr_pressure_gradient(cup2d_amr *a, double dt) {
  CHECK_AMR(a);
  if (a->fast) return cup2d_amr_pressure_gradient_fast(a, dt);
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc = gather(a, 2, a->f[CUP2D_PRES], a->lab[2]);
  if (rc) return rc;
  amr_gradp_kernel<<<grid_for(a->nb * 64), 256, 0, a->stream>>>(a->lab[2], a->f[CUP2D_TMPV], a->d_h, a->nb * 64, dt);
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

static int block_partials(cup2d_amr *a, int n_per_block) {
  CUP2D_CUDA(cudaMemcpyAsync(a->h_part.data(), a->d_part, (size_t)a->nb * n_per_block * sizeof(double), cudaMemcpyDeviceToHost,
                             a->stream));
  CUP2D_CUDA(cudaStreamSynchronize(a->stream));
  return CUP2D_OK;
}

/* adapt()'s per-block L-inf (main.cpp:4676-4697) on a multi-level mesh: vorticity of vel through the +-1 lab, the chi rule
 * of GradChiOnTmp through the {-4,-4,5,5,tensorial} chi lab (ghost tables built on first use); leaves the tagging field in
 * tmp like the reference does.  level_max = sim.levelMax (the finest level is level_max - 1). */
int cup2d_amr_adapt_tags(cup2d_amr *a, double rtol, int level_max, double *block_linf_out) {
  CHECK_AMR(a);
  if (!block_linf_out || level_max < 1 || level_max > 30) {
    set_error("cup2d_amr_adapt_tags: bad arguments");
    return CUP2D_EINVAL;
  }
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc;
  if ((rc = amr_dist_refresh(a, CUP2D_VEL)) || (rc = amr_dist_refresh(a, CUP2D_CHI))) return rc;
  if ((rc = gather(a, 1, a->f[CUP2D_VEL], a->lab[1])) || (rc = gather(a, 3, a->f[CUP2D_CHI], a->lab[3]))) return rc;
  amr_vorticity_kernel<<<grid_for(a->nb * 64), 256, 0, a->stream>>>(a->lab[1], a->f[CUP2D_TMP], a->d_h, a->nb * 64);
  amr_tag_block_kernel<<<grid_for(a->nb), 256, 0, a->stream>>>(a->lab[3], a->f[CUP2D_TMP], a->d_h,
                                                               a->h0 / (double)(1 << (level_max - 1)), rtol, a->d_part, a->nb);
  CUP2D_CUDA(cudaGetLastError());
  if ((rc = block_partials(a, 1))) return rc;
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
#else
static int dist_allreduce(cup2d_amr *, double &, double &, double &) { return CUP2D_OK; }
int amr_dist_refresh(cup2d_amr *, int) { return CUP2D_OK; }
int amr_dist_sum(cup2d_amr *, double *, int) { return CUP2D_OK; }
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

/* main.cpp:6607-6642: vold = vel; vel = vold + 0.5 K(vel)/h^2; vel = vold + K(vel)/h^2 (K flux-corrected) */
int cup2d_amr_advect_diffuse_rk2(cup2d_amr *a, double dt) {
  CHECK_AMR(a);
  CUP2D_CUDA(cudaSetDevice(a->device));
  const int64_t n = a->nb * 128;
  CUP2D_CUDA(cudaMemcpyAsync(a->f[CUP2D_VOLD], a->f[CUP2D_VEL], n * sizeof(double), cudaMemcpyDeviceToDevice, a->stream));
  for (int stage = 0; stage < 2; stage++) {
    int rc = cup2d_amr_advect_diffuse_rhs(a, dt);
    if (rc) return rc;
    amr_axpy_h2_kernel<<<grid_for(n), 256, 0, a->stream>>>(a->f[CUP2D_VEL], a->f[CUP2D_VOLD], a->f[CUP2D_TMPV], a->d_h, n,
                                                          stage == 0 ? 0.5 : 1.0);
    CUP2D_CUDA(cudaGetLastError());
  }
  return CUP2D_OK;
}

/* main.cpp:7007-7027 as one call: tmp = pressure_rhs(vel, u_def = tmpV, chi); pold = pres; pres = 0; tmp -= lap(pold) */
int cup2d_amr_poisson_rhs(cup2d_amr *a, double dt) {
  CHECK_AMR(a);
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc = cup2d_amr_pressure_rhs(a, dt, 0);
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
  amr_shift_kernel<<<grid_for(n), 256, 0, a->stream>>>(a->f[CUP2D_PRES], nullptr, nullptr, n, avg);
  if ((rc = weighted_mean(a, a->f[CUP2D_PRES], &avg))) return rc;
  amr_shift_kernel<<<grid_for(n), 256, 0, a->stream>>>(a->f[CUP2D_PRES], nullptr, a->f[CUP2D_POLD], n, avg);
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
  std::vector<int32_t> extra, n8(8 * nblocks);
  if (cup2d_amr_plan_neighbours(plan, n8.data())) return fail(CUP2D_EINVAL);
  for (int64_t k = b0; k < b1; k++)
    for (int j = 0; j < 8; j++)
      if (n8[8 * k + j] >= 0) extra.push_back(n8[8 * k + j]);
  const int64_t nirr_g = cup2d_amr_plan_irregular(plan, nullptr);
  std::vector<int32_t> irr(std::max<int64_t>(nirr_g, 1));
  cup2d_amr_plan_irregular(plan, irr.data());
  const int ncell[4] = {14 * 14 * 2, 10 * 10 * 2, 10 * 10, 16 * 16}; // (3: the chi lab of the tagging rule)
  for (int which = 0; which < 4; which++) {
    int64_t nrows = 0;
    const int64_t nnz = cup2d_amr_plan_ghosts(plan, which, &nrows, nullptr, nullptr, nullptr, nullptr, nullptr);
    if (nnz < 0) return fail(CUP2D_EINVAL);
    std::vector<int64_t> rp(nrows + 1);
    std::vector<int32_t> dst(std::max<int64_t>(nrows, 1)), sb(std::max<int64_t>(nnz, 1)), sc(std::max<int64_t>(nnz, 1));
    std::vector<double> w(std::max<int64_t>(nnz, 1));
    cup2d_amr_plan_ghosts(plan, which, &nrows, rp.data(), dst.data(), sb.data(), sc.data(), w.data());
    for (int64_t row = 0; row < nrows; row++) {
      const int32_t blk = irr[dst[row] / ncell[which]];
      if (blk < b0 || blk >= b1) continue;
      for (int64_t e = rp[row]; e < rp[row + 1]; e++) extra.push_back(sb[e]);
    }
  }
  {
    const int64_t nf = cup2d_amr_plan_faces(plan, nullptr);
    std::vector<int32_t> rec(5 * std::max<int64_t>(nf, 1));
    cup2d_amr_plan_faces(plan, rec.data());
    for (int64_t r = 0; r < nf; r++)
      if (rec[5 * r + 2] >= b0 && rec[5 * r + 2] < b1) extra.push_back(rec[5 * r]);
  }
  // this rank's rows of the Poisson matrix (as cup2d_amr_set_ranks)
  int64_t nnz = 0;
  const int64_t nr = cup2d_amr_plan_poisson(plan, nullptr, &nnz, nullptr, nullptr, nullptr, nullptr);
  if (nr < 0) return fail((int)nr);
  std::vector<int32_t> nbr(4 * nblocks), rows(std::max<int64_t>(nr, 1)), rowptr(nr + 1), col(std::max<int64_t>(nnz, 1));
  std::vector<double> val(std::max<int64_t>(nnz, 1));
  cup2d_amr_plan_poisson(plan, nbr.data(), &nnz, rows.data(), rowptr.data(), col.data(), val.data());
  const int64_t k0 = std::lower_bound(rows.begin(), rows.begin() + nr, (int32_t)(64 * b0)) - rows.begin();
  const int64_t k1 = std::lower_bound(rows.begin(), rows.begin() + nr, (int32_t)(64 * b1)) - rows.begin();
  std::vector<int32_t> my_rows(rows.begin() + k0, rows.begin() + k1), my_ptr(rowptr.begin() + k0, rowptr.begin() + k1 + 1);
  for (auto &r : my_rows) r -= (int32_t)(64 * b0);
  const int32_t e0 = my_ptr[0];
  for (auto &e : my_ptr) e -= e0;
  if ((rc = poisson_create_general_ranks_ex(nblocks, rank, nranks, rank_begin, nbr.data() + 4 * b0, k1 - k0, my_rows.data(),
                                            my_ptr.data(), col.data() + e0, val.data() + e0, (int64_t)extra.size(), extra.data(),
                                            device, &a->poisson)))
    return fail(rc);
  cup2d_sim *ps = a->poisson;
  a->stream = ps->stream;
  for (int f = 0; f < CUP2D_NFIELDS; f++) a->f[f] = ps->f[f];
  std::vector<int32_t> slot_of(nblocks, -1);
  for (int64_t k = 0; k < nloc; k++) slot_of[b0 + k] = (int32_t)k;
  for (int64_t k = 0; k < ps->nhalo; k++) slot_of[ps->halo_gid[k]] = (int32_t)(nloc + k);
  a->slot_of = slot_of;
  // cell size: own blocks and halo slots; the time step uses the smallest cell of the WHOLE mesh
  std::vector<double> h(ps->nslots, h0);
  a->hmin = h0;
  for (int64_t g = 0; g < nblocks; g++) {
    const double hg = h0 / (double)(1 << level_ij[3 * g]);
    a->hmin = std::min(a->hmin, hg);
    if (slot_of[g] >= 0) h[slot_of[g]] = hg;
  }
  a->h_ij.resize(2 * nloc);
  for (int64_t k = 0; k < nloc; k++) a->h_ij[2 * k] = level_ij[3 * (b0 + k) + 1], a->h_ij[2 * k + 1] = level_ij[3 * (b0 + k) + 2];
  a->h_part.resize(2 * nloc);
  if (cudaMalloc(&a->d_part, 2 * nloc * sizeof(double)) != cudaSuccess || cudaMalloc(&a->d_h, h.size() * sizeof(double)) != cudaSuccess ||
      cudaMemcpy(a->d_h, h.data(), h.size() * sizeof(double), cudaMemcpyHostToDevice) != cudaSuccess)
    return fail(CUP2D_ECUDA);
  if ((rc = amr_fast_setup_dist(a, slot_of, b0, b1))) return fail(rc);
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
  int64_t nnz = 0;
  const int64_t nr = cup2d_amr_plan_poisson(a->plan, nullptr, &nnz, nullptr, nullptr, nullptr, nullptr);
  if (nr < 0) return (int)nr;
  std::vector<int32_t> nbr(4 * a->nb), rows(std::max<int64_t>(nr, 1)), rowptr(nr + 1), col(std::max<int64_t>(nnz, 1));
  std::vector<double> val(std::max<int64_t>(nnz, 1));
  cup2d_amr_plan_poisson(a->plan, nbr.data(), &nnz, rows.data(), rowptr.data(), col.data(), val.data());
  const int64_t b0 = rank_begin[rank], b1 = rank_begin[rank + 1];
  const int64_t k0 = std::lower_bound(rows.begin(), rows.begin() + nr, (int32_t)(64 * b0)) - rows.begin();
  const int64_t k1 = std::lower_bound(rows.begin(), rows.begin() + nr, (int32_t)(64 * b1)) - rows.begin();
  std::vector<int32_t> my_rows(rows.begin() + k0, rows.begin() + k1), my_ptr(rowptr.begin() + k0, rowptr.begin() + k1 + 1);
  for (auto &r : my_rows) r -= (int32_t)(64 * b0);
  const int32_t e0 = my_ptr[0];
  for (auto &e : my_ptr) e -= e0;
  int rc = cup2d_poisson_create_general_ranks(a->nb, rank, nranks, rank_begin, nbr.data() + 4 * b0, k1 - k0, my_rows.data(),
                                              my_ptr.data(), col.data() + e0, val.data() + e0, a->device, &a->poisson);
  if (rc) return rc;
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
int cup2d_amr_poisson_solve(cup2d_amr *a, double tol_abs, double tol_rel, int max_restarts, int max_iter, int *iters,
                            double *err) {
  CHECK_AMR(a);
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc;
  if (!a->poisson) {
    int64_t nnz = 0;
    const int64_t nr = cup2d_amr_plan_poisson(a->plan, nullptr, &nnz, nullptr, nullptr, nullptr, nullptr);
    if (nr < 0) return (int)nr;
    std::vector<int32_t> nbr(4 * a->nb), rows(std::max<int64_t>(nr, 1)), rowptr(nr + 1), col(std::max<int64_t>(nnz, 1));
    std::vector<double> val(std::max<int64_t>(nnz, 1));
    cup2d_amr_plan_poisson(a->plan, nbr.data(), &nnz, rows.data(), rowptr.data(), col.data(), val.data());
    if ((rc = cup2d_poisson_create_general(a->nb, nbr.data(), nr, rows.data(), rowptr.data(), col.data(), val.data(), a->device,
                                           &a->poisson)))
      return rc;
  }
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
#endif

int cup2d_amr_sync(cup2d_amr *a) {
  CHECK_AMR(a);
  CUP2D_CUDA(cudaSetDevice(a->device));
  CUP2D_CUDA(cudaStreamSynchronize(a->stream));
  return CUP2D_OK;
}

} // extern "C"
