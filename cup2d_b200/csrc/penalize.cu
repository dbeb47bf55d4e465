// Penalisation phase on device-resident fields (SURVEY §8(f) rank 3; main.cpp:6643-6681, 6944-7002), on the uniform grid
// (cup2d_sim) and on multi-level meshes (cup2d_amr).
//
// A shape is what the reference keeps per shape in `obstacleBlocks` (main.cpp:3283-3286, 4245-4263): the list of
// blocks its body touches with, per block, its own chi X[8][8] and deformation velocity udef[8][8][2].  The host body
// model (out of scope) produces these every step; they are uploaded with cup2d_shape_set — a few hundred KB — and the
// velocity field never leaves the device:
//   cup2d_shape_integrals : the 7 sums {PM,PJ,PX,PY,UM,VM,AM} of main.cpp:6648-6679 (global across ranks); the 3x3
//                           solve for (u,v,omega) and the collision logic stay on the host
//   cup2d_penalize        : V = alpha V + (1-alpha)(u_s + omega x r + udef) where the shape owns the cell (6944-6979)
//   cup2d_udef_assemble   : tmpV = sum over shapes of udef where the shape's chi is not below the field's (6980-7002)
// One thread per cell of an obstacle block, 4 blocks per CTA.  The blend and the assembly use explicit
// round-to-nearest operations (no FMA contraction): they reproduce the reference bit for bit; the sums are reduced
// in a fixed order (deterministic, but not the reference's sequential order: 1e-13 relative).
//
// The cup2d_amr_* calls are the same on a multi-level mesh, with the cell size and the block position taken per block
// (Info::h, Info::origin: main.cpp:695-696): the blend and assembly kernels are shared, the cell size of block id is
// hb[id] there and h on the uniform grid.  cup2d_amr_shape_integrals reduces one obstacle block per CTA and adds the
// per-block results on the host in block order (deterministic; the reference's OpenMP reduction has no fixed order:
// agreement to rounding, not bitwise).
#include "sim.h"
#include "amr.h"
#include <algorithm>

namespace cup2d {

constexpr int NT = 256;

struct ShapeView {
  const int *ids;
  const double *X, *udef;
  int nob;
};

// cell centre relative to the shape's centre of mass: p = origin + h (i + 0.5) - C, origin = (8 i) h
// (main.cpp:695, 6667-6670)
__device__ __forceinline__ void rel_pos(const int2 b, double h, int ix, int iy, double cx, double cy, double &px,
                                        double &py) {
  px = __dsub_rn(__dadd_rn(__dmul_rn((double)(b.x * CUP2D_BS), h), __dmul_rn(h, (double)ix + 0.5)), cx);
  py = __dsub_rn(__dadd_rn(__dmul_rn((double)(b.y * CUP2D_BS), h), __dmul_rn(h, (double)iy + 0.5)), cy);
}

// PART 0: {PM, PJ, PX, PY} (geometry)   PART 1: {UM, VM, AM} (momentum)
template <int PART>
__global__ void __launch_bounds__(NT)
shape_integrals_kernel(ShapeView sh, const double *__restrict__ vel, const int2 *__restrict__ ij, double h,
                       double lambdt, double cx, double cy, double *partials, unsigned int *counter, Comm comm,
                       double *out) {
  constexpr int NS = PART == 0 ? 4 : 3;
  double sums[NS];
#pragma unroll
  for (int k = 0; k < NS; k++) sums[k] = 0.0;
  const int cell = threadIdx.x & 63, ix = cell & 7, iy = cell >> 3;
  const double hsq = h * h;
  for (int k = blockIdx.x * (NT / 64) + (threadIdx.x >> 6); k < sh.nob; k += gridDim.x * (NT / 64)) {
    const double x = sh.X[(size_t)k * 64 + cell];
    if (x <= 0) continue;
    const int id = sh.ids[k];
    const double xl = x >= 0.5 ? lambdt : 0.0;
    const double F = hsq * xl / (1 + xl);
    double px, py;
    rel_pos(ij[id], h, ix, iy, cx, cy, px, py);
    if (PART == 0) {
      sums[0] += F;
      sums[1] += F * (px * px + py * py);
      sums[2] += F * px;
      sums[3] += F * py;
    } else {
      const double2 v = reinterpret_cast<const double2 *>(vel)[(size_t)id * 64 + cell];
      const double2 ud = reinterpret_cast<const double2 *>(sh.udef)[(size_t)k * 64 + cell];
      const double du = v.x - ud.x, dv = v.y - ud.y;
      sums[0] += F * du;
      sums[1] += F * dv;
      sums[2] += F * (px * dv - py * du);
    }
  }
  grid_reduce<NS, NT>(sums, 0.0, partials, counter, comm, [=](const double *t, double) {
    for (int k = 0; k < NS; k++) out[(PART == 0 ? 0 : 4) + k] = t[k];
  });
}

// multi-level meshes: one CTA (64 threads) per obstacle block: part[k][0..6] = the block's share of {PM, PJ, PX, PY, UM, VM, AM}
__global__ void __launch_bounds__(64)
amr_shape_sums_kernel(ShapeView sh, const double *__restrict__ vel, const int2 *__restrict__ ij,
                      const double *__restrict__ hb, double lambdt, double cx, double cy, double *__restrict__ part) {
  __shared__ double s_w1[7];
  const int k = blockIdx.x, cell = threadIdx.x, ix = cell & 7, iy = cell >> 3;
  double sums[7] = {0, 0, 0, 0, 0, 0, 0};
  const double x = sh.X[(size_t)k * 64 + cell];
  if (x > 0) {
    const int id = sh.ids[k];
    const double h = hb[id];
    const double xl = x >= 0.5 ? lambdt : 0.0;
    const double F = (h * h) * xl / (1 + xl);
    double px, py;
    rel_pos(ij[id], h, ix, iy, cx, cy, px, py);
    const double2 v = reinterpret_cast<const double2 *>(vel)[(size_t)id * 64 + cell];
    const double2 ud = reinterpret_cast<const double2 *>(sh.udef)[(size_t)k * 64 + cell];
    const double du = v.x - ud.x, dv = v.y - ud.y;
    sums[0] = F;
    sums[1] = F * (px * px + py * py);
    sums[2] = F * px;
    sums[3] = F * py;
    sums[4] = F * du;
    sums[5] = F * dv;
    sums[6] = F * (px * dv - py * du);
  }
  warp_sum<7>(sums);
  if (threadIdx.x == 32)
    for (int q = 0; q < 7; q++) s_w1[q] = sums[q];
  __syncthreads();
  if (threadIdx.x == 0)
    for (int q = 0; q < 7; q++) part[(size_t)k * 7 + q] = sums[q] + s_w1[q];
}

// the cell size of block id is hb[id] on a multi-level mesh (hb != nullptr), h on the uniform grid
__global__ void __launch_bounds__(NT)
penalize_kernel(ShapeView sh, double *__restrict__ vel, const double *__restrict__ chi, const int2 *__restrict__ ij,
                const double *__restrict__ hb, double h, double inv1lam, double cx, double cy, double us, double vs,
                double omega) {
  const int cell = threadIdx.x & 63, ix = cell & 7, iy = cell >> 3;
  for (int k = blockIdx.x * (NT / 64) + (threadIdx.x >> 6); k < sh.nob; k += gridDim.x * (NT / 64)) {
    const double x = sh.X[(size_t)k * 64 + cell];
    const int id = sh.ids[k];
    if (chi[(size_t)id * 64 + cell] > x || x <= 0) continue;
    double px, py;
    rel_pos(ij[id], hb ? hb[id] : h, ix, iy, cx, cy, px, py);
    const double alpha = x > 0.5 ? inv1lam : 1.0, beta = __dsub_rn(1.0, alpha);
    const double2 ud = reinterpret_cast<const double2 *>(sh.udef)[(size_t)k * 64 + cell];
    const double US = __dadd_rn(__dsub_rn(us, __dmul_rn(omega, py)), ud.x);
    const double VS = __dadd_rn(__dadd_rn(vs, __dmul_rn(omega, px)), ud.y);
    double2 *vp = reinterpret_cast<double2 *>(vel) + (size_t)id * 64 + cell;
    double2 v = *vp;
    v.x = __dadd_rn(__dmul_rn(alpha, v.x), __dmul_rn(beta, US));
    v.y = __dadd_rn(__dmul_rn(alpha, v.y), __dmul_rn(beta, VS));
    *vp = v;
  }
}

__global__ void __launch_bounds__(NT)
udef_add_kernel(ShapeView sh, double *__restrict__ tmpv, const double *__restrict__ chi) {
  const int cell = threadIdx.x & 63;
  for (int k = blockIdx.x * (NT / 64) + (threadIdx.x >> 6); k < sh.nob; k += gridDim.x * (NT / 64)) {
    const int id = sh.ids[k];
    if (sh.X[(size_t)k * 64 + cell] < chi[(size_t)id * 64 + cell]) continue;
    const double2 ud = reinterpret_cast<const double2 *>(sh.udef)[(size_t)k * 64 + cell];
    double2 *tp = reinterpret_cast<double2 *>(tmpv) + (size_t)id * 64 + cell;
    double2 t = *tp;
    t.x += ud.x;
    t.y += ud.y;
    *tp = t;
  }
}

static ShapeView view_of(const Shape &sh) { return ShapeView{sh.d_ids, sh.d_X, sh.d_udef, sh.nob}; }
// grid of the obstacle-block kernels: 4 blocks per CTA, at most `cap` CTAs
static int ob_grid(int nob, int cap) { return std::max(1, std::min((nob + NT / 64 - 1) / (NT / 64), cap)); }

// a host table of n ints on the device, uploaded on first use
static int upload_once(int *&d, const int32_t *h, size_t n) {
  if (d) return CUP2D_OK;
  CUP2D_CUDA(cudaMalloc(&d, n * sizeof(int)));
  CUP2D_CUDA(cudaMemcpy(d, h, n * sizeof(int), cudaMemcpyHostToDevice));
  return CUP2D_OK;
}

int ensure_block_ij(cup2d_sim *s) { return upload_once(s->d_ij, s->ij.data() + 2 * s->gbegin, (size_t)s->nloc * 2); }

// ids, X and udef of nob obstacle blocks into `sh`, copied on `stream`
static int shape_upload(Shape &sh, int nob, const int32_t *ids, const double *X, const double *udef, cudaStream_t stream) {
  if (nob > sh.cap) {
    shape_free(sh);
    sh.d_ids = nullptr; sh.d_X = sh.d_udef = nullptr;
    sh.cap = 0;
    const int cap = nob + nob / 4 + 16; // the body moves: leave room so that most steps do not reallocate
    CUP2D_CUDA(cudaMalloc(&sh.d_ids, (size_t)cap * sizeof(int)));
    CUP2D_CUDA(cudaMalloc(&sh.d_X, (size_t)cap * 64 * sizeof(double)));
    CUP2D_CUDA(cudaMalloc(&sh.d_udef, (size_t)cap * 128 * sizeof(double)));
    sh.cap = cap;
  }
  sh.nob = nob;
  if (nob > 0) {
    CUP2D_CUDA(cudaMemcpyAsync(sh.d_ids, ids, (size_t)nob * sizeof(int), cudaMemcpyHostToDevice, stream));
    CUP2D_CUDA(cudaMemcpyAsync(sh.d_X, X, (size_t)nob * 64 * sizeof(double), cudaMemcpyHostToDevice, stream));
    CUP2D_CUDA(cudaMemcpyAsync(sh.d_udef, udef, (size_t)nob * 128 * sizeof(double), cudaMemcpyHostToDevice, stream));
  }
  return CUP2D_OK;
}

int shape_set(cup2d_sim *s, int shape, int nob, const int32_t *ids, const double *X, const double *udef) {
  if ((int)s->shapes.size() <= shape) s->shapes.resize(shape + 1);
  return shape_upload(s->shapes[shape], nob, ids, X, udef, s->stream);
}

void shapes_free(cup2d_sim *s) {
  for (auto &sh : s->shapes) shape_free(sh);
  s->shapes.clear();
}

int shape_integrals(cup2d_sim *s, int shape, double lambda, double dt, double cx, double cy, double *out) {
  int rc = ensure_block_ij(s);
  if (rc) return rc;
  const ShapeView v = view_of(s->shapes[shape]);
  const int grid = ob_grid(v.nob, s->num_sms * 8);
  const int2 *ij = reinterpret_cast<const int2 *>(s->d_ij);
  // ranks that hold no block of this shape still take part in the cross-rank sum (grid of one idle CTA)
  shape_integrals_kernel<0><<<grid, NT, 0, s->stream>>>(v, s->f[CUP2D_VEL], ij, s->h, lambda * dt, cx, cy,
                                                       s->d_partials, s->d_counter, s->comm, s->d_scal);
  shape_integrals_kernel<1><<<grid, NT, 0, s->stream>>>(v, s->f[CUP2D_VEL], ij, s->h, lambda * dt, cx, cy,
                                                       s->d_partials, s->d_counter, s->comm, s->d_scal);
  s->launches += 2;
  CUP2D_CUDA(cudaGetLastError());
  CUP2D_CUDA(cudaMemcpyAsync(s->h_scal, s->d_scal, 7 * sizeof(double), cudaMemcpyDeviceToHost, s->stream));
  CUP2D_CUDA(cudaStreamSynchronize(s->stream));
  for (int k = 0; k < 7; k++) out[k] = s->h_scal[k];
  return CUP2D_OK;
}

int shape_penalize(cup2d_sim *s, int shape, double lambda, double dt, double cx, double cy, double us, double vs,
                   double omega) {
  int rc = ensure_block_ij(s);
  if (rc) return rc;
  const ShapeView v = view_of(s->shapes[shape]);
  if (v.nob == 0) return CUP2D_OK;
  penalize_kernel<<<ob_grid(v.nob, s->num_sms * 8), NT, 0, s->stream>>>(v, s->f[CUP2D_VEL], s->f[CUP2D_CHI],
                                                                        reinterpret_cast<const int2 *>(s->d_ij), nullptr, s->h,
                                                                        1 / (1 + lambda * dt), cx, cy, us, vs, omega);
  s->launches++;
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

int udef_assemble(cup2d_sim *s) {
  CUP2D_CUDA(cudaMemsetAsync(s->f[CUP2D_TMPV], 0, (size_t)s->nloc * 128 * sizeof(double), s->stream));
  for (const auto &sh : s->shapes) {
    if (sh.nob == 0) continue;
    udef_add_kernel<<<ob_grid(sh.nob, s->num_sms * 8), NT, 0, s->stream>>>(view_of(sh), s->f[CUP2D_TMPV], s->f[CUP2D_CHI]);
    s->launches++;
  }
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

} // namespace cup2d

int amr_ensure_ij(cup2d_amr *a) { return cup2d::upload_once(a->d_ij, a->h_ij.data(), (size_t)a->nb * 2); }

using namespace cup2d;

#define CHECK_AMR_SHAPE(a, shape, must_exist)                                                     \
  CUP2D_REQUIRE((a) != nullptr, "null cup2d_amr handle");                                         \
  CUP2D_REQUIRE(shape >= 0 && shape < 64, "shape index out of range (0..63)");                    \
  CUP2D_REQUIRE(!(must_exist) || shape < (int)(a)->shapes.size(), "shape has not been set (cup2d_amr_shape_set)")

extern "C" {

int cup2d_amr_shape_set(cup2d_amr *a, int shape, int nob, const int32_t *block_ids, const double *chi, const double *udef) {
  CHECK_AMR_SHAPE(a, shape, false);
  CUP2D_REQUIRE(nob >= 0 && (nob == 0 || (block_ids && chi && udef)), "cup2d_amr_shape_set: bad arguments");
  for (int k = 0; k < nob; k++)
    CUP2D_REQUIRE(block_ids[k] >= 0 && block_ids[k] < a->nb, "cup2d_amr_shape_set: block id outside the mesh");
  CUP2D_CUDA(cudaSetDevice(a->device));
  if ((int)a->shapes.size() <= shape) a->shapes.resize(shape + 1);
  cup2d_amr::Shape &sh = a->shapes[shape];
  sh.has_dist = false;
  sh.has_surface = false;
  sh.ascending = true; // what cup2d_amr_collide needs of the ids (recorded, not enforced here)
  for (int k = 1; k < nob; k++) sh.ascending = sh.ascending && block_ids[k - 1] < block_ids[k];
  if (nob > sh.cap) { // the shape grows: its signed distance goes with the old arrays
    cudaFree(sh.d_dist);
    sh.d_dist = nullptr;
  }
  int rc = shape_upload(sh, nob, block_ids, chi, udef, a->stream);
  if (rc) return rc;
  if (nob > 0) CUP2D_CUDA(cudaStreamSynchronize(a->stream)); // the caller's arrays may be pageable and short-lived
  return CUP2D_OK;
}

int cup2d_amr_shape_integrals(cup2d_amr *a, int shape, double lambda, double dt, double cx, double cy, double *out7) {
  CHECK_AMR_SHAPE(a, shape, true);
  CUP2D_REQUIRE(out7, "cup2d_amr_shape_integrals: null output");
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc = amr_ensure_ij(a);
  if (rc) return rc;
  for (int q = 0; q < 7; q++) out7[q] = 0.0;
  const ShapeView v = view_of(a->shapes[shape]);
  if (v.nob == 0) return amr_dist_sum(a, out7, 7); // a rank that holds no block of this shape still takes part in the sum
  if (v.nob > a->shape_part_cap) {
    cudaFree(a->d_shape_part);
    a->d_shape_part = nullptr, a->shape_part_cap = 0;
    CUP2D_CUDA(cudaMalloc(&a->d_shape_part, (size_t)(v.nob + 64) * 7 * sizeof(double)));
    a->shape_part_cap = v.nob + 64;
  }
  amr_shape_sums_kernel<<<v.nob, 64, 0, a->stream>>>(v, a->f[CUP2D_VEL], reinterpret_cast<const int2 *>(a->d_ij), a->d_h,
                                                     lambda * dt, cx, cy, a->d_shape_part);
  CUP2D_CUDA(cudaGetLastError());
  a->h_shape_part.resize((size_t)v.nob * 7);
  CUP2D_CUDA(cudaMemcpyAsync(a->h_shape_part.data(), a->d_shape_part, (size_t)v.nob * 7 * sizeof(double), cudaMemcpyDeviceToHost,
                             a->stream));
  CUP2D_CUDA(cudaStreamSynchronize(a->stream));
  for (int k = 0; k < v.nob; k++)
    for (int q = 0; q < 7; q++) out7[q] += a->h_shape_part[(size_t)k * 7 + q];
  return amr_dist_sum(a, out7, 7);
}

int cup2d_amr_penalize(cup2d_amr *a, int shape, double lambda, double dt, double cx, double cy, double us, double vs,
                       double omega) {
  CHECK_AMR_SHAPE(a, shape, true);
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc = amr_ensure_ij(a);
  if (rc) return rc;
  const ShapeView v = view_of(a->shapes[shape]);
  if (v.nob == 0) return CUP2D_OK;
  penalize_kernel<<<ob_grid(v.nob, AMR_GRID_SMS * 8), NT, 0, a->stream>>>(v, a->f[CUP2D_VEL], a->f[CUP2D_CHI],
                                                                         reinterpret_cast<const int2 *>(a->d_ij), a->d_h, 0,
                                                                         1 / (1 + lambda * dt), cx, cy, us, vs, omega);
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

int cup2d_amr_udef_assemble(cup2d_amr *a) {
  CUP2D_REQUIRE(a != nullptr, "null cup2d_amr handle");
  CUP2D_CUDA(cudaSetDevice(a->device));
  CUP2D_CUDA(cudaMemsetAsync(a->f[CUP2D_TMPV], 0, (size_t)a->nb * 128 * sizeof(double), a->stream));
  for (const auto &sh : a->shapes) {
    if (sh.nob == 0) continue;
    udef_add_kernel<<<ob_grid(sh.nob, AMR_GRID_SMS * 8), NT, 0, a->stream>>>(view_of(sh), a->f[CUP2D_TMPV], a->f[CUP2D_CHI]);
  }
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

} // extern "C"
