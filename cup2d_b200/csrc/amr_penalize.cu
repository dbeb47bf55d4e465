// Penalisation phase on a multi-level mesh (SURVEY §8(f) rank 3 on the meshes of rank 2; main.cpp:6643-6681, 6944-7002):
// the calls of penalize.cu on the cup2d_amr context.  Same contract — a shape is the reference's per-shape list of obstacle
// blocks with their own chi and u_def (main.cpp:3283-3286), uploaded every step; the velocity never leaves the device —
// with the cell size and the block position taken per block (Info::h, Info::origin: main.cpp:695-696).
//   cup2d_amr_shape_integrals : {PM,PJ,PX,PY,UM,VM,AM} of main.cpp:6648-6679: one CTA per obstacle block reduces its 64 cells,
//                               the host adds the per-block results in block order (deterministic; the reference's OpenMP
//                               reduction has no fixed order: agreement to rounding, not bitwise)
//   cup2d_amr_penalize        : the blend of main.cpp:6944-6979, explicit round-to-nearest operations: bit-identical
//   cup2d_amr_udef_assemble   : tmpV = sum of u_def where the shape's chi is not below the field's (6980-7002): bit-identical
// Also here, because it needs the same per-block (i, j, h) tables: cup2d_amr_dump, dump()'s three files from a multi-level mesh
// (main.cpp:3367-3467), byte for byte.
// STATUS: like the rest of the multi-level device path: compiled for sm_90a, its logic also checked on the CPU through
// the host emulation (tests/host_emu/).
#include "sim.h"
#include "amr.h"
#include <algorithm>
#include <fcntl.h>
#include <string>
#include <unistd.h>

#define CUP2D_REQUIRE(cond, msg)                                                                  \
  do {                                                                                            \
    if (!(cond)) {                                                                                \
      cup2d::set_error(msg);                                                                      \
      return CUP2D_EINVAL;                                                                        \
    }                                                                                             \
  } while (0)

namespace cup2d {

struct AmrShapeView {
  const int *ids;
  const double *X, *udef;
  int nob;
};

// cell centre relative to the shape's centre of mass: p = origin + h (i + 0.5) - C, origin = (8 i) h  (main.cpp:695, 6667-6670)
__device__ __forceinline__ void amr_rel_pos(const int2 b, double h, int ix, int iy, double cx, double cy, double &px,
                                            double &py) {
  px = __dsub_rn(__dadd_rn(__dmul_rn((double)(b.x * CUP2D_BS), h), __dmul_rn(h, (double)ix + 0.5)), cx);
  py = __dsub_rn(__dadd_rn(__dmul_rn((double)(b.y * CUP2D_BS), h), __dmul_rn(h, (double)iy + 0.5)), cy);
}

// one CTA (64 threads) per obstacle block: part[k][0..6] = the block's share of {PM, PJ, PX, PY, UM, VM, AM}
__global__ void __launch_bounds__(64)
amr_shape_sums_kernel(AmrShapeView sh, const double *__restrict__ vel, const int2 *__restrict__ ij,
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
    amr_rel_pos(ij[id], h, ix, iy, cx, cy, px, py);
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

__global__ void __launch_bounds__(256)
amr_penalize_kernel(AmrShapeView sh, double *__restrict__ vel, const double *__restrict__ chi, const int2 *__restrict__ ij,
                    const double *__restrict__ hb, double inv1lam, double cx, double cy, double us, double vs, double omega) {
  const int cell = threadIdx.x & 63, ix = cell & 7, iy = cell >> 3;
  for (int k = blockIdx.x * 4 + (threadIdx.x >> 6); k < sh.nob; k += gridDim.x * 4) {
    const double x = sh.X[(size_t)k * 64 + cell];
    const int id = sh.ids[k];
    if (chi[(size_t)id * 64 + cell] > x || x <= 0) continue;
    double px, py;
    amr_rel_pos(ij[id], hb[id], ix, iy, cx, cy, px, py);
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

__global__ void __launch_bounds__(256)
amr_udef_add_kernel(AmrShapeView sh, double *__restrict__ tmpv, const double *__restrict__ chi) {
  const int cell = threadIdx.x & 63;
  for (int k = blockIdx.x * 4 + (threadIdx.x >> 6); k < sh.nob; k += gridDim.x * 4) {
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

// dump() on a multi-level mesh (main.cpp:3425-3453): as dump_pack_kernel (regrid.cu) with the block's own cell size
__global__ void __launch_bounds__(256)
amr_dump_pack_kernel(const double *__restrict__ vel, const int2 *__restrict__ ij, const double *__restrict__ hb, int b0, int nb,
                     float4 *__restrict__ xyz, float *__restrict__ attr) {
  const size_t ncell = (size_t)nb * 64;
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < ncell; i += (size_t)gridDim.x * 256) {
    const int k = (int)(i >> 6), x = (int)(i & 7), y = (int)((i >> 3) & 7);
    const int2 b = ij[b0 + k];
    const double h = hb[b0 + k];
    const double u0 = __dadd_rn(__dmul_rn((double)(b.x * CUP2D_BS), h), __dmul_rn(h, (double)x));
    const double v0 = __dadd_rn(__dmul_rn((double)(b.y * CUP2D_BS), h), __dmul_rn(h, (double)y));
    const float fu0 = (float)u0, fv0 = (float)v0, fu1 = (float)__dadd_rn(u0, h), fv1 = (float)__dadd_rn(v0, h);
    xyz[2 * i] = make_float4(fu0, fv0, fu0, fv1);
    xyz[2 * i + 1] = make_float4(fu1, fv1, fu1, fv0);
    const double2 q = reinterpret_cast<const double2 *>(vel)[(size_t)(b0 + k) * 64 + (i & 63)];
    attr[3 * i] = (float)q.x;
    attr[3 * i + 1] = (float)q.y;
    attr[3 * i + 2] = 0.0f;
  }
}

static AmrShapeView view_of(const cup2d_amr::Shape &sh) { return AmrShapeView{sh.d_ids, sh.d_X, sh.d_udef, sh.nob}; }
static int ob_grid(int nob) { return std::max(1, std::min((nob + 3) / 4, AMR_GRID_SMS * 8)); }

static int ensure_ij(cup2d_amr *a) {
  if (a->d_ij) return CUP2D_OK;
  CUP2D_CUDA(cudaMalloc(&a->d_ij, (size_t)a->nb * 2 * sizeof(int)));
  CUP2D_CUDA(cudaMemcpy(a->d_ij, a->h_ij.data(), (size_t)a->nb * 2 * sizeof(int), cudaMemcpyHostToDevice));
  return CUP2D_OK;
}

} // namespace cup2d

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
  if (nob > sh.cap) {
    cudaFree(sh.d_ids); cudaFree(sh.d_X); cudaFree(sh.d_udef);
    sh.d_ids = nullptr; sh.d_X = sh.d_udef = nullptr;
    sh.cap = 0;
    const int cap = nob + nob / 4 + 16;
    CUP2D_CUDA(cudaMalloc(&sh.d_ids, (size_t)cap * sizeof(int)));
    CUP2D_CUDA(cudaMalloc(&sh.d_X, (size_t)cap * 64 * sizeof(double)));
    CUP2D_CUDA(cudaMalloc(&sh.d_udef, (size_t)cap * 128 * sizeof(double)));
    sh.cap = cap;
  }
  sh.nob = nob;
  if (nob > 0) {
    CUP2D_CUDA(cudaMemcpyAsync(sh.d_ids, block_ids, (size_t)nob * sizeof(int), cudaMemcpyHostToDevice, a->stream));
    CUP2D_CUDA(cudaMemcpyAsync(sh.d_X, chi, (size_t)nob * 64 * sizeof(double), cudaMemcpyHostToDevice, a->stream));
    CUP2D_CUDA(cudaMemcpyAsync(sh.d_udef, udef, (size_t)nob * 128 * sizeof(double), cudaMemcpyHostToDevice, a->stream));
    CUP2D_CUDA(cudaStreamSynchronize(a->stream)); // the caller's arrays may be pageable and short-lived
  }
  return CUP2D_OK;
}

int cup2d_amr_shape_integrals(cup2d_amr *a, int shape, double lambda, double dt, double cx, double cy, double *out7) {
  CHECK_AMR_SHAPE(a, shape, true);
  CUP2D_REQUIRE(out7, "cup2d_amr_shape_integrals: null output");
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc = ensure_ij(a);
  if (rc) return rc;
  for (int q = 0; q < 7; q++) out7[q] = 0.0;
  const AmrShapeView v = view_of(a->shapes[shape]);
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
  int rc = ensure_ij(a);
  if (rc) return rc;
  const AmrShapeView v = view_of(a->shapes[shape]);
  if (v.nob == 0) return CUP2D_OK;
  amr_penalize_kernel<<<ob_grid(v.nob), 256, 0, a->stream>>>(v, a->f[CUP2D_VEL], a->f[CUP2D_CHI],
                                                             reinterpret_cast<const int2 *>(a->d_ij), a->d_h,
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
    amr_udef_add_kernel<<<ob_grid(sh.nob), 256, 0, a->stream>>>(view_of(sh), a->f[CUP2D_TMPV], a->f[CUP2D_CHI]);
  }
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

/* dump() of the velocity on a multi-level mesh (main.cpp:3367-3467): path.xdmf2 / .xyz.raw / .attr.raw, the reference's
 * three files byte for byte (float32 cell quads + (u, v, 0) in block order) */
int cup2d_amr_dump(cup2d_amr *a, double time, const char *path) {
  CUP2D_REQUIRE(a != nullptr && path && *path, "cup2d_amr_dump: bad arguments");
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc = ensure_ij(a);
  if (rc) return rc;
  const std::string base(path);
  const std::string xyz_path = base + ".xyz.raw", attr_path = base + ".attr.raw", xdmf_path = base + ".xdmf2";
  const bool dist = a->dist && a->nranks > 1;   // every rank writes its own byte range, the last one the descriptor (main.cpp:3387-3390)
  if ((!dist || a->rank == a->nranks - 1) &&
      (rc = dump_write_xdmf(xdmf_path, xyz_path, attr_path, time, (long)(dist ? a->nglobal : a->nb) * 64)))
    return rc;
  const int CHUNK = (int)std::min<int64_t>(a->nb, 16384);
  const size_t nx = (size_t)CHUNK * 64 * 8, na = (size_t)CHUNK * 64 * 3;
  float *d_buf = nullptr, *h_buf = nullptr;
  CUP2D_CUDA(cudaMalloc(&d_buf, (nx + na) * sizeof(float)));
  if (cudaMallocHost(&h_buf, (nx + na) * sizeof(float)) != cudaSuccess) {
    cudaFree(d_buf);
    set_error("cup2d_amr_dump: cannot allocate the pinned staging buffer");
    return CUP2D_ECUDA;
  }
  const int oflags = O_CREAT | O_WRONLY | (dist ? 0 : O_TRUNC);
  const int fx = open(xyz_path.c_str(), oflags, 0644), fa = open(attr_path.c_str(), oflags, 0644);
  rc = (fx < 0 || fa < 0) ? CUP2D_EINVAL : CUP2D_OK;
  for (int64_t b0 = 0; rc == CUP2D_OK && b0 < a->nb; b0 += CHUNK) {
    const int nb = (int)std::min<int64_t>(CHUNK, a->nb - b0);
    const size_t ncell = (size_t)nb * 64;
    amr_dump_pack_kernel<<<(int)std::min<size_t>((ncell + 255) / 256, AMR_GRID_SMS * 8), 256, 0, a->stream>>>(
        a->f[CUP2D_VEL], reinterpret_cast<const int2 *>(a->d_ij), a->d_h, (int)b0, nb, reinterpret_cast<float4 *>(d_buf), d_buf + nx);
    cudaMemcpyAsync(h_buf, d_buf, ncell * 8 * sizeof(float), cudaMemcpyDeviceToHost, a->stream);
    cudaMemcpyAsync(h_buf + nx, d_buf + nx, ncell * 3 * sizeof(float), cudaMemcpyDeviceToHost, a->stream);
    if (cudaStreamSynchronize(a->stream) != cudaSuccess) {
      rc = CUP2D_ECUDA;
      break;
    }
    const off_t cell0 = (off_t)((dist ? a->gbegin : 0) + b0) * 64;
    if (dump_write_all(fx, h_buf, ncell * 8 * sizeof(float), cell0 * 8 * (off_t)sizeof(float)) ||
        dump_write_all(fa, h_buf + nx, ncell * 3 * sizeof(float), cell0 * 3 * (off_t)sizeof(float)))
      rc = CUP2D_EINVAL;
  }
  if (fx >= 0) close(fx);
  if (fa >= 0) close(fa);
  cudaFreeHost(h_buf);
  cudaFree(d_buf);
  if (rc == CUP2D_EINVAL) set_error("cup2d_amr_dump: cannot write " + xyz_path + " / " + attr_path);
  if (rc == CUP2D_ECUDA) set_error(std::string("cup2d_amr_dump: ") + cudaGetErrorString(cudaGetLastError()));
  return rc;
}

} // extern "C"
