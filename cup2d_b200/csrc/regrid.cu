// Regridding input and field dump from device-resident data (SURVEY §8(f) rank 4).
//
//  * cup2d_adapt_tags:  what adapt() thresholds per block (main.cpp:4659-4689):
//      tmp = KernelVorticity(vel) (main.cpp:3343-3366), then GradChiOnTmp (main.cpp:4631-4656): a block that has
//      chi > 0 within `chi_cells` cells of it (corners included) gets its four centre cells set to 2 Rtol, then the
//      per-block L-inf.  Only nblocks doubles cross PCIe instead of the velocity and chi fields.
//  * cup2d_dump: the reference's dump() (main.cpp:3367-3467), same three files byte for byte: the float32 quad
//      corners and (u, v, 0) attributes are produced on the device in `infos` order and streamed through a pinned
//      staging buffer into the files (every rank writes its own byte range, as MPI_File_write_at_all does).
//      cup2d_amr_dump writes the same files from a multi-level mesh.
#include "rows.cuh"
#include "sim.h"
#include "amr.h"
#include <algorithm>
#include <cstdio>
#include <fcntl.h>
#include <string>
#include <unistd.h>

namespace cup2d {

constexpr int NT = 256;
constexpr int WPB = NT / 32;

// Body-proximity masks live in the first three 64-bit words of every block of the Krylov scratch vector kz (idle
// outside the Poisson solve and already peer-mapped, so the ordinary block halo pull moves them between GPUs):
//   word 0: bit (8*y + x) <-> chi(x, y) of this block is > 0 after the clamp of main.cpp:4644-4645
//   word 1 / 2: word 0 of the block's S / N neighbour (0 at a wall) — so that a block finds its DIAGONAL neighbours'
//   masks in its W / E neighbours' slots even when those are halo copies of another rank's blocks.
constexpr int MASK_STRIDE = 64; // 64-bit words per block of a scalar vector

__global__ void __launch_bounds__(NT)
chi_mask_kernel(const double *__restrict__ chi, unsigned long long *__restrict__ mask, int nrows) {
  __shared__ __align__(16) double s_scr[WPB * ROWS_SCRATCH];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double *sw = s_scr + warp * ROWS_SCRATCH;
  for (int row0 = (blockIdx.x * WPB + warp) * 32; row0 < nrows; row0 += gridDim.x * WPB * 32) {
    const int nv = min(32, nrows - row0);
    double c[8];
    rows_load1(chi, row0, nv, sw, lane, c);
    unsigned long long m = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) m |= (fmax(fmin(c[i], 1.0), 0.0) > 0.0) ? (1ull << i) : 0ull;
    m <<= 8 * (lane & 7);
    m |= __shfl_xor_sync(0xffffffffu, m, 1);
    m |= __shfl_xor_sync(0xffffffffu, m, 2);
    m |= __shfl_xor_sync(0xffffffffu, m, 4);
    if (lane < nv && (lane & 7) == 0) mask[(size_t)((row0 + lane) >> 3) * MASK_STRIDE] = m;
    __syncwarp();
  }
}

__global__ void __launch_bounds__(NT)
chi_mask_diag_kernel(unsigned long long *__restrict__ mask, const int4 *__restrict__ nbr, int nloc) {
  for (int k = blockIdx.x * NT + threadIdx.x; k < nloc; k += gridDim.x * NT) {
    const int4 nb = nbr[k];
    mask[(size_t)k * MASK_STRIDE + 1] = nb.z >= 0 ? mask[(size_t)nb.z * MASK_STRIDE] : 0ull;
    mask[(size_t)k * MASK_STRIDE + 2] = nb.w >= 0 ? mask[(size_t)nb.w * MASK_STRIDE] : 0ull;
  }
}

// parts of a block's 64-bit cell mask: the o columns / rows next to one of its edges
__device__ __forceinline__ unsigned long long cols_lo(int o) { return 0x0101010101010101ull * ((1ull << o) - 1ull); }
__device__ __forceinline__ unsigned long long cols_hi(int o) { return cols_lo(o) << (8 - o); }
__device__ __forceinline__ unsigned long long rows_lo(int o) { return o >= 8 ? ~0ull : (1ull << (8 * o)) - 1ull; }
__device__ __forceinline__ unsigned long long rows_hi(int o) { return rows_lo(o) << (8 * (8 - o)); }

// omega = (0.5/h) * (((u_S - u_N) + v_E) - v_W) with free-slip ghosts (tangential component copied at walls);
// CHI: additionally the body-proximity override.  One lane = one row of 8 cells, 8 lanes = one block.
template <bool CHI>
__global__ void __launch_bounds__(NT)
adapt_tag_kernel(const double *__restrict__ vel, double *__restrict__ tmp, double *__restrict__ linf,
                 const int4 *__restrict__ nbr, const unsigned long long *__restrict__ mask, int nrows,
                 double i2h, double two_rtol, int o) {
  __shared__ __align__(16) double s_scr[WPB * ROWS_SCRATCH];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double *sw = s_scr + warp * ROWS_SCRATCH;
  for (int row0 = (blockIdx.x * WPB + warp) * 32; row0 < nrows; row0 += gridDim.x * WPB * 32) {
    const int nv = min(32, nrows - row0);
    const int row = row0 + lane, slot = row >> 3, y = row & 7;
    const bool act = lane < nv;
    const int4 nb = act ? nbr[slot] : make_int4(-1, -1, -1, -1);
    double2 cv[8], c[8];
    chunk2_ld(vel, row0, nv, lane, cv);
    chunk2_to_rows(sw, nv, lane, cv, c);
    double w[8];
    if (act) {
      const double2 *f2 = reinterpret_cast<const double2 *>(vel);
      double un[8], us[8];
      double2 t[8];
      if (y < 7) rows_peek2(sw, lane + 1, t);
      else if (nb.w >= 0) grow_load2(vel, nb.w, 0, t);
      else {
#pragma unroll
        for (int i = 0; i < 8; i++) t[i] = c[i];
      }
#pragma unroll
      for (int i = 0; i < 8; i++) un[i] = t[i].x;
      if (y > 0) rows_peek2(sw, lane - 1, t);
      else if (nb.z >= 0) grow_load2(vel, nb.z, 7, t);
      else {
#pragma unroll
        for (int i = 0; i < 8; i++) t[i] = c[i];
      }
#pragma unroll
      for (int i = 0; i < 8; i++) us[i] = t[i].x;
      const double vW = nb.x >= 0 ? f2[(size_t)nb.x * 64 + y * 8 + 7].y : c[0].y;
      const double vE = nb.y >= 0 ? f2[(size_t)nb.y * 64 + y * 8 + 0].y : c[7].y;
#pragma unroll
      for (int i = 0; i < 8; i++) {
        const double e = i < 7 ? c[i + 1].y : vE, ww = i > 0 ? c[i - 1].y : vW;
        w[i] = i2h * (((us[i] - un[i]) + e) - ww);
      }
    } else {
#pragma unroll
      for (int i = 0; i < 8; i++) w[i] = 0.0;
    }
    if (CHI) {
      // lane y of a block looks at one of the 8 surrounding blocks (0..3 = W,E,S,N; 4..7 = SW,SE,NW,NE); the mask of
      // a diagonal block is word 1 (S) / 2 (N) of the W / E neighbour's slot.  Everyone adds the block's own mask.
      unsigned long long hit = 0;
      if (act) {
        hit = mask[(size_t)slot * MASK_STRIDE];
        const int src = y == 2 ? nb.z : y == 3 ? nb.w : (y & 1) ? nb.y : nb.x;
        if (src >= 0) {
          const int word = y < 4 ? 0 : (y < 6 ? 1 : 2);
          unsigned long long sel = ~0ull;
          if (y < 2 || y >= 4) sel &= (y & 1) ? cols_lo(o) : cols_hi(o); // E block: its first columns; W: its last
          if (y >= 2) sel &= (y == 2 || y == 4 || y == 5) ? rows_hi(o) : rows_lo(o); // S block: its top rows
          hit |= mask[(size_t)src * MASK_STRIDE + word] & sel;
        }
      }
      unsigned any = hit != 0ull;
      any |= __shfl_xor_sync(0xffffffffu, any, 1);
      any |= __shfl_xor_sync(0xffffffffu, any, 2);
      any |= __shfl_xor_sync(0xffffffffu, any, 4);
      if (any && (y == 3 || y == 4)) w[3] = w[4] = two_rtol; // TMP[3..4][3..4] = 2 Rtol (main.cpp:4647-4650)
    }
    double m = 0.0;
#pragma unroll
    for (int i = 0; i < 8; i++) m = fmax(m, fabs(w[i]));
    m = fmax(m, __shfl_xor_sync(0xffffffffu, m, 1));
    m = fmax(m, __shfl_xor_sync(0xffffffffu, m, 2));
    m = fmax(m, __shfl_xor_sync(0xffffffffu, m, 4));
    if (act && y == 0) linf[slot] = m;
    rows_store1(tmp, row0, nv, sw, lane, w);
  }
}

int launch_adapt_tags(cup2d_sim *s, double rtol, int chi_cells, double *linf_host) {
  if (s->nranks > 1) {
    int rc = halo_exchange_ptr(s, s->f[CUP2D_VEL], 2, CUP2D_VEL);
    if (rc) return rc;
  }
  if (!s->d_linf) CUP2D_CUDA(cudaMalloc(&s->d_linf, (size_t)s->nloc * sizeof(double)));
  const int nrows = (int)s->nloc * 8;
  const int grid = min((nrows + NT - 1) / NT, s->num_sms * 8);
  const int4 *nbr = reinterpret_cast<const int4 *>(s->d_nbr);
  ProfScope prof(s, KC_VORT);
  if (chi_cells > 0) {
    unsigned long long *mask = reinterpret_cast<unsigned long long *>(s->kz);
    int rc;
    chi_mask_kernel<<<grid, NT, 0, s->stream>>>(s->f[CUP2D_CHI], mask, nrows);
    if (s->nranks > 1 && (rc = halo_exchange_ptr(s, s->kz, 1, CUP2D_NFIELDS))) return rc;
    chi_mask_diag_kernel<<<min((int)((s->nloc + NT - 1) / NT), s->num_sms * 8), NT, 0, s->stream>>>(mask, nbr, (int)s->nloc);
    if (s->nranks > 1 && (rc = halo_exchange_ptr(s, s->kz, 1, CUP2D_NFIELDS))) return rc;
    adapt_tag_kernel<true><<<grid, NT, 0, s->stream>>>(s->f[CUP2D_VEL], s->f[CUP2D_TMP], s->d_linf, nbr, mask, nrows,
                                                       0.5 / s->h, 2.0 * rtol, chi_cells);
    s->launches += 3;
  } else {
    adapt_tag_kernel<false><<<grid, NT, 0, s->stream>>>(s->f[CUP2D_VEL], s->f[CUP2D_TMP], s->d_linf, nbr, nullptr,
                                                        nrows, 0.5 / s->h, 0.0, 0);
    s->launches++;
  }
  CUP2D_CUDA(cudaGetLastError());
  if (linf_host) {
    CUP2D_CUDA(cudaMemcpyAsync(linf_host, s->d_linf, (size_t)s->nloc * sizeof(double), cudaMemcpyDeviceToHost,
                               s->stream));
    CUP2D_CUDA(cudaStreamSynchronize(s->stream));
  }
  return CUP2D_OK;
}

// ------------------------------------------------------------------------------------------------
// dump(): one thread per cell of blocks [b0, b0+nb): 8 floats of quad corners + 3 floats of attribute
// (main.cpp:3431-3452).  origin = i*8*h0/2^level (main.cpp:695-696) = (8 i) h exactly (power-of-two scaling);
// no FMA contraction anywhere so that the doubles, and hence the narrowed floats, are the reference's.  The cell size
// of block id is hb[id] on a multi-level mesh (hb != nullptr), h on the uniform grid.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
dump_pack_kernel(const double *__restrict__ vel, const int2 *__restrict__ ij, const double *__restrict__ hb, double h,
                 int b0, int nb, float4 *__restrict__ xyz, float *__restrict__ attr) {
  const size_t ncell = (size_t)nb * 64;
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < ncell; i += (size_t)gridDim.x * 256) {
    const int k = (int)(i >> 6), x = (int)(i & 7), y = (int)((i >> 3) & 7);
    const int2 b = ij[b0 + k];
    const double hk = hb ? hb[b0 + k] : h;
    const double u0 = __dadd_rn(__dmul_rn((double)(b.x * CUP2D_BS), hk), __dmul_rn(hk, (double)x));
    const double v0 = __dadd_rn(__dmul_rn((double)(b.y * CUP2D_BS), hk), __dmul_rn(hk, (double)y));
    const float fu0 = (float)u0, fv0 = (float)v0, fu1 = (float)__dadd_rn(u0, hk), fv1 = (float)__dadd_rn(v0, hk);
    xyz[2 * i] = make_float4(fu0, fv0, fu0, fv1);
    xyz[2 * i + 1] = make_float4(fu1, fv1, fu1, fv0);
    const double2 q = reinterpret_cast<const double2 *>(vel)[(size_t)(b0 + k) * 64 + (i & 63)];
    attr[3 * i] = (float)q.x;
    attr[3 * i + 1] = (float)q.y;
    attr[3 * i + 2] = 0.0f;
  }
}

static int dump_write_all(int fd, const void *buf, size_t n, off_t off) {
  const char *p = static_cast<const char *>(buf);
  while (n > 0) {
    const ssize_t w = pwrite(fd, p, n, off);
    if (w <= 0) return -1;
    p += w;
    off += w;
    n -= (size_t)w;
  }
  return 0;
}

// the .xdmf2 descriptor of dump() (main.cpp:3380-3423), byte for byte
static int dump_write_xdmf(const std::string &xdmf_path, const std::string &xyz_path, const std::string &attr_path, double time,
                           long ncell_total) {
  auto basename_of = [](const std::string &p) { // main.cpp:3380-3385: after the last '/' that is not the final char
    size_t cut = 0;
    for (size_t j = 0; j + 1 < p.size(); j++)
      if (p[j] == '/') cut = j + 1;
    return p.substr(cut);
  };
  FILE *xmf = fopen(xdmf_path.c_str(), "w");
  if (!xmf) {
    set_error("dump: cannot open " + xdmf_path);
    return CUP2D_EINVAL;
  }
  fprintf(xmf,
          "<Xdmf\n    Version=\"2.0\">\n  <Domain>\n    <Grid>\n      <Time Value=\"%.16e\"/>\n      <Topology\n"
          "          Dimensions=\"%ld\"\n          TopologyType=\"Quadrilateral\"/>\n     <Geometry\n"
          "         GeometryType=\"XY\">\n       <DataItem\n           Dimensions=\"%ld 2\"\n"
          "           Format=\"Binary\">\n         %s\n       </DataItem>\n     </Geometry>\n       <Attribute\n"
          "           AttributeType=\"Vector\"\n           Name=\"vort\"\n           Center=\"Cell\">\n"
          "         <DataItem\n             Dimensions=\"3 %ld\"\n             Format=\"Binary\">\n           %s\n"
          "         </DataItem>\n       </Attribute>\n    </Grid>\n  </Domain>\n</Xdmf>\n",
          time, ncell_total, 4 * ncell_total, basename_of(xyz_path).c_str(), ncell_total, basename_of(attr_path).c_str());
  fclose(xmf);
  return CUP2D_OK;
}

// dump()'s three files path.xdmf2 / .xyz.raw / .attr.raw of the velocity `vel` of nb blocks, which are blocks
// [gbegin, gbegin + nb) of the nglobal blocks of the whole mesh: every rank writes its own byte range, as
// MPI_File_write_at_all does, and one of them (write_xdmf) the descriptor (main.cpp:3387-3390).  ij: (i, j) per block;
// hb / h: the cell size as in dump_pack_kernel; oflags: open() flags of the two raw files; grid_cap: the pack kernel's
// grid cap; who: the prefix of the error messages; launches (may be null): counts the pack kernel launches.
static int dump_write(cudaStream_t stream, const double *vel, const int *ij, const double *hb, double h, int64_t nb,
                      int64_t gbegin, int64_t nglobal, bool write_xdmf, int oflags, int grid_cap, const char *who,
                      double time, const char *path, int64_t *launches) {
  const std::string base(path);
  const std::string xyz_path = base + ".xyz.raw", attr_path = base + ".attr.raw", xdmf_path = base + ".xdmf2";
  if (write_xdmf) {
    const int rc = dump_write_xdmf(xdmf_path, xyz_path, attr_path, time, (long)nglobal * 64);
    if (rc) return rc;
  }
  // staging: CHUNK blocks at a time, device + pinned host (44 B per cell)
  const int CHUNK = (int)std::min<int64_t>(nb, 16384);
  const size_t nx = (size_t)CHUNK * 64 * 8, na = (size_t)CHUNK * 64 * 3;
  float *d_buf = nullptr, *h_buf = nullptr;
  CUP2D_CUDA(cudaMalloc(&d_buf, (nx + na) * sizeof(float)));
  if (cudaMallocHost(&h_buf, (nx + na) * sizeof(float)) != cudaSuccess) {
    cudaFree(d_buf);
    set_error(std::string(who) + ": cannot allocate the pinned staging buffer");
    return CUP2D_ECUDA;
  }
  const int fx = open(xyz_path.c_str(), oflags, 0644), fa = open(attr_path.c_str(), oflags, 0644);
  int rc = (fx < 0 || fa < 0) ? CUP2D_EINVAL : CUP2D_OK;
  for (int64_t b0 = 0; rc == CUP2D_OK && b0 < nb; b0 += CHUNK) {
    const int n = (int)std::min<int64_t>(CHUNK, nb - b0);
    const size_t ncell = (size_t)n * 64;
    dump_pack_kernel<<<(int)std::min<size_t>((ncell + 255) / 256, grid_cap), 256, 0, stream>>>(
        vel, reinterpret_cast<const int2 *>(ij), hb, h, (int)b0, n, reinterpret_cast<float4 *>(d_buf), d_buf + nx);
    if (launches) ++*launches;
    cudaMemcpyAsync(h_buf, d_buf, ncell * 8 * sizeof(float), cudaMemcpyDeviceToHost, stream);
    cudaMemcpyAsync(h_buf + nx, d_buf + nx, ncell * 3 * sizeof(float), cudaMemcpyDeviceToHost, stream);
    if (cudaStreamSynchronize(stream) != cudaSuccess) {
      rc = CUP2D_ECUDA;
      break;
    }
    const off_t cell0 = (off_t)(gbegin + b0) * 64; // MPI_Exscan offset (main.cpp:3387) + position in the range
    if (dump_write_all(fx, h_buf, ncell * 8 * sizeof(float), cell0 * 8 * (off_t)sizeof(float)) ||
        dump_write_all(fa, h_buf + nx, ncell * 3 * sizeof(float), cell0 * 3 * (off_t)sizeof(float)))
      rc = CUP2D_EINVAL;
  }
  if (fx >= 0) close(fx);
  if (fa >= 0) close(fa);
  cudaFreeHost(h_buf);
  cudaFree(d_buf);
  if (rc == CUP2D_EINVAL) set_error(std::string(who) + ": cannot write " + xyz_path + " / " + attr_path);
  if (rc == CUP2D_ECUDA) set_error(std::string(who) + ": " + cudaGetErrorString(cudaGetLastError()));
  return rc;
}

int dump_fields(cup2d_sim *s, double time, const char *path) {
  const int rc = ensure_block_ij(s);
  if (rc) return rc;
  // main.cpp:3390: the last rank writes the descriptor; the files are not truncated
  return dump_write(s->stream, s->f[CUP2D_VEL], s->d_ij, nullptr, s->h, s->nloc, s->gbegin, s->nglobal,
                    s->rank == s->nranks - 1, O_CREAT | O_WRONLY, s->num_sms * 8, "dump", time, path, &s->launches);
}

} // namespace cup2d

/* dump() of the velocity on a multi-level mesh (main.cpp:3367-3467): the three files of cup2d_dump, byte for byte, with
 * the cell size of every block its own */
extern "C" int cup2d_amr_dump(cup2d_amr *a, double time, const char *path) {
  CUP2D_REQUIRE(a != nullptr && path && *path, "cup2d_amr_dump: bad arguments");
  CUP2D_CUDA(cudaSetDevice(a->device));
  const int rc = amr_ensure_ij(a);
  if (rc) return rc;
  const bool dist = a->dist && a->nranks > 1; // every rank writes its own byte range, the last one the descriptor
  return cup2d::dump_write(a->stream, a->f[CUP2D_VEL], a->d_ij, a->d_h, 0, a->nb, a->gbegin, a->nglobal,
                           !dist || a->rank == a->nranks - 1, O_CREAT | O_WRONLY | (dist ? 0 : O_TRUNC),
                           cup2d::AMR_GRID_SMS * 8, "cup2d_amr_dump", time, path, nullptr);
}
