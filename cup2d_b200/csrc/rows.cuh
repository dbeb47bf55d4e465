// Warp-cooperative row access for the block-structured kernels.
//
// Compute mapping ("row layout"): one lane owns one row of 8 cells of one 8x8 block (8 lanes = one
// block, one warp = 4 consecutive blocks = 32 rows = one CHUNK of 2 KB (scalar) / 4 KB (vector) of
// CONTIGUOUS memory).  If every lane read its own row with 128-bit loads, each load instruction would
// touch 16-32 different 128-B lines and the kernels become L1/TEX-bound.  So global memory is only ever touched in "chunk layout": lane
// l holds the 16-byte pieces j*32+l (j = 0..3) of the chunk, i.e. fully coalesced 128-bit accesses.
// Element-wise work (axpy, dots, norms) is done directly in chunk layout; only stencils and the block
// preconditioner need row layout, and the two layouts are converted through a per-warp shared-memory
// scratch.  The scratch is unpadded and XOR-swizzled: piece p of row r lives at 16-byte slot
// 4r + (p ^ ((r>>1)&3)), which is bank-conflict-free both for the coalesced side (8 lanes = 2 rows x 4
// pieces) and for the row side (8 lanes = 8 consecutive rows, same piece).
#pragma once
#include "common.cuh"

namespace cup2d {

constexpr int RS2 = 9;                     // vector row stride in double2 (8 used + 1 pad = 144 B)
constexpr int ROWS_SCRATCH = 32 * RS2 * 2; // doubles per warp for kernels that touch vector fields
constexpr int SCR1 = 288;                  // doubles per warp for scalar-only kernels (preconditioner: 4*72)
constexpr int SCR_COOP = 320;              // rows_lap_coop: 256 for the chunk + 64 for the staged edge rows
#ifndef CUP2D_ROWS_COOP
#define CUP2D_ROWS_COOP 1 // 0: the SpMV kernels use the plain rows_lap_c as well (measurement variant)
#endif

__device__ __forceinline__ int swz(int r, int p) { return r * 4 + (p ^ ((r >> 1) & 3)); }

// ---- chunk layout <-> global ------------------------------------------------------------------
__device__ __forceinline__ void chunk_ld(const double *__restrict__ f, int row0, int nvalid, int lane,
                                         double2 (&c)[4]) {
  const double2 *src = reinterpret_cast<const double2 *>(f) + (size_t)row0 * 4;
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int i = j * 32 + lane;
    c[j] = (i >> 2) < nvalid ? src[i] : make_double2(0.0, 0.0);
  }
}
__device__ __forceinline__ void chunk_st(double *__restrict__ f, int row0, int nvalid, int lane,
                                         const double2 (&c)[4]) {
  double2 *dst = reinterpret_cast<double2 *>(f) + (size_t)row0 * 4;
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int i = j * 32 + lane;
    if ((i >> 2) < nvalid) dst[i] = c[j];
  }
}
// ---- chunk layout <-> row layout through the scratch -----------------------------------------------
// after chunk_to_rows the whole chunk stays parked in the scratch (rows_peek1 may read other rows)
__device__ __forceinline__ void chunk_to_rows(double *sw, int lane, const double2 (&c)[4], double (&r)[8]) {
  double2 *s2 = reinterpret_cast<double2 *>(sw);
  __syncwarp();
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int i = j * 32 + lane;
    s2[swz(i >> 2, i & 3)] = c[j];
  }
  __syncwarp();
#pragma unroll
  for (int p = 0; p < 4; p++) {
    const double2 v = s2[swz(lane, p)];
    r[2 * p] = v.x;
    r[2 * p + 1] = v.y;
  }
}
__device__ __forceinline__ void rows_to_chunk(double *sw, int lane, const double (&r)[8], double2 (&c)[4]) {
  double2 *s2 = reinterpret_cast<double2 *>(sw);
  __syncwarp();
#pragma unroll
  for (int p = 0; p < 4; p++) s2[swz(lane, p)] = make_double2(r[2 * p], r[2 * p + 1]);
  __syncwarp();
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int i = j * 32 + lane;
    c[j] = s2[swz(i >> 2, i & 3)];
  }
}
__device__ __forceinline__ void rows_peek1(const double *sw, int r, double (&c)[8]) {
  const double2 *s2 = reinterpret_cast<const double2 *>(sw);
#pragma unroll
  for (int p = 0; p < 4; p++) {
    const double2 v = s2[swz(r, p)];
    c[2 * p] = v.x;
    c[2 * p + 1] = v.y;
  }
}
// convenience: rows [row0, row0+nvalid) of a scalar field -> lane l gets row row0+l (zeros beyond)
__device__ __forceinline__ void rows_load1(const double *__restrict__ f, int row0, int nvalid,
                                           double *sw, int lane, double (&c)[8]) {
  double2 t[4];
  chunk_ld(f, row0, nvalid, lane, t);
  chunk_to_rows(sw, lane, t, c);
}
__device__ __forceinline__ void rows_store1(double *__restrict__ f, int row0, int nvalid, double *sw,
                                            int lane, const double (&c)[8]) {
  double2 t[4];
  rows_to_chunk(sw, lane, c, t);
  chunk_st(f, row0, nvalid, lane, t);
}

// ---- vector field (u,v interleaved): lane l gets row row0+l as 8 double2 (padded scratch) -----------
// chunk layout of a vector field: lane l holds pieces j*32+l, j = 0..7 (4 KB per warp, coalesced)
__device__ __forceinline__ void chunk2_ld(const double *__restrict__ f, int row0, int nvalid, int lane,
                                          double2 (&c)[8]) {
  const double2 *src = reinterpret_cast<const double2 *>(f) + (size_t)row0 * 8;
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const int i = j * 32 + lane;
    c[j] = (i >> 3) < nvalid ? src[i] : make_double2(0.0, 0.0);
  }
}
__device__ __forceinline__ void chunk2_st(double *__restrict__ f, int row0, int nvalid, int lane,
                                          const double2 (&c)[8]) {
  double2 *dst = reinterpret_cast<double2 *>(f) + (size_t)row0 * 8;
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const int i = j * 32 + lane;
    if ((i >> 3) < nvalid) dst[i] = c[j];
  }
}
__device__ __forceinline__ void chunk2_to_rows(double *sw, int nvalid, int lane, const double2 (&t)[8],
                                               double2 (&c)[8]) {
  double2 *s2 = reinterpret_cast<double2 *>(sw);
  __syncwarp();
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const int i = j * 32 + lane;
    s2[(i >> 3) * RS2 + (i & 7)] = t[j];
  }
  __syncwarp();
  if (lane < nvalid) {
#pragma unroll
    for (int p = 0; p < 8; p++) c[p] = s2[lane * RS2 + p];
  } else {
#pragma unroll
    for (int p = 0; p < 8; p++) c[p] = make_double2(0.0, 0.0);
  }
}
__device__ __forceinline__ void rows2_to_chunk(double *sw, int lane, const double2 (&c)[8], double2 (&t)[8]) {
  double2 *s2 = reinterpret_cast<double2 *>(sw);
  __syncwarp();
#pragma unroll
  for (int p = 0; p < 8; p++) s2[lane * RS2 + p] = c[p];
  __syncwarp();
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const int i = j * 32 + lane;
    t[j] = s2[(i >> 3) * RS2 + (i & 7)];
  }
}
__device__ __forceinline__ void rows_load2(const double *__restrict__ f, int row0, int nvalid,
                                           double *sw, int lane, double2 (&c)[8]) {
  const double2 *src = reinterpret_cast<const double2 *>(f) + (size_t)row0 * 8;
  double2 *s2 = reinterpret_cast<double2 *>(sw);
  __syncwarp();
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const int i = j * 32 + lane;
    if ((i >> 3) < nvalid) s2[(i >> 3) * RS2 + (i & 7)] = src[i];
  }
  __syncwarp();
  if (lane < nvalid) {
#pragma unroll
    for (int p = 0; p < 8; p++) c[p] = s2[lane * RS2 + p];
  } else {
#pragma unroll
    for (int p = 0; p < 8; p++) c[p] = make_double2(0.0, 0.0);
  }
}
__device__ __forceinline__ void rows_peek2(const double *sw, int r, double2 (&c)[8]) {
  const double2 *s2 = reinterpret_cast<const double2 *>(sw);
#pragma unroll
  for (int p = 0; p < 8; p++) c[p] = s2[r * RS2 + p];
}
__device__ __forceinline__ void rows_store2(double *__restrict__ f, int row0, int nvalid, double *sw,
                                            int lane, const double2 (&c)[8]) {
  double2 *dst = reinterpret_cast<double2 *>(f) + (size_t)row0 * 8;
  double2 *s2 = reinterpret_cast<double2 *>(sw);
  __syncwarp();
#pragma unroll
  for (int p = 0; p < 8; p++) s2[lane * RS2 + p] = c[p];
  __syncwarp();
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const int i = j * 32 + lane;
    if ((i >> 3) < nvalid) dst[i] = s2[(i >> 3) * RS2 + (i & 7)];
  }
}
// plain per-lane global row access (used only by the few lanes that touch a NEIGHBOUR block's edge row)
__device__ __forceinline__ void grow_load1(const double *__restrict__ f, int slot, int y, double (&c)[8]) {
  const double2 *p = reinterpret_cast<const double2 *>(f + (size_t)slot * 64 + y * 8);
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const double2 v = p[k];
    c[2 * k] = v.x;
    c[2 * k + 1] = v.y;
  }
}
__device__ __forceinline__ void grow_load2(const double *__restrict__ f, int slot, int y, double2 (&c)[8]) {
  const double2 *p = reinterpret_cast<const double2 *>(f + (size_t)slot * 128 + y * 16);
#pragma unroll
  for (int k = 0; k < 8; k++) c[k] = p[k];
}

// Rows of the Poisson matrix that are NOT the same-level 5-point stencil (coarse-fine interpolation rows
// of main.cpp:5915-5997 pushed through cooPushBackRow; SURVEY.md §8(f) rank 1).  They live in a small
// CSR side table and override the stencil result of the cells they belong to: blk[slot] = -1 (block is
// fully regular) or k, tab[k*64 + cell] = -1 or the CSR row index.
struct IrrView {
  const int *blk = nullptr;
  const int *tab = nullptr;
  const int *rowptr = nullptr;
  const int *col = nullptr;
  const double *val = nullptr;
};

// Neighbour rows that live in HALO slots (slot >= nloc) of a multi-rank context.  In the Krylov loop the producing
// kernel of a vector pushes its perimeter rows straight into the neighbours' halo slots over NVLink and raises a flag
// (poisson.cu: push_rows / push_finish); the consuming stencil kernel waits for the flags of the ranks it has halo
// blocks of — lazily, only in the lanes that touch a halo slot, so that interior rows never wait — and then reads the
// slots with coherent loads (the data arrived while this kernel was running).
struct NoGate {
  static constexpr bool on = false;
  int nloc = 0;
  __device__ __forceinline__ void wait() const {}
};
struct HaloGate {
  static constexpr bool on = true;
  int nloc;                  // slots >= nloc are halo slots
  unsigned mask;             // ranks this rank has halo blocks of
  unsigned long long target; // push epoch the flags must have reached
  Comm comm;
  __device__ __forceinline__ void wait() const {
    const unsigned long long *mine = comm.mb[comm.rank];
    for (int r = 0; r < comm.nranks; r++)
      if ((mask >> r) & 1u) wait_flag(mine + MB_PUSHED + r, target, comm, CW_PUSHED, r);
  }
};
template <class G> __device__ __forceinline__ double nb_ld1(const double *z, int slot, int off, const G &g) {
  const double *p = z + (size_t)slot * 64 + off;
  if (G::on && slot >= g.nloc) return ld_coherent(p);
  return *p;
}
template <class G> __device__ __forceinline__ void nb_row1(const double *z, int slot, int y, double (&c)[8], const G &g) {
  const double2 *p = reinterpret_cast<const double2 *>(z + (size_t)slot * 64 + y * 8);
  const bool halo = G::on && slot >= g.nloc;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const double2 v = halo ? ld_coherent2(p + k) : p[k];
    c[2 * k] = v.x;
    c[2 * k + 1] = v.y;
  }
}

// Undivided 5-point Laplacian rows of a scalar field for the warp's 32 rows, ghost = the cell itself at
// a domain wall (Neumann rows of main.cpp:7100-7107 / ScalarLab::Neumann2D main.cpp:3210-3245).
// Returns the own row in c and the Laplacian in out.  Summation order S,W,E,N then -4C.
// rows_lap_c: the caller already holds the chunk of z (so that other global loads can be in flight too)
template <class G = NoGate>
__device__ __forceinline__ void rows_lap_c(const double2 (&cz)[4], const double *__restrict__ z, int row0,
                                           int nvalid, const int4 *__restrict__ nbr, double *sw, int lane,
                                           double (&c)[8], double (&out)[8], const IrrView irr = IrrView(),
                                           const G gate = G());
__device__ __forceinline__ void rows_lap(const double *__restrict__ z, int row0, int nvalid,
                                         const int4 *__restrict__ nbr, double *sw, int lane,
                                         double (&c)[8], double (&out)[8], const IrrView irr = IrrView()) {
  double2 cz[4];
  chunk_ld(z, row0, nvalid, lane, cz);
  rows_lap_c(cz, z, row0, nvalid, nbr, sw, lane, c, out, irr);
}
// ---- rows_lap_coop: the variant the SpMV kernels use (k_init and the right-hand-side kernel, with their higher register
// pressure, keep the plain form below) ----
// The L1 data pipe (shared-memory and global-load wavefronts together) bounds the stencil kernels about as much as DRAM
// does, and the neighbour accesses are most of its global part.  So:
//  * the edge rows of the S/N neighbour blocks come in with ONE warp-wide 128-bit load: lanes 0..15 fetch the four 16-byte
//    pieces of row 0 of the N neighbour of each of the warp's four blocks, lanes 16..31 row 7 of the S neighbours (8 wavefronts
//    instead of 32 for eight quarter-empty per-lane loads); the pieces are staged behind the chunk in the scratch;
//  * every lane then reads the rows above and below through (base, swizzle key) pairs — the neighbouring lane's row of the
//    chunk, a staged edge row, or its own row at a wall (Neumann: ghost = own cell) — piece by piece, with no arrays and
//    no branches in the stencil loop;
//  * a W/E ghost cell whose block belongs to the warp's own chunk (in Hilbert order four consecutive, 4-aligned blocks form
//    a 2x2 square, so one of the two does) is read from the scratch.
template <class G>
__device__ __forceinline__ void rows_lap_coop(const double2 (&cz)[4], const double *__restrict__ z, int row0,
                                              int nvalid, const int4 *__restrict__ nbr, double *sw, int lane,
                                              double (&c)[8], double (&out)[8], const IrrView irr, const G gate) {
  const int row = row0 + lane, slot = row >> 3, y = row & 7;
  const int4 nb = lane < nvalid ? nbr[slot] : make_int4(-1, -1, -1, -1);
  // staging rows behind the chunk: row 2b = N edge row of block b (pieces in place), row 2b+1 = S edge row of block b
  // (piece p at p ^ 3): exactly the 16-byte bank groups the chunk rows 8b+8 / 8b-1 would occupy, so an edge lane's reads
  // stay conflict-free with the reads of the seven other lanes of its quarter warp
  double2 *stage = reinterpret_cast<double2 *>(sw + 256);
  {
    const int b = (lane >> 2) & 3, piece = lane & 3;
    const int nbN = __shfl_sync(0xffffffffu, nb.w, 8 * b), nbS = __shfl_sync(0xffffffffu, nb.z, 8 * b);
    const int src = lane < 16 ? nbN : nbS;
    double2 v = make_double2(0.0, 0.0);
    if (src >= 0) {
      const bool halo = G::on && src >= gate.nloc;
      if (halo) gate.wait();
      const double2 *p = reinterpret_cast<const double2 *>(z + (size_t)src * 64 + (lane < 16 ? 0 : 56)) + piece;
      v = halo ? ld_coherent2(p) : *p;
    }
    __syncwarp(); // the previous user of the scratch is done with it
    stage[lane < 16 ? 8 * b + piece : 8 * b + 4 + (piece ^ 3)] = v;
  }
  chunk_to_rows(sw, lane, cz, c); // (its barriers also publish the staged rows)
  if (lane < nvalid) {
    if (G::on) { // pushed halo rows: wait (once, only here) for the ranks that own them
      if (nb.x >= gate.nloc || nb.y >= gate.nloc) gate.wait();
    }
    const double2 *s2 = reinterpret_cast<const double2 *>(sw);
    const int own_key = (lane >> 1) & 3;
    // rows above / below: (base, key) with piece k at base[k ^ key]
    const double2 *bu = y < 7 ? s2 + (lane + 1) * 4 : (nb.w >= 0 ? stage + (lane >> 3) * 8 : s2 + lane * 4);
    const int ku = y < 7 ? ((lane + 1) >> 1) & 3 : (nb.w >= 0 ? 0 : own_key);
    const double2 *bd = y > 0 ? s2 + (lane - 1) * 4 : (nb.z >= 0 ? stage + (lane >> 3) * 8 + 4 : s2 + lane * 4);
    const int kd = y > 0 ? ((lane - 1) >> 1) & 3 : (nb.z >= 0 ? 3 : own_key);
    const int s0 = row0 >> 3;
    const unsigned nblk = (unsigned)((nvalid + 7) >> 3), lW = (unsigned)(nb.x - s0), lE = (unsigned)(nb.y - s0);
    const double gW = lW < nblk ? s2[swz((int)lW * 8 + y, 3)].y : (nb.x >= 0 ? nb_ld1(z, nb.x, y * 8 + 7, gate) : c[0]);
    const double gE = lE < nblk ? s2[swz((int)lE * 8 + y, 0)].x : (nb.y >= 0 ? nb_ld1(z, nb.y, y * 8 + 0, gate) : c[7]);
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const double2 u = bu[k ^ ku], d = bd[k ^ kd];
      const int i = 2 * k;
      const double w0 = i > 0 ? c[i - 1] : gW, e1 = i + 1 < 7 ? c[i + 2] : gE;
      out[i] = (((d.x + w0) + c[i + 1]) + u.x) - 4.0 * c[i];         // summation order S,W,E,N then -4C
      out[i + 1] = (((d.y + c[i]) + e1) + u.y) - 4.0 * c[i + 1];
    }
    if (irr.blk) { // general rows override the stencil (rare: block faces at coarse-fine interfaces)
      const int k = irr.blk[slot];
      if (k >= 0) {
#pragma unroll
        for (int i = 0; i < 8; i++) {
          const int idx = irr.tab[k * 64 + y * 8 + i];
          if (idx >= 0) {
            double acc = 0.0;
            for (int j = irr.rowptr[idx]; j < irr.rowptr[idx + 1]; j++) {
              const int cj = irr.col[j];
              acc = fma(irr.val[j], (G::on && cj >= gate.nloc * 64) ? ld_coherent(z + cj) : z[cj], acc);
            }
            out[i] = acc;
          }
        }
      }
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; i++) out[i] = 0.0;
  }
}

template <class G>
__device__ __forceinline__ void rows_lap_c(const double2 (&cz)[4], const double *__restrict__ z, int row0,
                                           int nvalid, const int4 *__restrict__ nbr, double *sw, int lane,
                                           double (&c)[8], double (&out)[8], const IrrView irr, const G gate) {
  chunk_to_rows(sw, lane, cz, c);
  const int row = row0 + lane, slot = row >> 3, y = row & 7;
  if (lane < nvalid) {
    const int4 nb = nbr[slot];
    if (G::on) { // pushed halo rows: wait (once, only here) for the ranks that own them
      if (nb.x >= gate.nloc || nb.y >= gate.nloc || (y == 7 && nb.w >= gate.nloc) || (y == 0 && nb.z >= gate.nloc)) gate.wait();
    }
    double up[8], dn[8];
    if (y < 7) rows_peek1(sw, lane + 1, up);
    else if (nb.w >= 0) nb_row1(z, nb.w, 0, up, gate);
    else {
#pragma unroll
      for (int i = 0; i < 8; i++) up[i] = c[i];
    }
    if (y > 0) rows_peek1(sw, lane - 1, dn);
    else if (nb.z >= 0) nb_row1(z, nb.z, 7, dn, gate);
    else {
#pragma unroll
      for (int i = 0; i < 8; i++) dn[i] = c[i];
    }
    const double gW = nb.x >= 0 ? nb_ld1(z, nb.x, y * 8 + 7, gate) : c[0];
    const double gE = nb.y >= 0 ? nb_ld1(z, nb.y, y * 8 + 0, gate) : c[7];
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const double e = i < 7 ? c[i + 1] : gE;
      const double w = i > 0 ? c[i - 1] : gW;
      out[i] = (((dn[i] + w) + e) + up[i]) - 4.0 * c[i];
    }
    if (irr.blk) { // general rows override the stencil (rare: block faces at coarse-fine interfaces)
      const int k = irr.blk[slot];
      if (k >= 0) {
#pragma unroll
        for (int i = 0; i < 8; i++) {
          const int idx = irr.tab[k * 64 + y * 8 + i];
          if (idx >= 0) {
            double acc = 0.0;
            for (int j = irr.rowptr[idx]; j < irr.rowptr[idx + 1]; j++) {
              const int cj = irr.col[j];
              acc = fma(irr.val[j], (G::on && cj >= gate.nloc * 64) ? ld_coherent(z + cj) : z[cj], acc);
            }
            out[i] = acc;
          }
        }
      }
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; i++) out[i] = 0.0;
  }
}
} // namespace cup2d
