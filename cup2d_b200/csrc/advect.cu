// Fused advection-diffusion RK stage:  out = old + coef * K(in) / h^2
//
// K is the reference's KernelAdvectDiffuse (main.cpp:5441-5503): WENO5 upwind differences
// (main.cpp:162-208) of both velocity components + 5-point diffusion, undivided.  The Lab assembly
// (BlockLab::load, main.cpp:2270-2440) and the free-slip ghost fill (VectorLab::applyBCface,
// main.cpp:3131-3154) become the tile loader of this kernel; the RK update loops
// (main.cpp:6618-6626, 6634-6642) are fused into the store.
//
// One CTA = one tile of 4x4 blocks (32x32 cells), 128 threads.  Data path (round 2: no staging buffer, no repack):
//   HBM --16-byte cp.async (SASS LDGSTS), one per cell, lanes along the 8 cells = 128 contiguous bytes of a block row; 11-13
//        per thread, no registers in between (build option: one cp.async.bulk per block row on an mbarrier, CUP2D_ADV_LDGSTS=0)-->
//        the padded (u,v)-interleaved plane P[38][39] (3-cell ghost ring, row stride odd in 16-byte units), every cell exactly
//        where the stencil reads it
//   x pass: warp = the 8 rows of its block row, lane = (8-cell segment, row): 128-bit conflict-free LDS -> partial results R
//   y pass: lane = column, warp = the same block row: reads only what ITS OWN warp wrote to R (__syncwarp, no CTA barrier
//        between the passes), + old, 128-bit coalesced stores
//   per line of 8 cells: all advected one way -> branch-free upwind core (mirrored line if from the right), else general core
// Wall ghosts exist only in the perimeter tiles of the domain and are synthesised there after the copies landed.
//
// Arithmetic: all FP64; this kernel is bound by the FP64 pipe, not by HBM — see weno.cuh for the algebra that brings a
// flux down to 10 FP64 instructions and DESIGN.md 3.1 for the instruction budget per cell.
#include "sim.h"
#include "weno.cuh"
#include <vector>

namespace cup2d {

#ifndef CUP2D_ADV_CTAS
#define CUP2D_ADV_CTAS 4 // resident CTAs per SM the register allocation is bounded for (shared memory allows 5)
#endif
#ifndef CUP2D_ADV_LDGSTS
// 1: the tile is filled by 16-byte cp.async (SASS LDGSTS) issued by all threads, 13 per thread;  0: by per-row bulk copies
// (SASS UBLKCP + mbarrier).  A bulk copy issued by a divergent thread costs ~8 warp instructions (ELECT/R2UR loop over the
// lanes) and a tile needs 216 of them, which makes the bulk-copy fill the slower one.
#define CUP2D_ADV_LDGSTS 1
#endif

#ifndef CUP2D_ADV_SPECIALIZE
#define CUP2D_ADV_SPECIALIZE 1 // 1: the x and the y pass get their own copy of the line code; 0: one copy with run-time strides
#endif
#ifndef CUP2D_ADV_FASTPATH
#define CUP2D_ADV_FASTPATH 1 // 0: every line goes through the general core (measurement variant)
#endif

constexpr int TC = 32;          // tile cells per side
constexpr int GH = 3;           // ghost width (stencil -3..+3, main.cpp:5442)
constexpr int TW = TC + 2 * GH; // 38
constexpr int PS = 39;          // plane row stride in cells (16-byte units; odd: conflict-free for lanes along y)
constexpr int RS = 33;          // partial-result plane stride
constexpr int NT_ADV = 128;
constexpr int OFF_P = 0;
constexpr int OFF_R = OFF_P + TW * PS * 16;
constexpr int OFF_BAR = OFF_R + TC * RS * 16;
constexpr int OFF_SLOTS = OFF_BAR + 16;
constexpr int ADV_SMEM = OFF_SLOTS + TILE_SLOTS * 4; // 39.8 KB

#if CUP2D_ADV_LDGSTS
__device__ __forceinline__ void ldgsts16(void *smem_dst, const void *gmem_src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void ldgsts_wait_all() {
  asm volatile("cp.async.wait_all;" ::: "memory");
}
#endif

// MODE 0: out = tot (raw K, undivided)   1: old == in (stage 1)   2: old is a separate field (stage 2)
// The compiler specialises the fully unrolled line code for each of the two passes (immediate shared-memory offsets, no
// selects): 2350 instructions for both copies together, about what round 1's single run-time-strided copy took.
// DEVFAC: the dt-dependent factors come from device memory (StepFactors, written by k_step_factors) instead of the
// by-value arguments, so that a time step captured in a CUDA graph needs no host-supplied dt.
template <int MODE, bool DEVFAC>
__global__ void __launch_bounds__(NT_ADV, CUP2D_ADV_CTAS)
advect_stage_kernel(const double *__restrict__ in, const double *__restrict__ old,
                    double *__restrict__ out, const int *__restrict__ tiles,
                    const int *__restrict__ tile_org, int nbx, int nby,
                    int nloc, double afac_arg, double dfac_arg, double ofac, const StepFactors *__restrict__ sf) {
  // the line core delivers 3 x the upwind differences: the third goes into the advection factor
  const double afac3 = (DEVFAC ? sf->afac : afac_arg) * (1.0 / 3.0), dfac = DEVFAC ? sf->dfac : dfac_arg;
  extern __shared__ __align__(128) unsigned char smem[];
  double2 *P = reinterpret_cast<double2 *>(smem + OFF_P);
  double2 *R = reinterpret_cast<double2 *>(smem + OFF_R);
  uint64_t *bar = reinterpret_cast<uint64_t *>(smem + OFF_BAR);
  int *s_slots = reinterpret_cast<int *>(smem + OFF_SLOTS);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int tile = blockIdx.x;
  if (tid < TILE_SLOTS) s_slots[tid] = tiles[tile * TILE_SLOTS + tid];
  if (tid == 0) {
    mbar_init(bar, NT_ADV);
    fence_mbar_init();
  }
  __syncthreads();

  // ---- stage 0: fill the plane ----
#if !CUP2D_ADV_LDGSTS
  {
    // copy A (every thread): row r of interior block blk;  copy B (threads 0..87): a ghost row piece
    const int blk = tid >> 3, r = tid & 7;
    const int slotA = s_slots[blk];
    int slotB = -1, srcB = 0, dstB = 0;
    uint32_t nB = 0;
    if (tid < 32) { // W neighbours: cells 5..7 of every row
      slotB = s_slots[16 + blk], nB = 48, srcB = r * 128 + 80, dstB = (GH + 8 * blk + r) * PS;
    } else if (tid < 64) { // E neighbours: cells 0..2
      slotB = s_slots[20 + blk - 4], nB = 48, srcB = r * 128, dstB = (GH + 8 * (blk - 4) + r) * PS + GH + TC;
    } else if (tid < 76) { // S neighbours: rows 5..7
      const int t = tid - 64, k = t / 3, j = t - 3 * k;
      slotB = s_slots[24 + k], nB = 128, srcB = (5 + j) * 128, dstB = j * PS + GH + 8 * k;
    } else if (tid < 88) { // N neighbours: rows 0..2
      const int t = tid - 76, k = t / 3, j = t - 3 * k;
      slotB = s_slots[28 + k], nB = 128, srcB = j * 128, dstB = (GH + TC + j) * PS + GH + 8 * k;
    }
    const uint32_t bytes = (slotA >= 0 ? 128u : 0u) + (slotB >= 0 ? nB : 0u);
    mbar_arrive_expect_tx(bar, bytes);
    const unsigned char *src = reinterpret_cast<const unsigned char *>(in);
    if (slotA >= 0)
      tma_load_1d(P + (GH + 8 * (blk >> 2) + r) * PS + GH + 8 * (blk & 3), src + (size_t)slotA * 1024 + r * 128, 128u, bar);
    if (slotB >= 0) tma_load_1d(P + dstB, src + (size_t)slotB * 1024 + srcB, nB, bar);
  }
#else
  {
    const double2 *src = reinterpret_cast<const double2 *>(in);
    // interior: 1024 cells, 8 per thread; lanes run along the 8 cells of a row (128 contiguous bytes)
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const int idx = i * NT_ADV + tid, blk = idx >> 6, c = idx & 63;
      const int slot = s_slots[blk];
      if (slot >= 0) ldgsts16(P + (GH + 8 * (blk >> 2) + (c >> 3)) * PS + GH + 8 * (blk & 3) + (c & 7), src + (size_t)slot * 64 + c);
    }
    // W/E ghost columns: 2 sides x 32 rows x 3 cells = 192;  S/N ghost rows: 2 sides x 3 rows x 32 cells = 192
    for (int idx = tid; idx < 384; idx += NT_ADV) {
      int slot, sc, dst;
      if (idx < 192) {
        const int side = idx / 96, t = idx - 96 * side, row = t / 3, j = t - 3 * row;
        slot = s_slots[16 + 4 * side + (row >> 3)];
        sc = (row & 7) * 8 + (side ? j : 5 + j);
        dst = (GH + row) * PS + (side ? GH + TC + j : j);
      } else {
        const int u = idx - 192, side = u / 96, t = u - 96 * side, j = t >> 5, col = t & 31;
        slot = s_slots[24 + 4 * side + (col >> 3)];
        sc = (side ? j : 5 + j) * 8 + (col & 7);
        dst = (side ? GH + TC + j : j) * PS + GH + col;
      }
      if (slot >= 0) ldgsts16(P + dst, src + (size_t)slot * 64 + sc);
    }
  }
#endif
  // y-pass ownership (known now, so the `old` loads of stage 2 can be in flight during everything else)
  const int yx = lane, ys = warp;
  const int yb = ys * 4 + (yx >> 3);
  const int yslot = s_slots[yb];
  const bool store = yslot >= 0 && yslot < nloc;
  double2 oldv[8];
  if (MODE == 2) {
    const double2 *oldp = reinterpret_cast<const double2 *>(old) + (size_t)(store ? yslot : 0) * 64 + (yx & 7);
#pragma unroll
    for (int c = 0; c < 8; c++) oldv[c] = store ? oldp[c * 8] : make_double2(0.0, 0.0);
  }
  const int gx0 = tile_org[2 * tile] * CUP2D_BS, gy0 = tile_org[2 * tile + 1] * CUP2D_BS;
  const int NX = nbx * CUP2D_BS, NY = nby * CUP2D_BS;
#if !CUP2D_ADV_LDGSTS
  if (warp == 0) mbar_wait(bar, 0); // one warp polls the mbarrier; the others park at the CTA barrier
#else
  ldgsts_wait_all();
#endif
  __syncthreads();

  // ---- wall ghosts (perimeter tiles of the domain only): the wall-adjacent cell, normal component negated
  //      (VectorLab::applyBCface main.cpp:3131-3154).  Reads cells inside the domain, writes cells outside: no hazard. ----
  if (gx0 < GH || gy0 < GH || gx0 + TC + GH > NX || gy0 + TC + GH > NY) {
    for (int idx = tid; idx < TW * TW; idx += NT_ADV) {
      const int ty = idx / TW, tx = idx - ty * TW;
      const int lx = tx - GH, ly = ty - GH;
      const bool xin = (unsigned)lx < (unsigned)TC, yin = (unsigned)ly < (unsigned)TC;
      if (!xin && !yin) continue; // corner ghosts are never read (cross-shaped stencil)
      int gx = gx0 + lx, gy = gy0 + ly;
      double sgu = 1.0, sgv = 1.0;
      if (gx < 0) { gx = 0; sgu = -1.0; } else if (gx >= NX) { gx = NX - 1; sgu = -1.0; }
      if (gy < 0) { gy = 0; sgv = -1.0; } else if (gy >= NY) { gy = NY - 1; sgv = -1.0; }
      if (sgu > 0.0 && sgv > 0.0) continue; // inside the domain: loaded (a domain smaller than the tile ends inside it)
      const double2 v = P[(gy - gy0 + GH) * PS + (gx - gx0 + GH)];
      P[ty * PS + tx] = make_double2(sgu * v.x, sgv * v.y);
    }
    __syncthreads();
  }

  double2 *outp = reinterpret_cast<double2 *>(out) + (size_t)(store ? yslot : 0) * 64 + (yx & 7);
  // x pass: warp = the 8 rows of block row `warp`, lane = (segment, row): thread = 8 consecutive cells of one row (u advects)
  // y pass: lane = column, thread = 8 consecutive cells of one column = one block column (v advects)
  // 16-byte bank groups: P row stride 39 = 7 (mod 8), R row stride 33 = 1 (mod 8): the 8 rows of a quarter warp never collide.
  const int xrow = 8 * warp + (lane & 7), xseg = lane >> 3;
  auto run_pass = [&](const int pass) {
    const double2 *q = pass == 0 ? P + (xrow + GH) * PS + 8 * xseg : P + (8 * ys) * PS + (yx + GH);
    const int es = pass == 0 ? 1 : PS;
    double2 *r = pass == 0 ? R + xrow * RS + 8 * xseg : R + (8 * ys) * RS + yx;
    const int rs = pass == 0 ? 1 : RS;
    // which way the eight cells of this line are advected: sign of the advecting component (high words only)
    unsigned pos = 0;
    {
      const int *qh = reinterpret_cast<const int *>(q) + 2 * pass + 1;
#pragma unroll
      for (int c = 0; c < 8; c++) pos |= qh[4 * (c + 3) * es] >= 0 ? (8u << c) : 0u;
    }
    // One result per cell, in the order the line core delivers them (c = 0..7 along the direction of traversal):
    //   x pass: partial sums to R;  y pass: + partial sums, RK update, store.  ci = cell index along the line.
    auto finish = [&](const int ci, const double2 cell, const double2 oldc, const double aU, double du3, double dv3, double Eu, double Ev) {
      if (pass == 0) { // afac*u*dudx + dfac*(u_E + u_W - 2u)
        r[ci * rs] = make_double2(fma(aU, du3, dfac * Eu), fma(aU, dv3, dfac * Ev));
      } else {
        const double2 p = r[ci * rs];
        const double tu = fma(aU, du3, fma(dfac, Eu, p.x));
        const double tv = fma(aU, dv3, fma(dfac, Ev, p.y));
        if (store) {
          double2 o;
          if (MODE == 0) {
            o.x = tu;
            o.y = tv;
          } else if (MODE == 1) { // old == in: the cell values are at hand
            o.x = fma(ofac, tu, cell.x);
            o.y = fma(ofac, tv, cell.y);
          } else {
            o.x = fma(ofac, tu, oldc.x); // V = Vold + coef*tmpV/h^2, main.cpp:6618-6626
            o.y = fma(ofac, tv, oldc.y);
          }
          outp[ci * 8] = o;
        }
      }
    };
    if (CUP2D_ADV_FASTPATH && (pos == 0x7f8u || pos == 0u)) {
      // the whole line is advected one way (the rule away from stagnation lines): straight-line upwind core; from the
      // right = the mirrored line (weno.cuh): window index k -> 13-k, cell c -> 7-c, differences negated
      const bool rev = pos == 0u;
      const double2 *qq = rev ? q + 13 * es : q;
      const int ee = rev ? -es : es;
      const double af = rev ? -afac3 : afac3;
      weno_line_upwind([&](int k, double &x, double &y) {
        const double2 v = qq[k * ee];
        x = v.x;
        y = v.y;
      }, [&](int c, double du3, double dv3, double Eu, double Ev) {
        const double2 cell = qq[(c + 3) * ee];
        const int ci = rev ? 7 - c : c;
        // `old` sits in registers in cell order: picked by a select, not by a run-time register index
        const double2 oldc = MODE == 2 ? (rev ? oldv[7 - c] : oldv[c]) : cell;
        finish(ci, cell, oldc, af * (pass == 0 ? cell.x : cell.y), du3, dv3, Eu, Ev);
      });
    } else {
      weno_line_core([&](int k, double &x, double &y) {
        const double2 v = q[k * es];
        x = v.x;
        y = v.y;
      }, pos, [&](int c, double du3, double dv3, double Eu, double Ev) {
        const double2 cell = q[(c + 3) * es];
        finish(c, cell, MODE == 2 ? oldv[c] : cell, afac3 * (pass == 0 ? cell.x : cell.y), du3, dv3, Eu, Ev);
      });
    }
    __syncwarp(); // the y pass of a warp reads the R rows its own x pass wrote
  };
#if CUP2D_ADV_SPECIALIZE
  run_pass(0); // two copies of the line code, each with its pass folded in (immediate shared-memory offsets, no selects)
  run_pass(1);
#else
#pragma unroll 1
  for (int pass = 0; pass < 2; pass++) run_pass(pass); // one copy, run-time strides
#endif
}

typedef void (*adv_fn)(const double *, const double *, double *, const int *, const int *, int,
                       int, int, double, double, double, const StepFactors *);

// dev: null (factors from dt) or the device-resident factors of the current step
int launch_advect(cup2d_sim *s, const double *in, const double *old, double *out, double coef,
                  double dt, bool raw, const StepFactors *dev) {
  static PerDeviceOnce constants;
  int rc = constants.run(s->device, []() -> int {
    CUP2D_CUDA(cudaMemcpyToSymbol(cW, hW, sizeof hW));
    return (int)CUP2D_OK;
  });
  if (rc) return rc;
  const int mode = raw ? 0 : (old == in ? 1 : 2);
  const adv_fn fn = dev ? (mode == 0 ? advect_stage_kernel<0, true> : mode == 1 ? advect_stage_kernel<1, true> : advect_stage_kernel<2, true>)
                        : (mode == 0 ? advect_stage_kernel<0, false> : mode == 1 ? advect_stage_kernel<1, false> : advect_stage_kernel<2, false>);
  static PerDeviceOnce configured[6];
  rc = configured[mode + (dev ? 3 : 0)].run(s->device, [fn]() -> int {
    CUP2D_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, ADV_SMEM));
    return (int)CUP2D_OK;
  });
  if (rc) return rc;
  const double afac = -dt * s->h; // main.cpp:5447
  const double dfac = s->nu * dt; // main.cpp:5446
  const double ofac = coef / (s->h * s->h);
  ProfScope prof(s, KC_ADVECT);
  fn<<<s->ntiles, NT_ADV, ADV_SMEM, s->stream>>>(in, old, out, s->d_tiles, s->d_tile_org, s->nbx,
                                                 s->nby, (int)s->nloc, afac, dfac, ofac, dev);
  s->launches++;
  CUP2D_CUDA(cudaGetLastError());
  return CUP2D_OK;
}

} // namespace cup2d
