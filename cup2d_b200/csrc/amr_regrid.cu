// Regrid of a multi-level context in place: adapt()'s field transfer (main.cpp:4902-5195) on the device.
//
// cup2d_amr_regrid(a, n, new_level_ij) moves the context onto a new block list that is one refine / compress step away from
// its current one (what cup2d_amr_adapt_mesh returns).  Every new block is, by a (level, i, j) lookup in the old mesh:
//   - the same block: copied (one launch over all transferred fields, 128-bit loads and stores);
//   - a child of a refined old block: the parent's {-1,-1,2,2,tensorial} lab on the OLD mesh, with wall ghosts (kinds 4 / 5
//     of the plan, rows of the refined parents only), then the 2-D Taylor expression of main.cpp:5012-5028 per 2x2 group of
//     child cells, in the reference's operation order with explicit round-to-nearest adds and multiplies (no FMA contraction);
//     velocities come from the vector lab, whose Taylor ghosts carry component 0 in both components (DESIGN.md 7.1);
//   - the parent of four compressed old blocks: (b[i00] + b[i01] + b[i10] + b[i11]) / 4 in that order (main.cpp:5160-5164).
// Refine and compress read old data only.  Transferred: tmp, chi, vel, vold, pres, pold (the fields adapt() transfers).  tmpV
// is scratch the reference leaves undefined on new blocks; here it is zero on the whole new mesh.
// Then the context swaps its internals for those of the new mesh: plan, cell sizes, coarse faces, block index tables, lab
// buffers and Poisson context (rebuilt lazily on first use, as after cup2d_amr_create); shapes are cleared, their block ids
// naming old blocks.  Handle, stream, device, h0, nu and the fast flag are kept.  Peak memory: old plus new fields.
// cup2d_amr_adapt adds adapt()'s refine / compress decision and the order of the new list on the device (the kernels below
// the transfer's), and feeds the same transfer (regrid_apply) from the device without cup2d_amr_regrid's host classification.
#include "sim.h"
#include <algorithm>
#include <cstring>
#include <array>
#include <map>
#include <string>
#include <vector>

#include "amr.h"
#include "curve.h"

namespace cup2d {

__device__ __forceinline__ double add_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
__device__ __forceinline__ double mul_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}

constexpr int RG_NF = 6; // transferred fields
struct RgFields {        // per transferred field: old and new arrays, components
  const double *src[RG_NF];
  double *dst[RG_NF];
  int dim[RG_NF];
  int off2[RG_NF + 1];   // prefix sums of 32 * dim: double2 slots of one block, over the fields
};

// unchanged blocks: (new block, old block) pairs; one thread per double2 of every transferred field of a pair
__global__ void amr_regrid_copy_kernel(RgFields F, const int2 *__restrict__ pairs, int64_t npairs) {
  const int per = F.off2[RG_NF];
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < npairs * per; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t q = t / per;
    int s = (int)(t - q * per), f = 0;
    while (s >= F.off2[f + 1]) f++;
    s -= F.off2[f];
    const int2 pr = pairs[q];
    const int64_t n2 = 32 * F.dim[f];
    reinterpret_cast<double2 *>(F.dst[f])[pr.x * n2 + s] = reinterpret_cast<const double2 *>(F.src[f])[pr.y * n2 + s];
  }
}

// one value of a compressed parent: the average of the 2x2 cells (i, j) .. (i+1, j+1), component d, of child block b
__device__ __forceinline__ double rg_average4(const double *b, int dim, int i, int j, int d) {
  const double v00 = b[dim * (8 * j + i) + d], v01 = b[dim * (8 * (j + 1) + i) + d];
  const double v10 = b[dim * (8 * j + i + 1) + d], v11 = b[dim * (8 * (j + 1) + i + 1) + d];
#ifdef __CUDA_ARCH__
  return __ddiv_rn(add_rn(add_rn(add_rn(v00, v01), v10), v11), 4.0);
#else
  return (((v00 + v01) + v10) + v11) / 4;
#endif
}

// compressed groups: children[4] (J*2 + I order) -> new block; one thread per output value of every transferred field
__global__ void amr_regrid_compress_kernel(RgFields F, const int *__restrict__ dst, const int4 *__restrict__ kids, int64_t ngroups) {
  const int per = 2 * F.off2[RG_NF]; // doubles of one block over the fields
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < ngroups * per; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t q = t / per;
    int s = (int)(t - q * per), f = 0;
    while (s >= 2 * F.off2[f + 1]) f++;
    s -= 2 * F.off2[f];
    const int dim = F.dim[f], d = s % dim, cell = s / dim, ox = cell & 7, oy = cell >> 3;
    const int4 k4 = kids[q];
    const int I = ox >> 2, J = oy >> 2, kid = J == 0 ? (I == 0 ? k4.x : k4.y) : (I == 0 ? k4.z : k4.w);
    const int i = 2 * (ox & 3), j = 2 * (oy & 3);
    F.dst[f][(int64_t)dst[q] * 64 * dim + s] = rg_average4(F.src[f] + (int64_t)kid * 64 * dim, dim, i, j, d);
  }
}

// labs of the refined parents: lab[field][row] = sum_e w[e] * src[field][...], rows of the field's kind (4: vector, 5: scalar),
// accumulated in table order with explicit round-to-nearest operations; one thread per row of every field
struct RgLab {
  const int64_t *rowptr[2];
  const int *sb[2], *sc[2];
  const double *w[2];
  int64_t rbeg[RG_NF + 1]; // prefix sums of the rows over the fields
  double *lab[RG_NF];
};
__global__ void amr_regrid_lab_kernel(RgFields F, RgLab L) {
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < L.rbeg[RG_NF]; t += (int64_t)gridDim.x * blockDim.x) {
    int f = 0;
    while (t >= L.rbeg[f + 1]) f++;
    const int64_t r = t - L.rbeg[f];
    const int dim = F.dim[f], k = dim == 2 ? 0 : 1;
    double acc = 0.0;
    for (int64_t e = L.rowptr[k][r]; e < L.rowptr[k][r + 1]; e++)
      acc = add_rn(acc, mul_rn(L.w[k][e], F.src[f][(int64_t)L.sb[k][e] * 64 * dim + L.sc[k][e]]));
    L.lab[f][r] = acc;
  }
}

// the four cells of the 2x2 group (i, j) of child (I, J), component d, from the parent's lab um (main.cpp:5012-5028) into
// the child's block b
__device__ __forceinline__ void rg_refine_group(const double *um, double *b, int dim, int d, int I, int J, int i, int j) {
  constexpr int nm = 10;
  const int i0 = i / 2 + 4 * I + 1, j0 = j / 2 + 4 * J + 1, im = i0 - 1, ip = i0 + 1, jm = j0 - 1, jp = j0 + 1;
  const double l00 = um[dim * (nm * j0 + i0) + d], l0p = um[dim * (nm * jp + i0) + d], lm0 = um[dim * (nm * j0 + im) + d];
  const double lmm = um[dim * (nm * jm + im) + d], lmp = um[dim * (nm * jp + im) + d], lp0 = um[dim * (nm * j0 + ip) + d];
  const double lpm = um[dim * (nm * jm + ip) + d], lpp = um[dim * (nm * jp + ip) + d], l0m = um[dim * (nm * jm + i0) + d];
  const double x = mul_rn(0.5, add_rn(lp0, -lm0)), y = mul_rn(0.5, add_rn(l0p, -l0m));
  const double x2 = add_rn(add_rn(lp0, lm0), -mul_rn(2.0, l00)), y2 = add_rn(add_rn(l0p, l0m), -mul_rn(2.0, l00));
  const double xy = mul_rn(0.25, add_rn(add_rn(lpp, lmm), -add_rn(lpm, lmp)));
  const double c = add_rn(mul_rn(0.03125, x2), mul_rn(0.03125, y2)), e = mul_rn(0.0625, xy);
  const double ax = mul_rn(0.25, x), ay = mul_rn(0.25, y);
  b[dim * (8 * j + i) + d] = add_rn(add_rn(l00, add_rn(mul_rn(-0.25, x), -ay)), add_rn(c, e));
  b[dim * (8 * j + i + 1) + d] = add_rn(add_rn(l00, add_rn(ax, -ay)), add_rn(c, -e));
  b[dim * (8 * (j + 1) + i) + d] = add_rn(add_rn(l00, add_rn(mul_rn(-0.25, x), ay)), add_rn(c, -e));
  b[dim * (8 * (j + 1) + i + 1) + d] = add_rn(add_rn(l00, add_rn(ax, ay)), add_rn(c, e));
}

// children of the refined parents from their labs (main.cpp:4982-5031): one thread per (parent, field, child, 2x2 group,
// component) evaluates the four cells of its group.  child_dst[4 q + J*2 + I] = new block of child (I, J) of parent q.
__global__ void amr_regrid_refine_kernel(RgFields F, RgLab L, const int *__restrict__ child_dst, int64_t nparents) {
  const int per = 2 * F.off2[RG_NF]; // 64 * dim threads per field and parent
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < nparents * per; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t q = t / per;
    int s = (int)(t - q * per), f = 0;
    while (s >= 2 * F.off2[f + 1]) f++;
    s -= 2 * F.off2[f];
    const int dim = F.dim[f], d = s % dim, g = s / dim, child = g >> 4, gi = g & 3, gj = (g >> 2) & 3;
    rg_refine_group(L.lab[f] + q * 100 * dim, F.dst[f] + (int64_t)child_dst[4 * q + child] * 64 * dim, dim, d, child & 1,
                    child >> 1, 2 * gi, 2 * gj);
  }
}

// ---- the same transfer on a distributed context (cup2d_amr_create_ranks) --------------------------------------------------
// Every rank computes its own new blocks only and reads the old blocks wherever they live: old global block g is local
// block g - rb[r] of rank r (the old partition), read through the peer mapping of rank r's field array.  Same arithmetic,
// operand order and round-to-nearest operations as the one-rank kernels above, so the values are the same bits.
struct RgPeer {
  const double *base[RG_NF][MAX_RANKS]; // per field: every rank's old array as mapped here (this rank: its own)
  int64_t rb[MAX_RANKS + 1];
  int nranks;
  __device__ __forceinline__ const double *block(int f, int64_t g, int dim) const {
    int r = 0;
    while (r + 1 < nranks && g >= rb[r + 1]) r++;
    return base[f][r] + (g - rb[r]) * 64 * dim;
  }
};

// (new local block, old global block) pairs
__global__ void amr_regrid_peer_copy_kernel(RgFields F, RgPeer P, const int2 *__restrict__ pairs, int64_t npairs) {
  const int per = F.off2[RG_NF];
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < npairs * per; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t q = t / per;
    int s = (int)(t - q * per), f = 0;
    while (s >= F.off2[f + 1]) f++;
    s -= F.off2[f];
    const int2 pr = pairs[q];
    const int64_t n2 = 32 * F.dim[f];
    reinterpret_cast<double2 *>(F.dst[f])[pr.x * n2 + s] = reinterpret_cast<const double2 *>(P.block(f, pr.y, F.dim[f]))[s];
  }
}

// compressed groups: old global children -> new local block
__global__ void amr_regrid_peer_compress_kernel(RgFields F, RgPeer P, const int *__restrict__ dst, const int4 *__restrict__ kids,
                                                int64_t ngroups) {
  const int per = 2 * F.off2[RG_NF];
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < ngroups * per; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t q = t / per;
    int s = (int)(t - q * per), f = 0;
    while (s >= 2 * F.off2[f + 1]) f++;
    s -= 2 * F.off2[f];
    const int dim = F.dim[f], d = s % dim, cell = s / dim, ox = cell & 7, oy = cell >> 3;
    const int4 k4 = kids[q];
    const int I = ox >> 2, J = oy >> 2, kid = J == 0 ? (I == 0 ? k4.x : k4.y) : (I == 0 ? k4.z : k4.w);
    F.dst[f][(int64_t)dst[q] * 64 * dim + s] = rg_average4(P.block(f, kid, dim), dim, 2 * (ox & 3), 2 * (oy & 3), d);
  }
}

// labs of the refined parents, sources named by old global block
__global__ void amr_regrid_peer_lab_kernel(RgFields F, RgPeer P, RgLab L) {
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < L.rbeg[RG_NF]; t += (int64_t)gridDim.x * blockDim.x) {
    int f = 0;
    while (t >= L.rbeg[f + 1]) f++;
    const int64_t r = t - L.rbeg[f];
    const int dim = F.dim[f], k = dim == 2 ? 0 : 1;
    double acc = 0.0;
    for (int64_t e = L.rowptr[k][r]; e < L.rowptr[k][r + 1]; e++)
      acc = add_rn(acc, mul_rn(L.w[k][e], P.block(f, L.sb[k][e], dim)[L.sc[k][e]]));
    L.lab[f][r] = acc;
  }
}

// children of the refined parents; child_dst = new local block, or -1 for a child another rank holds
__global__ void amr_regrid_peer_refine_kernel(RgFields F, RgLab L, const int *__restrict__ child_dst, int64_t nparents) {
  const int per = 2 * F.off2[RG_NF];
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < nparents * per; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t q = t / per;
    int s = (int)(t - q * per), f = 0;
    while (s >= 2 * F.off2[f + 1]) f++;
    s -= 2 * F.off2[f];
    const int dim = F.dim[f], d = s % dim, g = s / dim, child = g >> 4, gi = g & 3, gj = (g >> 2) & 3;
    const int cd = child_dst[4 * q + child];
    if (cd < 0) continue;
    rg_refine_group(L.lab[f] + q * 100 * dim, F.dst[f] + (int64_t)cd * 64 * dim, dim, d, child & 1, child >> 1, 2 * gi, 2 * gj);
  }
}

// ---- adapt()'s decision on the device (cup2d_amr_adapt): cup2d_amr_adapt_mesh (csrc/amr_plan.cpp) kernel by kernel ------
// The old mesh is looked up through its (level, i, j) keys sorted with the block ids (AdIndex: binary search; state() walks
// up the ancestors as Mesh::state does).  The host updates the states in place in the reference's loop order; the kernels
// below run every block of a pass at once and still give the host's answer, because no pass reads what it writes:
//   - the finer-neighbour pass at level lv (amr_plan.cpp: main.cpp:4735-4785) reads the states of level lv+1 only, final
//     after that level's passes, and writes the states of level lv only;
//   - the same-level pass (main.cpp:4791-4823) reads `== REFINE` of level lv and turns COMPRESS into LEAVE only, so no write
//     changes what another block reads; it reads one state array and writes another all the same;
//   - the sibling pass (main.cpp:4825-4860) is idempotent within each group of four: a group whose four states are COMPRESS
//     is left alone, every other group loses all its COMPRESS states whichever member is visited first.  Each block writes
//     its own state into a second array from the group as it was.
// Levels are processed from level_max-1 down to 0, one launch per pass and level, as the host's outer loop.  Neighbour
// enumeration uses the host's order and skip rules (skin skips; positions outside the domain skipped, not wrapped).
enum { AD_LEAVE = 0, AD_REFINE = 1, AD_COMPRESS = 2 };
typedef unsigned long long u64;

// (l, i, j) -> sortable key; l <= 20 and i, j < 2^29 (checked before the decision)
__device__ __forceinline__ u64 ad_key(int l, int i, int j) { return ((u64)l << 58) | ((u64)i << 29) | (u64)j; }

struct AdIndex {           // the old mesh: keys sorted ascending with their block ids
  const u64 *key;
  const int *id;
  int64_t n;
  __device__ int find(int l, int i, int j) const {
    const u64 k = ad_key(l, i, j);
    int64_t lo = 0, hi = n;
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (key[mid] < k) lo = mid + 1;
      else hi = mid;
    }
    return lo < n && key[lo] == k ? id[lo] : -1;
  }
  __device__ int state(int l, int i, int j) const { // Mesh::state: >= 0 block id, -1 refined further, -2 covered by a coarser block
    const int k = find(l, i, j);
    if (k >= 0) return k;
    while (l > 0) {
      l--, i >>= 1, j >>= 1;
      if (find(l, i, j) >= 0) return -2;
    }
    return -1;
  }
};

struct AdMesh {
  const int *lij;          // [n][3] old blocks
  AdIndex idx;
  int bpdx, bpdy, level_max;
  int64_t n;
};

// the host's `neighbours` skip rules: (x, y) is not visited from block (I, J) of an NX x NY level
__device__ __forceinline__ bool ad_skip(int x, int y, int I, int J, int NX, int NY) {
  const bool xskin = I == 0 || I == NX - 1, yskin = J == 0 || J == NY - 1;
  const int xskip = I == 0 ? -1 : 1, yskip = J == 0 ? -1 : 1;
  return (x == 0 && y == 0) || (x == xskip && xskin) || (y == yskip && yskin) || I + x < 0 || I + x >= NX || J + y < 0 ||
         J + y >= NY;
}

// (key, id) of every old block; the tail up to the power of two `npad` sorts last
__global__ void amr_adapt_index_kernel(const int *__restrict__ lij, u64 *key, int *id, int64_t n, int64_t npad) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < npad; k += (int64_t)gridDim.x * blockDim.x) {
    key[k] = k < n ? ad_key(lij[3 * k], lij[3 * k + 1], lij[3 * k + 2]) : ~0ull;
    id[k] = k < n ? (int)k : 0x7fffffff;
  }
}

// one compare-exchange pass (k, j) of a bitonic sort of (key, val) pairs into ascending (key, val) order; n a power of two.
// Launched log2(n) (log2(n) + 1) / 2 times; thread i owns the pair (i, i ^ j) with i < i ^ j, so a pass has no conflicts.
__global__ void amr_adapt_bitonic_kernel(u64 *key, int *val, int64_t n, int64_t k, int64_t j) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = i ^ j;
    if (p <= i) continue;
    const u64 ki = key[i], kp = key[p];
    const int vi = val[i], vp = val[p];
    const bool greater = ki > kp || (ki == kp && vi > vp);
    if (greater == ((i & k) == 0)) {
      key[i] = kp, key[p] = ki;
      val[i] = vp, val[p] = vi;
    }
  }
}

// thresholds (main.cpp:4682-4688): no Refine at level_max-1, no Compress at level 0
__global__ void amr_adapt_state_kernel(AdMesh M, const double *__restrict__ linf, double rtol, double ctol, int *st) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < M.n; k += (int64_t)gridDim.x * blockDim.x) {
    const int l = M.lij[3 * k];
    int s = linf[k] > rtol ? AD_REFINE : linf[k] < ctol ? AD_COMPRESS : AD_LEAVE;
    if ((s == AD_REFINE && l == M.level_max - 1) || (s == AD_COMPRESS && l == 0)) s = AD_LEAVE;
    st[k] = s;
  }
}

// finer neighbours (main.cpp:4735-4785) of the blocks of level lv: in place, reads level lv+1, writes level lv
__global__ void amr_adapt_finer_kernel(AdMesh M, int *st, int lv) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < M.n; k += (int64_t)gridDim.x * blockDim.x) {
    const int l = M.lij[3 * k], I = M.lij[3 * k + 1], J = M.lij[3 * k + 2];
    if (l != lv || st[k] == AD_REFINE || l == M.level_max - 1) continue;
    const int NX = M.bpdx << l, NY = M.bpdy << l;
    int s = st[k];
    bool done = false;
    for (int x = -1; x < 2 && !done; x++)
      for (int y = -1; y < 2 && !done; y++) {
        if (ad_skip(x, y, I, J, NX, NY) || M.idx.state(l, I + x, J + y) != -1) continue;
        if (s == AD_COMPRESS) s = AD_LEAVE;
        const int Bstep = abs(x) + abs(y) == 2 ? 3 : 1;
        for (int B = 0; B <= 1; B += Bstep) {
          const int aux = abs(x) == 1 ? B % 2 : B / 2;
          const int iN = 2 * I + (x > 0 ? x : 0) + x + (B % 2) * (1 - abs(x)); // |x|, |y| <= 1: max(0, 1-|x|) = 1-|x|
          const int jN = 2 * J + (y > 0 ? y : 0) + y + aux * (1 - abs(y));
          const int q = M.idx.find(lv + 1, iN, jN);
          if (q >= 0 && st[q] == AD_REFINE) {
            s = AD_REFINE;
            done = true;
            break;
          }
        }
      }
    st[k] = s;
  }
}

// a same-level neighbour refines (main.cpp:4791-4823): level lv from `in` into `out`, every other state copied
__global__ void amr_adapt_same_kernel(AdMesh M, const int *__restrict__ in, int *__restrict__ out, int lv) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < M.n; k += (int64_t)gridDim.x * blockDim.x) {
    const int l = M.lij[3 * k], I = M.lij[3 * k + 1], J = M.lij[3 * k + 2];
    int s = in[k];
    if (l == lv && s == AD_COMPRESS) {
      const int NX = M.bpdx << l, NY = M.bpdy << l;
      for (int x = -1; x < 2 && s == AD_COMPRESS; x++)
        for (int y = -1; y < 2; y++) {
          if (ad_skip(x, y, I, J, NX, NY)) continue;
          const int q = M.idx.find(l, I + x, J + y);
          if (q >= 0 && in[q] == AD_REFINE) {
            s = AD_LEAVE;
            break;
          }
        }
    }
    out[k] = s;
  }
}

// all four siblings compress, or none does (main.cpp:4825-4860): from `in` into `out`
__global__ void amr_adapt_siblings_kernel(AdMesh M, const int *__restrict__ in, int *__restrict__ out) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < M.n; k += (int64_t)gridDim.x * blockDim.x) {
    int s = in[k];
    if (s == AD_COMPRESS) {
      const int l = M.lij[3 * k], i0 = 2 * (M.lij[3 * k + 1] / 2), j0 = 2 * (M.lij[3 * k + 2] / 2);
      for (int a = 0; a < 2; a++)
        for (int b = 0; b < 2; b++) {
          const int q = M.idx.find(l, i0 + a, j0 + b);
          if (q < 0 || in[q] != AD_COMPRESS) s = AD_LEAVE;
        }
    }
    out[k] = s;
  }
}

// what old block k contributes: (new blocks, copy pairs, refined parents, compressed groups)
__device__ __forceinline__ int4 ad_count(int s, int i, int j) {
  if (s == AD_REFINE) return make_int4(4, 0, 1, 0);
  if (s == AD_COMPRESS) return i % 2 == 0 && j % 2 == 0 ? make_int4(1, 0, 0, 1) : make_int4(0, 0, 0, 0);
  return make_int4(1, 1, 0, 0);
}
__global__ void amr_adapt_count_kernel(AdMesh M, const int *__restrict__ st, int4 *cnt) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < M.n; k += (int64_t)gridDim.x * blockDim.x)
    cnt[k] = ad_count(st[k], M.lij[3 * k + 1], M.lij[3 * k + 2]);
}

// one step (distance d) of an inclusive Hillis-Steele scan of the four counts; launched log2(n) times, ping-pong
__global__ void amr_adapt_scan_kernel(const int4 *__restrict__ in, int4 *__restrict__ out, int64_t n, int64_t d) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
    int4 v = in[k];
    if (k >= d) {
      const int4 u = in[k - d];
      v.x += u.x, v.y += u.y, v.z += u.z, v.w += u.w;
    }
    out[k] = v;
  }
}

// the new blocks in the host's emission order (main.cpp:4926-5195) at the exclusive offsets, with their Encode keys and
// emission indices for the sort (keys padded to the power of two `npad`); the refined parents in old-block order
__global__ void amr_adapt_emit_kernel(AdMesh M, const int *__restrict__ st, const int4 *__restrict__ incl, Curve curve,
                                      int *out_lij, u64 *key, int *val, int64_t nnew, int64_t npad, int *parents) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < M.n; k += (int64_t)gridDim.x * blockDim.x) {
    const int l = M.lij[3 * k], i = M.lij[3 * k + 1], j = M.lij[3 * k + 2], s = st[k];
    const int4 c = ad_count(s, i, j), e = incl[k];
    int q = e.x - c.x;
    auto put = [&](int nl, int ni, int nj) {
      out_lij[3 * q] = nl, out_lij[3 * q + 1] = ni, out_lij[3 * q + 2] = nj;
      key[q] = (u64)curve.encode(nl, ni, nj);
      val[q] = q;
      q++;
    };
    if (s == AD_REFINE) {
      for (int b = 0; b < 2; b++)
        for (int a = 0; a < 2; a++) put(l + 1, 2 * i + a, 2 * j + b);
      parents[e.z - 1] = (int)k;
    } else if (c.x) {
      if (s == AD_COMPRESS) put(l - 1, i / 2, j / 2);
      else put(l, i, j);
    }
  }
  for (int64_t q = nnew + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < npad; q += (int64_t)gridDim.x * blockDim.x)
    key[q] = ~0ull, val[q] = 0x7fffffff;
}

// sorted position p -> new block list, and emission index -> p
__global__ void amr_adapt_rank_kernel(const int *__restrict__ val, const int *__restrict__ out_lij, int *new_lij, int *rank,
                                      int64_t nnew) {
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < nnew; p += (int64_t)gridDim.x * blockDim.x) {
    const int q = val[p];
    rank[q] = (int)p;
    for (int c = 0; c < 3; c++) new_lij[3 * p + c] = out_lij[3 * q + c];
  }
}

// the transfer's inputs, as cup2d_amr_regrid classifies them: copy pairs, the new positions of the children of every
// refined parent, the compressed groups (their sibling ids from the index, J*2 + I order)
__global__ void amr_adapt_transfer_kernel(AdMesh M, const int *__restrict__ st, const int4 *__restrict__ incl,
                                          const int *__restrict__ rank, int2 *pairs, int *child_dst, int4 *kids, int *cdst) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < M.n; k += (int64_t)gridDim.x * blockDim.x) {
    const int l = M.lij[3 * k], i = M.lij[3 * k + 1], j = M.lij[3 * k + 2], s = st[k];
    const int4 c = ad_count(s, i, j), e = incl[k];
    const int q = e.x - c.x;
    if (c.y) pairs[e.y - 1] = make_int2(rank[q], (int)k);
    if (c.z)
      for (int t = 0; t < 4; t++) child_dst[4 * (e.z - 1) + t] = rank[q + t];
    if (c.w) {
      cdst[e.w - 1] = rank[q];
      kids[e.w - 1] = make_int4((int)k, M.idx.find(l, i + 1, j), M.idx.find(l, i, j + 1), M.idx.find(l, i + 1, j + 1));
    }
  }
}

static int rg_grid(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, AMR_GRID_SMS * 16)); }

// device buffers of one call, freed with it
struct RgScratch {
  std::vector<void *> p;
  bool ok = true;
  template <class T> T *get(size_t n) {
    T *d = nullptr;
    if (cudaMalloc(&d, std::max<size_t>(n, 1) * sizeof(T)) != cudaSuccess) {
      ok = false;
      return nullptr;
    }
    p.push_back((void *)d);
    return d;
  }
  template <class T> T *up(const std::vector<T> &h) {
    T *d = get<T>(h.size());
    if (d && !h.empty() && cudaMemcpy(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice) != cudaSuccess) ok = false;
    return d;
  }
  ~RgScratch() {
    for (void *q : p) cudaFree(q);
  }
};

static int64_t pow2_at_least(int64_t n) {
  int64_t m = 1;
  while (m < n) m <<= 1;
  return m;
}

static void bitonic_sort(cudaStream_t stream, u64 *key, int *val, int64_t n) {
  for (int64_t k = 2; k <= n; k <<= 1)
    for (int64_t j = k >> 1; j > 0; j >>= 1) amr_adapt_bitonic_kernel<<<rg_grid(n), 256, 0, stream>>>(key, val, n, k, j);
}

// The transfer and the swap of a regrid whose classification is on the device (see the head of this file): copy pairs
// (new block, old block), compressed groups (kids[g] -> cdst[g]) and refined parents (children child_dst[4 q + J*2 + I]);
// `parents` (host, any order, matching child_dst) selects the lab rows, new_level_ij[nnew][3] the new context's mesh.
static int regrid_apply(cup2d_amr *a, const char *who, int64_t nnew, const int32_t *new_level_ij, int bpdx, int bpdy,
                        const std::vector<int32_t> &parents, const int2 *d_pairs, int64_t np, const int4 *d_kids,
                        const int *d_cdst, int64_t ng, const int *d_child) {
  // the new context (plan = 2:1 check, zeroed fields, cell sizes, coarse faces); the old one stays valid until the swap
  cup2d_amr *n = nullptr;
  int rc = cup2d_amr_create(nnew, new_level_ij, bpdx, bpdy, a->h0, a->nu, a->device, &n);
  if (rc) return rc;
  auto fail = [&](int code) {
    cup2d_amr_destroy(n);
    return code;
  };
  // lab rows of the refined parents on the old mesh (kind 4: vector, 5: scalar)
  std::vector<int64_t> rp[2];
  std::vector<int32_t> sb[2], sc[2];
  std::vector<double> w[2];
  for (int k = 0; k < 2; k++)
    if ((rc = amr_plan_subset_rows(a->plan, 4 + k, (int64_t)parents.size(), parents.data(), rp[k], sb[k], sc[k], w[k]))) return fail(rc);
  const int fields[RG_NF] = {CUP2D_TMP, CUP2D_CHI, CUP2D_VEL, CUP2D_VOLD, CUP2D_PRES, CUP2D_POLD};
  RgFields F;
  F.off2[0] = 0;
  for (int f = 0; f < RG_NF; f++) {
    F.src[f] = a->f[fields[f]], F.dst[f] = n->f[fields[f]], F.dim[f] = dim_of(fields[f]);
    F.off2[f + 1] = F.off2[f] + 32 * F.dim[f];
  }
  const int64_t nq = (int64_t)parents.size();
  bool launched;
  {
    RgScratch S;
    RgLab L = {};
    for (int k = 0; k < 2; k++) L.rowptr[k] = S.up(rp[k]), L.sb[k] = S.up(sb[k]), L.sc[k] = S.up(sc[k]), L.w[k] = S.up(w[k]);
    L.rbeg[0] = 0;
    for (int f = 0; f < RG_NF; f++) L.rbeg[f + 1] = L.rbeg[f] + (int64_t)rp[F.dim[f] == 2 ? 0 : 1].size() - 1;
    for (int f = 0; f < RG_NF; f++) L.lab[f] = S.get<double>((size_t)nq * 100 * F.dim[f]);
    if (!S.ok) {
      set_error(std::string(who) + ": out of device memory");
      return fail(CUP2D_ECUDA);
    }
    if (np) amr_regrid_copy_kernel<<<rg_grid(np * F.off2[RG_NF]), 256, 0, a->stream>>>(F, d_pairs, np);
    if (ng) amr_regrid_compress_kernel<<<rg_grid(ng * 2 * F.off2[RG_NF]), 256, 0, a->stream>>>(F, d_cdst, d_kids, ng);
    if (nq) {
      amr_regrid_lab_kernel<<<rg_grid(L.rbeg[RG_NF]), 256, 0, a->stream>>>(F, L);
      amr_regrid_refine_kernel<<<rg_grid(nq * 2 * F.off2[RG_NF]), 256, 0, a->stream>>>(F, L, d_child, nq);
    }
    launched = cudaGetLastError() == cudaSuccess && cudaStreamSynchronize(a->stream) == cudaSuccess;
  }
  if (!launched) {
    set_error(std::string(who) + ": transfer kernels failed");
    return fail(CUP2D_ECUDA);
  }
  // swap: the handle takes the new mesh's internals; handle, stream, device, h0, nu, the fast flag and the graph switch stay
  std::swap(*a, *n);
  std::swap(a->stream, n->stream);
  a->fast = n->fast;
  a->use_graph = n->use_graph;
  cup2d_amr_destroy(n); // the old mesh: plan, fields, tables, Poisson context, shapes, the graphs of enqueued steps
  return CUP2D_OK;
}

// ---- distributed contexts ------------------------------------------------------------------------------------------------
// The whole adapt runs on every rank: the same arguments (checked), the same global tags (gathered over the peer mapping),
// the same decision kernels over the whole list, the same new list and classification, the same new partition.  Then each
// rank builds its share of the new mesh (cup2d_amr_create_ranks) and fills its own new blocks from the old blocks of
// whichever rank holds them.  Three bounded peer barriers on the old context, all the all-reduce of amr_dist_sum_vec:
// the argument check (for a regrid it also orders every rank's last writes of its old fields before the reads), the tags
// (every rank's tags and old fields final before anyone reads them), and the end of the reads (before anyone frees the old
// arrays).  A rank that never arrives makes the others return CUP2D_ECOMM instead of waiting.

// The reference's new partition (main.cpp:5196-5205, 5332-5349) from the number of new blocks each rank produces (a copy:
// the old block's owner; the children of a refined block: its owner; a compressed parent: the owner of its (even i, even j)
// sibling, to which the reference moves the other three first).  Full rebalance if max / min > 1.01 or a rank produces none:
// total / nranks each, the first total % nranks ranks one more.  Otherwise (n_r - n_{r+1}) / 4 blocks, C division truncating
// toward zero, go from rank r to rank r+1 (a negative number the other way).  Returns the new rank_begin.
static std::vector<int64_t> rebalance(const std::vector<int64_t> &n) {
  const int W = (int)n.size();
  int64_t total = 0, mx = n[0], mn = n[0];
  for (int64_t v : n) total += v, mx = std::max(mx, v), mn = std::min(mn, v);
  std::vector<int64_t> cnt(W), rb(W + 1, 0);
  if (mn == 0 || (double)mx / (double)mn > 1.01) {
    for (int r = 0; r < W; r++) cnt[r] = total / W + (r < total % W ? 1 : 0);
  } else {
    for (int r = 0; r < W; r++) {
      const int64_t left = r == 0 ? 0 : (n[r] - n[r - 1]) / 4, right = r == W - 1 ? 0 : (n[r] - n[r + 1]) / 4;
      cnt[r] = n[r] - left - right;
    }
  }
  for (int r = 0; r < W; r++) rb[r + 1] = rb[r] + cnt[r];
  return rb;
}

// owner rank of global block g under the partition rb
static int owner_of(const std::vector<int64_t> &rb, int64_t g) {
  return (int)(std::upper_bound(rb.begin(), rb.end(), g) - rb.begin()) - 1;
}

// one bounded all-rank barrier on the old context that also checks that every rank passed the same `mine` values (bitwise):
// each rank contributes its row of an nranks x K table, the sum gives every rank every row
static int dist_agree(cup2d_amr *a, const char *who, const std::vector<double> &mine) {
  const int K = (int)mine.size(), W = a->nranks;
  if (W == 1) return CUP2D_OK;
  std::vector<double> v((size_t)W * K, 0.0);
  std::copy(mine.begin(), mine.end(), v.begin() + (size_t)a->rank * K);
  int rc = amr_dist_sum_vec(a, v.data(), W * K);
  if (rc) return rc;
  for (int r = 1; r < W; r++)
    if (memcmp(v.data(), v.data() + (size_t)r * K, K * sizeof(double)) != 0) {
      set_error(std::string(who) + ": the ranks passed different arguments");
      return CUP2D_ECOMM;
    }
  return CUP2D_OK;
}

// 64-bit FNV-1a of a block list, as two doubles (exact: 32 bits each)
static void list_hash(const int32_t *lij, int64_t n, std::vector<double> &out) {
  u64 h = 1469598103934665603ull;
  for (int64_t k = 0; k < 3 * n; k++) h = (h ^ (u64)(uint32_t)lij[k]) * 1099511628211ull;
  out.push_back((double)(h >> 32));
  out.push_back((double)(h & 0xffffffffull));
}

// The global classification of a regrid, on the host: copy pairs (new, old), compressed groups kids[g] -> cdst[g], refined
// parents with child_dst[4 q + J*2 + I] (global block ids throughout).  Moves every rank of the distributed context `a` onto
// its range of the new list under the reference's partition; no-op (changed = false) if neither list nor partition changes.
struct RgPlanHost {
  std::vector<int2> pairs;
  std::vector<int4> kids;
  std::vector<int32_t> cdst, parents, child_dst;
};
static int regrid_apply_dist(cup2d_amr *a, const char *who, int64_t nnew, const int32_t *new_level_ij, int bpdx, int bpdy,
                             const RgPlanHost &C, bool *changed) {
  const int W = a->nranks, me = a->rank;
  const std::vector<int64_t> &orb = a->rank_begin;
  std::vector<int64_t> produced(W, 0);
  for (const int2 &p : C.pairs) produced[owner_of(orb, p.y)]++;
  for (int32_t p : C.parents) produced[owner_of(orb, p)] += 4;
  for (const int4 &k : C.kids) produced[owner_of(orb, k.x)]++;
  const std::vector<int64_t> rb = rebalance(produced);
  bool empty = false;
  for (int r = 0; r < W; r++) empty |= rb[r + 1] <= rb[r];
  int bx = 0, by = 0;
  const std::vector<int> &old = amr_plan_level_ij(a->plan, &bx, &by);
  *changed = !(nnew == a->nglobal && std::equal(old.begin(), old.end(), new_level_ij) && rb == orb);
  if (empty || !*changed) { // every rank takes this branch; the barrier ends the peer reads of the tag gather first
    int rc = dist_agree(a, who, {3.0});
    if (rc || !empty) return rc;
    set_error(std::string(who) + ": the new mesh has fewer blocks than ranks (" + std::to_string(nnew) + " for " +
              std::to_string(W) + ")");
    return CUP2D_EINVAL;
  }
  cup2d_amr *n = nullptr;
  int rc = cup2d_amr_create_ranks(nnew, new_level_ij, bpdx, bpdy, a->h0, a->nu, me, W, rb.data(), a->device, &n);
  if (rc) return rc;
  auto fail = [&](int code) {
    cup2d_amr_destroy(n);
    return code;
  };
  // this rank's share: new blocks in [b0, b1), numbered locally; sources stay global
  const int64_t b0 = rb[me], b1 = rb[me + 1];
  auto mine = [&](int64_t g) { return g >= b0 && g < b1; };
  std::vector<int2> pairs;
  std::vector<int4> kids;
  std::vector<int32_t> cdst, parents, child;
  for (const int2 &p : C.pairs)
    if (mine(p.x)) pairs.push_back(make_int2((int)(p.x - b0), p.y));
  for (size_t g = 0; g < C.kids.size(); g++)
    if (mine(C.cdst[g])) kids.push_back(C.kids[g]), cdst.push_back((int32_t)(C.cdst[g] - b0));
  for (size_t q = 0; q < C.parents.size(); q++) {
    bool any = false;
    for (int c = 0; c < 4; c++) any |= mine(C.child_dst[4 * q + c]);
    if (!any) continue;
    parents.push_back(C.parents[q]);
    for (int c = 0; c < 4; c++) child.push_back(mine(C.child_dst[4 * q + c]) ? (int32_t)(C.child_dst[4 * q + c] - b0) : -1);
  }
  std::vector<int64_t> rp[2];
  std::vector<int32_t> sb[2], sc[2];
  std::vector<double> w[2];
  for (int k = 0; k < 2; k++)
    if ((rc = amr_plan_subset_rows(a->plan, 4 + k, (int64_t)parents.size(), parents.data(), rp[k], sb[k], sc[k], w[k]))) return fail(rc);
  const int fields[RG_NF] = {CUP2D_TMP, CUP2D_CHI, CUP2D_VEL, CUP2D_VOLD, CUP2D_PRES, CUP2D_POLD};
  RgFields F;
  RgPeer P;
  memset(&P, 0, sizeof P);
  F.off2[0] = 0;
  for (int f = 0; f < RG_NF; f++) {
    F.src[f] = nullptr, F.dst[f] = n->f[fields[f]], F.dim[f] = dim_of(fields[f]);
    F.off2[f + 1] = F.off2[f] + 32 * F.dim[f];
    for (int r = 0; r < W; r++) {
      P.base[f][r] = static_cast<const double *>(cup2d_peer_field_ptr(a->poisson, r, fields[f]));
      if (!P.base[f][r]) {
        set_error(std::string(who) + ": peers not attached");
        return fail(CUP2D_ESTATE);
      }
    }
  }
  for (int r = 0; r <= W; r++) P.rb[r] = orb[r];
  P.nranks = W;
  const int64_t np = (int64_t)pairs.size(), ng = (int64_t)kids.size(), nq = (int64_t)parents.size();
  bool launched;
  {
    RgScratch S;
    RgLab L = {};
    for (int k = 0; k < 2; k++) L.rowptr[k] = S.up(rp[k]), L.sb[k] = S.up(sb[k]), L.sc[k] = S.up(sc[k]), L.w[k] = S.up(w[k]);
    L.rbeg[0] = 0;
    for (int f = 0; f < RG_NF; f++) L.rbeg[f + 1] = L.rbeg[f] + (int64_t)rp[F.dim[f] == 2 ? 0 : 1].size() - 1;
    for (int f = 0; f < RG_NF; f++) L.lab[f] = S.get<double>((size_t)nq * 100 * F.dim[f]);
    const int2 *d_pairs = S.up(pairs);
    const int4 *d_kids = S.up(kids);
    const int *d_cdst = S.up(cdst), *d_child = S.up(child);
    if (!S.ok) {
      set_error(std::string(who) + ": out of device memory");
      return fail(CUP2D_ECUDA);
    }
    if (np) amr_regrid_peer_copy_kernel<<<rg_grid(np * F.off2[RG_NF]), 256, 0, a->stream>>>(F, P, d_pairs, np);
    if (ng) amr_regrid_peer_compress_kernel<<<rg_grid(ng * 2 * F.off2[RG_NF]), 256, 0, a->stream>>>(F, P, d_cdst, d_kids, ng);
    if (nq) {
      amr_regrid_peer_lab_kernel<<<rg_grid(L.rbeg[RG_NF]), 256, 0, a->stream>>>(F, P, L);
      amr_regrid_peer_refine_kernel<<<rg_grid(nq * 2 * F.off2[RG_NF]), 256, 0, a->stream>>>(F, L, d_child, nq);
    }
    launched = cudaGetLastError() == cudaSuccess && cudaStreamSynchronize(a->stream) == cudaSuccess;
  }
  if (!launched) {
    set_error(std::string(who) + ": transfer kernels failed");
    return fail(CUP2D_ECUDA);
  }
  // every rank done reading before anyone frees its old arrays
  if ((rc = dist_agree(a, who, {4.0}))) return fail(rc);
  // one rank attaches itself; several re-exchange their blobs (cup2d_amr_peer_export / _attach) before the next peer call
  const char none = 0;
  if (W == 1 && (rc = cup2d_amr_peer_attach(n, &none))) return fail(rc);
  const bool use_graph = a->use_graph;
  std::swap(*a, *n); // a distributed context's stream belongs to its Poisson context: the new mesh's stream comes along
  a->use_graph = use_graph;
  cup2d_amr_destroy(n);
  return CUP2D_OK;
}

// the distributed adapt / regrid entry: the argument check and barrier, then (adapt) the tags of every rank into d_linf
// [nglobal]; `own` = this rank's tags on the device
static int dist_gather_tags(cup2d_amr *a, const double *own, double *d_linf) {
  const int W = a->nranks;
  cup2d_sim *ps = a->poisson;
  if (W > 1) { // this rank's tags into its Krylov scratch kz (exported, idle outside the Poisson solve), then a barrier
    CUP2D_CUDA(cudaMemcpyAsync(ps->kz, own, (size_t)a->nb * sizeof(double), cudaMemcpyDeviceToDevice, a->stream));
    int rc = dist_agree(a, "cup2d_amr_adapt", {2.0});
    if (rc) return rc;
  }
  for (int r = 0; r < W; r++) {
    const double *src = r == a->rank ? own : static_cast<const double *>(ps->peer_base[r][CUP2D_NFIELDS]);
    CUP2D_CUDA(cudaMemcpyAsync(d_linf + a->rank_begin[r], src, (size_t)(a->rank_begin[r + 1] - a->rank_begin[r]) * sizeof(double),
                               cudaMemcpyDeviceToDevice, a->stream));
  }
  return CUP2D_OK;
}

} // namespace cup2d

using namespace cup2d;

extern "C" {

/* Regrid in place onto new_level_ij[nblocks_new][3] (any order; cup2d_amr_adapt_mesh gives the reference's): see the head of
 * this file.  CUP2D_EINVAL (context untouched) if the new mesh is not one refine / compress step from the current one or not
 * 2:1 balanced; CUP2D_ESTATE for contexts of cup2d_amr_set_ranks.  An identical block list is a no-op.  Distributed contexts:
 * every rank passes the whole new list (regrid_apply_dist). */
int cup2d_amr_regrid(cup2d_amr *a, int64_t nblocks_new, const int32_t *new_level_ij) {
  if (!a || nblocks_new <= 0 || !new_level_ij) {
    set_error("cup2d_amr_regrid: bad arguments");
    return CUP2D_EINVAL;
  }
  if (a->nranks > 1 && !a->dist) {
    set_error("cup2d_amr_regrid: contexts of cup2d_amr_set_ranks (operators replicated on several ranks) cannot be regridded");
    return CUP2D_ESTATE;
  }
  int bpdx = 0, bpdy = 0;
  const std::vector<int> &old = amr_plan_level_ij(a->plan, &bpdx, &bpdy);
  const int64_t nold = a->nglobal;
  if (a->dist) {
    std::vector<double> args = {1.0, (double)nblocks_new};
    list_hash(new_level_ij, nblocks_new, args);
    CUP2D_CUDA(cudaSetDevice(a->device));
    const int rc = dist_agree(a, "cup2d_amr_regrid", args);
    if (rc) return rc;
  } else if (nblocks_new == nold && std::equal(old.begin(), old.end(), new_level_ij)) {
    return CUP2D_OK;
  }
  std::map<std::array<int, 3>, int> index;
  for (int64_t k = 0; k < nold; k++) index[{old[3 * k], old[3 * k + 1], old[3 * k + 2]}] = (int)k;
  auto find = [&](int l, int i, int j) {
    auto it = index.find({l, i, j});
    return it == index.end() ? -1 : it->second;
  };
  // classify the new blocks; every old block must be used exactly once (copied, refined into all four children, or one of a
  // compressed group)
  std::vector<int2> pairs;
  std::vector<int32_t> parents, child_dst, cdst;
  std::vector<int4> kids;
  std::map<int, int> parent_slot;
  std::vector<int> used(nold, 0);
  auto reject = [&](const std::string &why) {
    set_error("cup2d_amr_regrid: the new mesh is not one refine / compress step away from the current one: " + why);
    return CUP2D_EINVAL;
  };
  for (int64_t n = 0; n < nblocks_new; n++) {
    const int l = new_level_ij[3 * n], i = new_level_ij[3 * n + 1], j = new_level_ij[3 * n + 2];
    const std::string where = "new block " + std::to_string(n);
    if (l < 0 || l > 20 || i < 0 || j < 0) return reject(where + " has a bad index");
    int k = find(l, i, j);
    if (k >= 0) {
      pairs.push_back(make_int2((int)n, k));
      used[k]++;
    } else if (l > 0 && (k = find(l - 1, i / 2, j / 2)) >= 0) {
      auto it = parent_slot.find(k);
      if (it == parent_slot.end()) {
        it = parent_slot.emplace(k, (int)parents.size()).first;
        parents.push_back(k);
        child_dst.insert(child_dst.end(), 4, -1);
      }
      int &slot = child_dst[4 * it->second + 2 * (j % 2) + (i % 2)];
      if (slot >= 0) return reject(where + " is duplicated");
      slot = (int)n;
      used[k]++;
    } else {
      int c[4];
      for (int b = 0; b < 2; b++)
        for (int q = 0; q < 2; q++) c[2 * b + q] = find(l + 1, 2 * i + q, 2 * j + b);
      if (c[0] < 0 || c[1] < 0 || c[2] < 0 || c[3] < 0) return reject(where + " is neither an old block, nor a child of one, nor the parent of four");
      for (int q = 0; q < 4; q++) used[c[q]]++;
      kids.push_back(make_int4(c[0], c[1], c[2], c[3]));
      cdst.push_back((int)n);
    }
  }
  for (size_t q = 0; q < parents.size(); q++) {
    for (int c = 0; c < 4; c++)
      if (child_dst[4 * q + c] < 0) return reject("old block " + std::to_string(parents[q]) + " is refined without all four children");
    used[parents[q]] -= 3;
  }
  for (int64_t k = 0; k < nold; k++)
    if (used[k] != 1) return reject("old block " + std::to_string(k) + (used[k] ? " is used twice" : " is not covered"));
  if (a->dist) {
    bool changed = false;
    return regrid_apply_dist(a, "cup2d_amr_regrid", nblocks_new, new_level_ij, bpdx, bpdy, RgPlanHost{pairs, kids, cdst, parents, child_dst},
                             &changed);
  }
  RgScratch S;
  const int2 *d_pairs = S.up(pairs);
  const int4 *d_kids = S.up(kids);
  const int *d_cdst = S.up(cdst), *d_child = S.up(child_dst);
  if (!S.ok) {
    set_error("cup2d_amr_regrid: out of device memory");
    return CUP2D_ECUDA;
  }
  return regrid_apply(a, "cup2d_amr_regrid", nblocks_new, new_level_ij, bpdx, bpdy, parents, d_pairs, (int64_t)pairs.size(),
                      d_kids, d_cdst, (int64_t)kids.size(), d_child);
}

/* adapt() in one call: tagging (block_linf == NULL) or the caller's per-block values, the refine / compress decision and the
 * order of the new list on the device (bitwise cup2d_amr_adapt_mesh), then the transfer of cup2d_amr_regrid fed from the
 * device.  Downloaded: the new block list (the host builds its plan) and the refined parents (their lab rows). */
int cup2d_amr_adapt(cup2d_amr *a, const double *block_linf, double rtol, double ctol, int level_max, int64_t *nblocks_out,
                    int32_t *changed_out) {
  if (!a || level_max < 1 || level_max > 20) {
    set_error("cup2d_amr_adapt: bad arguments");
    return CUP2D_EINVAL;
  }
  if (a->nranks > 1 && !a->dist) {
    set_error("cup2d_amr_adapt: contexts of cup2d_amr_set_ranks (operators replicated on several ranks) cannot be regridded");
    return CUP2D_ESTATE;
  }
  int bpdx = 0, bpdy = 0;
  const std::vector<int> &old = amr_plan_level_ij(a->plan, &bpdx, &bpdy);
  const int64_t nold = a->nglobal;
  if (((int64_t)std::max(bpdx, bpdy) << (level_max - 1)) >= (1 << 29)) {
    set_error("cup2d_amr_adapt: the finest level has 2^29 blocks or more per direction");
    return CUP2D_EINVAL;
  }
  for (int64_t k = 0; k < nold; k++)
    if (old[3 * k] >= level_max) {
      set_error("cup2d_amr_adapt: block " + std::to_string(k) + " is at or above level_max");
      return CUP2D_EINVAL;
    }
  CUP2D_CUDA(cudaSetDevice(a->device));
  if (a->dist) {
    const int rc = dist_agree(a, "cup2d_amr_adapt", {0.0, rtol, ctol, (double)level_max, block_linf ? 1.0 : 0.0});
    if (rc) return rc;
  }
  RgScratch S;
  const double *d_linf = a->d_part;
  if (block_linf) {
    d_linf = S.up(std::vector<double>(block_linf, block_linf + a->nb)); // a distributed context: this rank's blocks
  } else {
    const int rc = amr_adapt_tags_enqueue(a, rtol, level_max);
    if (rc) return rc;
  }
  if (a->dist) { // every rank's tags, in global block order
    double *all = S.get<double>(nold);
    if (!S.ok) {
      set_error("cup2d_amr_adapt: out of device memory");
      return CUP2D_ECUDA;
    }
    const int rc = dist_gather_tags(a, d_linf, all);
    if (rc) return rc;
    d_linf = all;
  }
  const int64_t npad = pow2_at_least(nold);
  const CurveTables tables(bpdx, bpdy);
  const int64_t *d_zsave = S.up(tables.zsave);
  const int32_t *d_inv = S.up(tables.inv);
  int *d_lij = S.up(old);
  u64 *d_key = S.get<u64>(npad);
  int *d_id = S.get<int>(npad), *st = S.get<int>(nold), *st2 = S.get<int>(nold);
  int4 *sa = S.get<int4>(nold), *sb = S.get<int4>(nold);
  if (!S.ok) {
    set_error("cup2d_amr_adapt: out of device memory");
    return CUP2D_ECUDA;
  }
  cudaStream_t stream = a->stream;
  const int g = rg_grid(nold);
  // the old mesh's index, the states, the 2:1 passes level by level, the sibling agreement
  amr_adapt_index_kernel<<<rg_grid(npad), 256, 0, stream>>>(d_lij, d_key, d_id, nold, npad);
  bitonic_sort(stream, d_key, d_id, npad);
  const AdMesh M{d_lij, AdIndex{d_key, d_id, nold}, bpdx, bpdy, level_max, nold};
  amr_adapt_state_kernel<<<g, 256, 0, stream>>>(M, d_linf, rtol, ctol, st);
  for (int lv = level_max - 1; lv >= 0; lv--) {
    amr_adapt_finer_kernel<<<g, 256, 0, stream>>>(M, st, lv);
    if (lv == 0) break;
    amr_adapt_same_kernel<<<g, 256, 0, stream>>>(M, st, st2, lv);
    std::swap(st, st2);
  }
  amr_adapt_siblings_kernel<<<g, 256, 0, stream>>>(M, st, st2);
  std::swap(st, st2);
  // offsets of every old block's contribution: inclusive scan of the counts (ends in sa)
  amr_adapt_count_kernel<<<g, 256, 0, stream>>>(M, st, sa);
  for (int64_t d = 1; d < nold; d <<= 1) {
    amr_adapt_scan_kernel<<<g, 256, 0, stream>>>(sa, sb, nold, d);
    std::swap(sa, sb);
  }
  int4 tot;
  CUP2D_CUDA(cudaGetLastError());
  CUP2D_CUDA(cudaMemcpyAsync(&tot, sa + nold - 1, sizeof(int4), cudaMemcpyDeviceToHost, stream));
  CUP2D_CUDA(cudaStreamSynchronize(stream));
  const int64_t nnew = tot.x, np = tot.y, nq = tot.z, ng = tot.w, npad2 = pow2_at_least(nnew);
  // the new list in emission order, sorted by (Encode, emission index) as the host's std::sort of (key, q) pairs
  int *out_lij = S.get<int>(3 * nnew), *new_lij = S.get<int>(3 * nnew), *rank = S.get<int>(nnew);
  int *d_parents = S.get<int>(nq), *d_child = S.get<int>(4 * nq), *d_cdst = S.get<int>(ng);
  u64 *key2 = S.get<u64>(npad2);
  int *val2 = S.get<int>(npad2);
  int2 *d_pairs = S.get<int2>(np);
  int4 *d_kids = S.get<int4>(ng);
  if (!S.ok) {
    set_error("cup2d_amr_adapt: out of device memory");
    return CUP2D_ECUDA;
  }
  amr_adapt_emit_kernel<<<rg_grid(std::max(nold, npad2)), 256, 0, stream>>>(M, st, sa, tables.curve(level_max, d_zsave, d_inv),
                                                                           out_lij, key2, val2, nnew, npad2, d_parents);
  bitonic_sort(stream, key2, val2, npad2);
  amr_adapt_rank_kernel<<<rg_grid(nnew), 256, 0, stream>>>(val2, out_lij, new_lij, rank, nnew);
  amr_adapt_transfer_kernel<<<g, 256, 0, stream>>>(M, st, sa, rank, d_pairs, d_child, d_kids, d_cdst);
  CUP2D_CUDA(cudaGetLastError());
  std::vector<int32_t> nl((size_t)3 * nnew), parents((size_t)nq);
  CUP2D_CUDA(cudaMemcpyAsync(nl.data(), new_lij, nl.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
  if (nq) CUP2D_CUDA(cudaMemcpyAsync(parents.data(), d_parents, parents.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
  CUP2D_CUDA(cudaStreamSynchronize(stream));
  if (a->dist) { // the global classification to the host: every rank takes its share of it
    RgPlanHost C;
    C.pairs.resize(np), C.kids.resize(ng), C.cdst.resize(ng), C.child_dst.resize(4 * nq);
    C.parents = parents;
    if (np) CUP2D_CUDA(cudaMemcpy(C.pairs.data(), d_pairs, np * sizeof(int2), cudaMemcpyDeviceToHost));
    if (ng) CUP2D_CUDA(cudaMemcpy(C.kids.data(), d_kids, ng * sizeof(int4), cudaMemcpyDeviceToHost));
    if (ng) CUP2D_CUDA(cudaMemcpy(C.cdst.data(), d_cdst, ng * sizeof(int), cudaMemcpyDeviceToHost));
    if (nq) CUP2D_CUDA(cudaMemcpy(C.child_dst.data(), d_child, 4 * nq * sizeof(int), cudaMemcpyDeviceToHost));
    bool changed = false;
    const int rc = regrid_apply_dist(a, "cup2d_amr_adapt", nnew, nl.data(), bpdx, bpdy, C, &changed);
    if (rc) return rc;
    if (nblocks_out) *nblocks_out = nnew;
    if (changed_out) *changed_out = changed;
    return CUP2D_OK;
  }
  const bool same = nnew == nold && std::equal(old.begin(), old.end(), nl.begin());
  const int rc = same ? CUP2D_OK : regrid_apply(a, "cup2d_amr_adapt", nnew, nl.data(), bpdx, bpdy, parents, d_pairs, np, d_kids,
                                                d_cdst, ng, d_child);
  if (rc) return rc;
  if (nblocks_out) *nblocks_out = nnew;
  if (changed_out) *changed_out = !same;
  return CUP2D_OK;
}

/* the partition of the context's block list: rank_begin[nranks+1] (NULL: only nranks); {0, nb} for a plain context */
int32_t cup2d_amr_rank_begin(const cup2d_amr *a, int64_t *rank_begin_out) {
  if (!a) {
    set_error("cup2d_amr_rank_begin: bad arguments");
    return CUP2D_EINVAL;
  }
  const std::vector<int64_t> plain = {0, a->nb};
  const std::vector<int64_t> &rb = a->rank_begin.empty() ? plain : a->rank_begin;
  if (rank_begin_out) std::copy(rb.begin(), rb.end(), rank_begin_out);
  return (int32_t)rb.size() - 1;
}

/* the context's block list [n][3] (level, i, j) into level_ij_out (NULL: only the count) */
int64_t cup2d_amr_blocks(const cup2d_amr *a, int32_t *level_ij_out) {
  if (!a) {
    set_error("cup2d_amr_blocks: bad arguments");
    return CUP2D_EINVAL;
  }
  int bpdx = 0, bpdy = 0;
  const std::vector<int> &lij = amr_plan_level_ij(a->plan, &bpdx, &bpdy);
  if (level_ij_out) std::copy(lij.begin(), lij.end(), level_ij_out);
  return (int64_t)lij.size() / 3;
}

} // extern "C"
