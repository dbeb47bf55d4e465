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
#include "sim.h"
#include <algorithm>
#include <array>
#include <map>
#include <string>
#include <vector>

#include "amr.h"

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
    const double *b = F.src[f] + (int64_t)kid * 64 * dim;
    const double v00 = b[dim * (8 * j + i) + d], v01 = b[dim * (8 * (j + 1) + i) + d];
    const double v10 = b[dim * (8 * j + i + 1) + d], v11 = b[dim * (8 * (j + 1) + i + 1) + d];
#ifdef __CUDA_ARCH__
    F.dst[f][(int64_t)dst[q] * 64 * dim + s] = __ddiv_rn(add_rn(add_rn(add_rn(v00, v01), v10), v11), 4.0);
#else
    F.dst[f][(int64_t)dst[q] * 64 * dim + s] = (((v00 + v01) + v10) + v11) / 4;
#endif
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
    const double *um0 = L.lab[f];
    const int I = child & 1, J = child >> 1, i = 2 * gi, j = 2 * gj;
    const double *um = um0 + q * 100 * dim;
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
    double *b = F.dst[f] + (int64_t)child_dst[4 * q + child] * 64 * dim;
    b[dim * (8 * j + i) + d] = add_rn(add_rn(l00, add_rn(mul_rn(-0.25, x), -ay)), add_rn(c, e));
    b[dim * (8 * j + i + 1) + d] = add_rn(add_rn(l00, add_rn(ax, -ay)), add_rn(c, -e));
    b[dim * (8 * (j + 1) + i) + d] = add_rn(add_rn(l00, add_rn(mul_rn(-0.25, x), ay)), add_rn(c, -e));
    b[dim * (8 * (j + 1) + i + 1) + d] = add_rn(add_rn(l00, add_rn(ax, ay)), add_rn(c, e));
  }
}

static int rg_grid(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, AMR_GRID_SMS * 16)); }

} // namespace cup2d

using namespace cup2d;

extern "C" {

/* Regrid in place onto new_level_ij[nblocks_new][3] (any order; cup2d_amr_adapt_mesh gives the reference's): see the head of
 * this file.  CUP2D_EINVAL (context untouched) if the new mesh is not one refine / compress step from the current one or not
 * 2:1 balanced; CUP2D_ESTATE for multi-rank contexts.  An identical block list is a no-op. */
int cup2d_amr_regrid(cup2d_amr *a, int64_t nblocks_new, const int32_t *new_level_ij) {
  if (!a || nblocks_new <= 0 || !new_level_ij) {
    set_error("cup2d_amr_regrid: bad arguments");
    return CUP2D_EINVAL;
  }
  if (a->dist || a->nranks > 1) {
    set_error("cup2d_amr_regrid: contexts on several ranks cannot be regridded (blocks would have to migrate between ranks)");
    return CUP2D_ESTATE;
  }
  int bpdx = 0, bpdy = 0;
  const std::vector<int> &old = amr_plan_level_ij(a->plan, &bpdx, &bpdy);
  const int64_t nold = a->nb;
  if (nblocks_new == nold && std::equal(old.begin(), old.end(), new_level_ij)) return CUP2D_OK;
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
  // the new context (plan = 2:1 check, zeroed fields, cell sizes, coarse faces); the old one stays valid until the swap
  cup2d_amr *n = nullptr;
  int rc = cup2d_amr_create(nblocks_new, new_level_ij, bpdx, bpdy, a->h0, a->nu, a->device, &n);
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
  std::vector<void *> tmp;
  auto up = [&](const auto &h, auto **d) -> bool {
    using T = typename std::remove_reference<decltype(h[0])>::type;
    if (cudaMalloc(d, std::max<size_t>(h.size(), 1) * sizeof(T)) != cudaSuccess) return false;
    tmp.push_back((void *)*d);
    return cudaMemcpy(*d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice) == cudaSuccess;
  };
  auto release = [&] {
    for (void *p : tmp) cudaFree(p);
  };
  int2 *d_pairs = nullptr;
  int4 *d_kids = nullptr;
  int *d_cdst = nullptr, *d_child = nullptr;
  RgLab L = {};
  bool ok = up(pairs, &d_pairs) && up(kids, &d_kids) && up(cdst, &d_cdst) && up(child_dst, &d_child);
  for (int k = 0; k < 2 && ok; k++) {
    int64_t *r = nullptr;
    int *b = nullptr, *c = nullptr;
    double *ww = nullptr;
    ok = up(rp[k], &r) && up(sb[k], &b) && up(sc[k], &c) && up(w[k], &ww);
    L.rowptr[k] = r, L.sb[k] = b, L.sc[k] = c, L.w[k] = ww;
  }
  L.rbeg[0] = 0;
  for (int f = 0; f < RG_NF; f++) L.rbeg[f + 1] = L.rbeg[f] + (int64_t)rp[F.dim[f] == 2 ? 0 : 1].size() - 1;
  for (int f = 0; f < RG_NF && ok; f++) {
    ok = cudaMalloc(&L.lab[f], std::max<size_t>((size_t)parents.size() * 100 * F.dim[f], 1) * sizeof(double)) == cudaSuccess;
    if (ok) tmp.push_back(L.lab[f]);
  }
  if (!ok) {
    release();
    set_error("cup2d_amr_regrid: out of device memory");
    return fail(CUP2D_ECUDA);
  }
  const int64_t np = (int64_t)pairs.size(), ng = (int64_t)kids.size(), nq = (int64_t)parents.size();
  if (np) amr_regrid_copy_kernel<<<rg_grid(np * F.off2[RG_NF]), 256, 0, a->stream>>>(F, d_pairs, np);
  if (ng) amr_regrid_compress_kernel<<<rg_grid(ng * 2 * F.off2[RG_NF]), 256, 0, a->stream>>>(F, d_cdst, d_kids, ng);
  if (nq) {
    amr_regrid_lab_kernel<<<rg_grid(L.rbeg[RG_NF]), 256, 0, a->stream>>>(F, L);
    amr_regrid_refine_kernel<<<rg_grid(nq * 2 * F.off2[RG_NF]), 256, 0, a->stream>>>(F, L, d_child, nq);
  }
  const bool launched = cudaGetLastError() == cudaSuccess && cudaStreamSynchronize(a->stream) == cudaSuccess;
  release();
  if (!launched) {
    set_error("cup2d_amr_regrid: transfer kernels failed");
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

} // extern "C"
