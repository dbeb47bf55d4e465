// The collision model on a multi-level mesh (main.cpp:6705-6943, with collision() / compute_j() at 209-291) on the obstacle
// blocks the device already holds (cup2d_amr_ongrid, or cup2d_amr_shape_set + cup2d_amr_shape_set_dist).
//
// cup2d_amr_collide(a, n, shapes, sums20): for every shape i the reference walks the other shapes j in index order, their
// common obstacle blocks k in ascending block order and the cells (iy, ix) of each, and accumulates over the cells where both
// chi are positive the 14 sums of 6764-6810 (i's mass, position, momentum and chi grad dist; the same of j).  Each sum is one
// serial chain per shape, so the result is reproduced bit for bit only if it is added in that order.  Kernels (stable names):
//   amr_collide_match_kernel  every unordered pair (a, b) with both shapes non-empty: each obstacle block of the shorter list
//                             a is looked up by binary search in b's ascending ids -> its position in b, or -1
//   amr_collide_sums_kernel   one CTA per shape i, partners j in order: the CTA compacts the pair's matches (ascending block
//                             order) 256 at a time, evaluates the 14 per-cell values of 4 common blocks at a time, one thread
//                             per cell, in the reference's expression order (cells that do not contribute hold +0.0, which
//                             leaves a sum that is never -0.0 unchanged), and 14 threads each add one quantity's values in
//                             cell order to their running sum: the serial chain of the reference, no tree or warp reduction
// The 20 N sums (Z slots zero, the layout of 6814-6837) come back in one download; the host then runs the pair loop of
// 6863-6943 with collision() / compute_j() restated in the reference's expression order, pairs in (i ascending, j > i
// ascending) order.  The file is compiled without FMA contraction, device (-fmad=false) and host (-ffp-contract=off) code
// alike (Makefile), like the reference's host build, so every expression rounds as it does there.
#include "sim.h"
#include "amr.h"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

namespace cup2d {

constexpr int CO_MAXSH = 64;
constexpr int CO_NT = 256;       // threads of the sums kernel: a chunk of 256 matches, 4 common blocks of 64 cells per batch
constexpr int CO_MATCH_NT = 128;

struct CoShapes {                // every shape's obstacle blocks
  const int *ids[CO_MAXSH];
  const double *X[CO_MAXSH], *udef[CO_MAXSH], *dist[CO_MAXSH];
};
struct CoMotion { double u, v, omega, cx, cy; }; // rigid motion and centre of mass of one shape (main.cpp:6740-6750)
struct CoPair { int a, b, na, nb, off; };        // walk a's ids (the shorter list) in b's; matches at off .. off + na - 1

// matches of every pair, flattened: g in [pair.off, pair.off + pair.na) -> position of a's block in b's ids, or -1
__global__ void __launch_bounds__(CO_MATCH_NT)
amr_collide_match_kernel(const CoShapes S, const CoPair *__restrict__ pairs, int npairs, int total, int *__restrict__ match) {
  for (int g = blockIdx.x * CO_MATCH_NT + threadIdx.x; g < total; g += gridDim.x * CO_MATCH_NT) {
    int lo = 0, hi = npairs - 1; // the last pair with off <= g
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (pairs[mid].off <= g) lo = mid;
      else hi = mid - 1;
    }
    const CoPair P = pairs[lo];
    const int key = S.ids[P.a][g - P.off];
    const int *ib = S.ids[P.b];
    int l = 0, r = P.nb; // the first position of b with id >= key
    while (l < r) {
      const int m = (l + r) >> 1;
      if (ib[m] < key) l = m + 1;
      else r = m;
    }
    match[g] = l < P.nb && ib[l] == key ? l : -1;
  }
}

// main.cpp:6766-6810 for one shape's values at one cell: chi, chi pos, chi (u + omega x r + u_def), chi grad dist (one-sided
// differences at the block edges, central inside)
__device__ __forceinline__ void co_cell(double c, const double *__restrict__ dist, const double2 U, const CoMotion &m, double p0,
                                        double p1, int ix, int iy, double *o) {
  const double ur0 = -m.omega * (p1 - m.cy), ur1 = m.omega * (p0 - m.cx);
  const double *D = dist + iy * 8;
  const double dx = ix == 0 ? D[1] - D[0] : ix == 7 ? D[7] - D[6] : 0.5 * (D[ix + 1] - D[ix - 1]);
  const double dy = iy == 0 ? dist[8 + ix] - dist[ix] : iy == 7 ? dist[56 + ix] - dist[48 + ix]
                                                                 : 0.5 * (D[8 + ix] - D[ix - 8]);
  o[0] = c;
  o[1] = c * p0;
  o[2] = c * p1;
  o[3] = c * (m.u + ur0 + U.x);
  o[4] = c * (m.v + ur1 + U.y);
  o[5] = c * dx;
  o[6] = c * dy;
}

// one CTA per shape i: sums[i][20] in the reference's order (see the file comment)
__global__ void __launch_bounds__(CO_NT)
amr_collide_sums_kernel(const CoShapes S, const CoMotion *__restrict__ mo, const int *__restrict__ pidx, const CoPair *__restrict__ pairs,
                        int nshapes, const int *__restrict__ match, const int2 *__restrict__ ij, const double *__restrict__ hb,
                        double *__restrict__ sums) {
  __shared__ double s_v[14 * CO_NT]; // [quantity][group * 64 + cell]: 0..6 shape i, 7..13 the partner
  __shared__ int2 s_q[CO_NT];        // the chunk's common blocks (position in i's list, in j's), ascending
  __shared__ int s_w[CO_NT / 32];    // matches per warp
  __shared__ unsigned s_n[8];        // contributing cells per group, [batch parity][group]
  const int i = blockIdx.x, t = threadIdx.x, lane = t & 31, w = t >> 5, grp = t >> 6, cell = t & 63, ix = cell & 7, iy = cell >> 3;
  double acc = 0; // thread t < 14: the running sum of quantity t
  if (t < 8) s_n[t] = 0;
  int batch = 0;
  __syncthreads();
  for (int j = 0; j < nshapes; j++) {
    const int p = j == i ? -1 : pidx[i * nshapes + j];
    if (p < 0) continue;
    const CoPair P = pairs[p];
    const bool i_is_a = P.a == i;
    for (int c0 = 0; c0 < P.na; c0 += CO_NT) {
      const int ka = c0 + t, kb = ka < P.na ? match[P.off + ka] : -1;
      int x = kb >= 0; // inclusive scan of the match flags within the warp, then across the warps: order is kept
      for (int d = 1; d < 32; d <<= 1) {
        const int y = __shfl_sync(0xffffffffu, x, (lane - d) & 31);
        if (lane >= d) x += y;
      }
      if (lane == 31) s_w[w] = x;
      __syncthreads();
      int base = 0, nq = 0;
      for (int q = 0; q < CO_NT / 32; q++) {
        base += q < w ? s_w[q] : 0;
        nq += s_w[q];
      }
      if (kb >= 0) s_q[base + x - 1] = i_is_a ? make_int2(ka, kb) : make_int2(kb, ka);
      __syncthreads();
      for (int g0 = 0; g0 < nq; g0 += 4, batch++) {
        unsigned *cnt = s_n + 4 * (batch & 1);
        if (t < 4) s_n[4 * ((batch + 1) & 1) + t] = 0; // the other parity: last read before the previous batch's barrier
        if (g0 + grp < nq) {
          const int2 e = s_q[g0 + grp];
          const double ci = S.X[i][(size_t)e.x * 64 + cell], cj = S.X[j][(size_t)e.y * 64 + cell];
          double v[14] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
          if (!(ci <= 0.0 || cj <= 0.0)) { // main.cpp:6764
            const int id = S.ids[i][e.x];
            const double h = hb[id];
            const int2 b = ij[id];
            const double p0 = (double)(b.x * CUP2D_BS) * h + h * (ix + 0.5), p1 = (double)(b.y * CUP2D_BS) * h + h * (iy + 0.5);
            co_cell(ci, S.dist[i] + (size_t)e.x * 64, reinterpret_cast<const double2 *>(S.udef[i])[(size_t)e.x * 64 + cell], mo[i],
                    p0, p1, ix, iy, v);
            co_cell(cj, S.dist[j] + (size_t)e.y * 64, reinterpret_cast<const double2 *>(S.udef[j])[(size_t)e.y * 64 + cell], mo[j],
                    p0, p1, ix, iy, v + 7);
            atomicAdd(&cnt[grp], 1u);
          }
          for (int q = 0; q < 14; q++) s_v[q * CO_NT + t] = v[q];
        }
        __syncthreads();
        if (t < 14) {
          const double *sv = s_v + t * CO_NT;
          for (int g = 0; g < 4 && g0 + g < nq; g++)
            if (cnt[g])
              for (int c = 0; c < 64; c++) acc += sv[g * 64 + c];
        }
        __syncthreads();
      }
    }
  }
  // the 20 slots of main.cpp:6814-6837: {M, PosX, PosY, PosZ, MomX, MomY, MomZ, vecX, vecY, vecZ} of i, then of the partners
  const int slot[7] = {0, 1, 2, 4, 5, 7, 8}, zslot[6] = {3, 6, 9, 13, 16, 19};
  if (t < 14) sums[(size_t)i * 20 + (t / 7) * 10 + slot[t % 7]] = acc;
  else if (t < 20) sums[(size_t)i * 20 + zslot[t - 14]] = 0.0;
}

// ---- the pair loop (main.cpp:6863-6943) and collision() / compute_j() (209-291), restated on the host ----
static void co_cross(const double a[3], const double b[3], double r[3]) {
  r[0] = a[1] * b[2] - a[2] * b[1];
  r[1] = a[2] * b[0] - a[0] * b[2];
  r[2] = a[0] * b[1] - a[1] * b[0];
}
static double co_dot(const double a[3], const double b[3]) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// J = I^-1 ((Rc - R) x N) for the inertia tensor I = {{1, 0, 0}, {0, 1, 0}, {0, 0, Iz}}, inverted as a general symmetric 3x3
// matrix (adjugate times the reciprocal determinant), which is what fixes the rounding
static void co_angular(const double Rc[3], const double R[3], const double N[3], double Iz, double J[3]) {
  const double m00 = 1.0, m01 = 0.0, m02 = 0.0, m11 = 1.0, m12 = 0.0, m22 = Iz;
  double c00 = m22 * m11 - m12 * m12, c01 = m02 * m12 - m22 * m01, c02 = m01 * m12 - m02 * m11;
  double c11 = m22 * m00 - m02 * m02, c12 = m01 * m02 - m00 * m12, c22 = m00 * m11 - m01 * m01;
  const double rdet = 1.0 / ((m00 * c00) + (m01 * c01) + (m02 * c02));
  c00 *= rdet, c01 *= rdet, c02 *= rdet, c11 *= rdet, c12 *= rdet, c22 *= rdet;
  const double d[3] = {Rc[0] - R[0], Rc[1] - R[1], Rc[2] - R[2]};
  double q[3];
  co_cross(d, N, q);
  J[0] = c00 * q[0] + c01 * q[1] + c02 * q[2];
  J[1] = c01 * q[0] + c11 * q[1] + c12 * q[2];
  J[2] = c02 * q[0] + c12 * q[1] + c22 * q[2];
}

// the impulse of a perfectly elastic contact (e = 1) at C with normal N between bodies 1 and 2: v, o (linear and angular
// velocity), C1 / C2 (centres of mass), vc (the overlap's mean velocity) -> hv, ho
static void co_impulse(double m1, double m2, double Iz1, double Iz2, const double v1[3], const double v2[3], const double o1[3],
                       const double o2[3], const double C1[3], const double C2[3], const double N[3], const double C[3],
                       const double vc1[3], const double vc2[3], double hv1[3], double hv2[3], double ho1[3], double ho2[3]) {
  const double e = 1.0;
  const double k1[3] = {N[0] / m1, N[1] / m1, N[2] / m1}, k2[3] = {-N[0] / m2, -N[1] / m2, -N[2] / m2};
  double J1[3], J2[3];
  co_angular(C, C1, N, Iz1, J1);
  co_angular(C, C2, N, Iz2, J2);
  for (int q = 0; q < 3; q++) J2[q] = -J2[q];
  const double d1[3] = {C[0] - C1[0], C[1] - C1[1], C[2] - C1[2]}, d2[3] = {C[0] - C2[0], C[1] - C2[1], C[2] - C2[2]};
  double w1[3], w2[3]; // o x (C - Ci): the rotational velocity at the contact
  co_cross(o1, d1, w1);
  co_cross(o2, d2, w2);
  double u1[3], u2[3], dv[3], dvc[3];
  for (int q = 0; q < 3; q++) {
    u1[q] = vc1[q] - v1[q] - w1[q];
    u2[q] = vc2[q] - v2[q] - w2[q];
    dvc[q] = vc1[q] - vc2[q];
    dv[q] = v1[q] - v2[q] + u1[q] - u2[q];
  }
  const double nom = e * co_dot(dvc, N) + co_dot(dv, N) + co_dot(w1, N) - co_dot(w2, N);
  const double mN[3] = {-N[0], -N[1], -N[2]};
  double x1[3], x2[3];
  co_cross(J1, d1, x1);
  co_cross(J2, d2, x2);
  const double denom = -(1.0 / m1 + 1.0 / m2) + co_dot(x1, mN) - co_dot(x2, mN);
  const double impulse = nom / (denom + 1e-21);
  for (int q = 0; q < 3; q++) {
    hv1[q] = v1[q] + k1[q] * impulse;
    hv2[q] = v2[q] + k2[q] * impulse;
    ho1[q] = o1[q] + J1[q] * impulse;
    ho2[q] = o2[q] + J2[q] * impulse;
  }
}

// main.cpp:6863-6943 on one thread: pairs i < j in order, each seeing the motion earlier pairs left
static void co_pairs(int n, const double *s, cup2d_rigid *R) {
  for (int i = 0; i < n; i++)
    for (int j = i + 1; j < n; j++) {
      const double *c = s + 20 * i, *co = s + 20 * j; // collisions[i], collisions[j]
      if (c[0] < 2.0 || c[10] < 2.0) continue;
      if (co[0] < 2.0 || co[10] < 2.0) continue;
      if (std::fabs(c[1] / c[0] - co[1] / co[0]) > R[i].length || std::fabs(c[2] / c[0] - co[2] / co[0]) > R[i].length) continue;
      const double *iv = c + 7, *jv = c + 17;
      const double norm_i = std::sqrt(co_dot(iv, iv)), norm_j = std::sqrt(co_dot(jv, jv));
      const double m[3] = {iv[0] / norm_i - jv[0] / norm_j, iv[1] / norm_i - jv[1] / norm_j, iv[2] / norm_i - jv[2] / norm_j};
      const double inorm = 1.0 / std::sqrt(co_dot(m, m));
      const double N[3] = {m[0] * inorm, m[1] * inorm, m[2] * inorm};
      const double vc1[3] = {c[4] / c[0], c[5] / c[0], c[6] / c[0]}, vc2[3] = {c[14] / c[10], c[15] / c[10], c[16] / c[10]};
      const double hit[3] = {vc2[0] - vc1[0], vc2[1] - vc1[1], vc2[2] - vc1[2]};
      if (co_dot(hit, N) <= 0) continue;
      const double inv_iM = 1.0 / c[0], inv_jM = 1.0 / c[10];
      const double C[3] = {0.5 * (c[1] * inv_iM + c[11] * inv_jM), 0.5 * (c[2] * inv_iM + c[12] * inv_jM),
                           0.5 * (c[3] * inv_iM + c[13] * inv_jM)};
      const double v1[3] = {R[i].u, R[i].v, 0.0}, v2[3] = {R[j].u, R[j].v, 0.0};
      const double o1[3] = {0, 0, R[i].omega}, o2[3] = {0, 0, R[j].omega};
      const double C1[3] = {R[i].center_of_mass[0], R[i].center_of_mass[1], 0}, C2[3] = {R[j].center_of_mass[0], R[j].center_of_mass[1], 0};
      double hv1[3], hv2[3], ho1[3], ho2[3];
      co_impulse(R[i].M, R[j].M, R[i].J, R[j].J, v1, v2, o1, o2, C1, C2, N, C, vc1, vc2, hv1, hv2, ho1, ho2);
      R[i].u = hv1[0], R[i].v = hv1[1], R[i].omega = ho1[2];
      R[j].u = hv2[0], R[j].v = hv2[1], R[j].omega = ho2[2];
    }
}

static int co_grow(void **p, size_t *cap, size_t bytes) {
  if (bytes <= *cap) return CUP2D_OK;
  cudaFree(*p);
  *p = nullptr, *cap = 0;
  CUP2D_CUDA(cudaMalloc(p, bytes));
  *cap = bytes;
  return CUP2D_OK;
}

} // namespace cup2d

using namespace cup2d;

extern "C" {

int cup2d_amr_shape_set_dist(cup2d_amr *a, int shape, const double *dist) {
  if (!a || shape < 0 || shape >= (int)a->shapes.size()) {
    set_error("cup2d_amr_shape_set_dist: no such shape (cup2d_amr_shape_set first)");
    return CUP2D_EINVAL;
  }
  cup2d_amr::Shape &sh = a->shapes[shape];
  if (sh.nob > 0 && !dist) {
    set_error("cup2d_amr_shape_set_dist: null dist");
    return CUP2D_EINVAL;
  }
  CUP2D_CUDA(cudaSetDevice(a->device));
  if (!sh.d_dist && sh.cap > 0) CUP2D_CUDA(cudaMalloc(&sh.d_dist, (size_t)sh.cap * 64 * sizeof(double)));
  if (sh.nob > 0) {
    CUP2D_CUDA(cudaMemcpyAsync(sh.d_dist, dist, (size_t)sh.nob * 64 * sizeof(double), cudaMemcpyHostToDevice, a->stream));
    CUP2D_CUDA(cudaStreamSynchronize(a->stream)); // the caller's array may be pageable and short-lived
  }
  sh.has_dist = true;
  return CUP2D_OK;
}

int cup2d_amr_collide(cup2d_amr *a, int nshapes, cup2d_rigid *shapes, double *sums20) {
  if (!a || nshapes < 1 || nshapes > CO_MAXSH || !shapes) {
    set_error("cup2d_amr_collide: bad arguments (1..64 shapes)");
    return CUP2D_EINVAL;
  }
  if (a->dist || a->nranks > 1) {
    set_error("cup2d_amr_collide: contexts on several ranks are not supported");
    return CUP2D_ESTATE;
  }
  for (int s = 0; s < nshapes; s++) {
    if (s >= (int)a->shapes.size()) {
      set_error("cup2d_amr_collide: shape " + std::to_string(s) + " has not been set");
      return CUP2D_EINVAL;
    }
    if (!a->shapes[s].ascending) {
      set_error("cup2d_amr_collide: the block ids of shape " + std::to_string(s) + " are not strictly ascending");
      return CUP2D_EINVAL;
    }
    if (!a->shapes[s].has_dist) {
      set_error("cup2d_amr_collide: shape " + std::to_string(s) + " has no dist (cup2d_amr_ongrid or cup2d_amr_shape_set_dist)");
      return CUP2D_ESTATE;
    }
  }
  // staged tables: motions [n], pair index [n][n], pairs
  std::vector<CoMotion> mo(nshapes);
  for (int s = 0; s < nshapes; s++)
    mo[s] = CoMotion{shapes[s].u, shapes[s].v, shapes[s].omega, shapes[s].center_of_mass[0], shapes[s].center_of_mass[1]};
  std::vector<int> pidx((size_t)nshapes * nshapes, -1);
  std::vector<CoPair> pairs;
  int total = 0;
  for (int i = 0; i < nshapes; i++)
    for (int j = i + 1; j < nshapes; j++) {
      const int ni = a->shapes[i].nob, nj = a->shapes[j].nob;
      if (ni == 0 || nj == 0) continue;
      pidx[(size_t)i * nshapes + j] = pidx[(size_t)j * nshapes + i] = (int)pairs.size();
      pairs.push_back(ni <= nj ? CoPair{i, j, ni, nj, total} : CoPair{j, i, nj, ni, total});
      total += std::min(ni, nj);
    }
  const size_t b_mo = mo.size() * sizeof(CoMotion), b_pidx = pidx.size() * sizeof(int), b_pairs = pairs.size() * sizeof(CoPair);
  std::vector<unsigned char> stage(b_mo + b_pidx + b_pairs);
  memcpy(stage.data(), mo.data(), b_mo);
  memcpy(stage.data() + b_mo, pidx.data(), b_pidx);
  if (b_pairs) memcpy(stage.data() + b_mo + b_pidx, pairs.data(), b_pairs);
  CoShapes S = {};
  for (int s = 0; s < nshapes; s++) {
    const cup2d_amr::Shape &sh = a->shapes[s];
    S.ids[s] = sh.d_ids, S.X[s] = sh.d_X, S.udef[s] = sh.d_udef, S.dist[s] = sh.d_dist;
  }
  CUP2D_CUDA(cudaSetDevice(a->device));
  int rc = amr_ensure_ij(a);
  if (rc || (rc = co_grow((void **)&a->d_co_stage, &a->co_stage_cap, stage.size())) ||
      (rc = co_grow((void **)&a->d_co_match, &a->co_match_cap, (size_t)std::max(total, 1) * sizeof(int))) ||
      (rc = co_grow((void **)&a->d_co_sums, &a->co_sums_cap, (size_t)CO_MAXSH * 20 * sizeof(double))))
    return rc;
  CUP2D_CUDA(cudaMemcpyAsync(a->d_co_stage, stage.data(), stage.size(), cudaMemcpyHostToDevice, a->stream));
  const CoMotion *d_mo = reinterpret_cast<const CoMotion *>(a->d_co_stage);
  const int *d_pidx = reinterpret_cast<const int *>(a->d_co_stage + b_mo);
  const CoPair *d_pairs = reinterpret_cast<const CoPair *>(a->d_co_stage + b_mo + b_pidx);
  if (total > 0) {
    const int grid = std::min((total + CO_MATCH_NT - 1) / CO_MATCH_NT, AMR_GRID_SMS * 8);
    amr_collide_match_kernel<<<grid, CO_MATCH_NT, 0, a->stream>>>(S, d_pairs, (int)pairs.size(), total, a->d_co_match);
  }
  amr_collide_sums_kernel<<<nshapes, CO_NT, 0, a->stream>>>(S, d_mo, d_pidx, d_pairs, nshapes, a->d_co_match,
                                                            reinterpret_cast<const int2 *>(a->d_ij), a->d_h, a->d_co_sums);
  CUP2D_CUDA(cudaGetLastError());
  std::vector<double> sums((size_t)nshapes * 20);
  CUP2D_CUDA(cudaMemcpyAsync(sums.data(), a->d_co_sums, sums.size() * sizeof(double), cudaMemcpyDeviceToHost, a->stream));
  CUP2D_CUDA(cudaStreamSynchronize(a->stream));
  co_pairs(nshapes, sums.data(), shapes);
  if (sums20) std::copy(sums.begin(), sums.end(), sums20);
  return CUP2D_OK;
}

} // extern "C"
