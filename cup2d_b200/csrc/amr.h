// Shared declarations of the multi-level device path (csrc/amr_ops.cu: table-gather baseline; csrc/amr_fast.cu: per-block
// lab loader on the WENO line core).  See amr_ops.cu for the status of this path.
#pragma once
#include <vector>

struct cup2d_amr_plan;
struct cup2d_amr;
extern "C" {
void cup2d_amr_destroy(cup2d_amr *a);
int cup2d_amr_plan_create(int64_t nblocks, const int32_t *level_ij, int32_t bpdx, int32_t bpdy, cup2d_amr_plan **out);
void cup2d_amr_plan_destroy(cup2d_amr_plan *p);
int64_t cup2d_amr_plan_stencil(cup2d_amr_plan *p, int which, int64_t *rowptr, int32_t *src_block, int32_t *src_cellcomp,
                               double *weight);
int64_t cup2d_amr_plan_faces(cup2d_amr_plan *p, int32_t *out);
int64_t cup2d_amr_plan_poisson(cup2d_amr_plan *p, int32_t *nbr_out, int64_t *nnz_out, int32_t *irr_rows, int32_t *irr_rowptr,
                               int32_t *irr_col, double *irr_val);
int cup2d_amr_advect_diffuse_rhs(cup2d_amr *a, double dt);
int cup2d_amr_pressure_rhs(cup2d_amr *a, double dt, int with_laplacian);
int cup2d_amr_pressure_gradient(cup2d_amr *a, double dt);
int cup2d_amr_advect_diffuse_rhs_fast(cup2d_amr *a, double dt);
int cup2d_amr_pressure_rhs_fast(cup2d_amr *a, double dt, int with_laplacian);
int cup2d_amr_pressure_gradient_fast(cup2d_amr *a, double dt);
int cup2d_amr_laplacian_fast(cup2d_amr *a, double dt);
}

namespace cup2d {

constexpr int AMR_GRID_SMS = 132; // SMs of an H100 SXM: the grid-stride launches of this path are capped at a few waves of them

struct Csr {
  int64_t *rowptr = nullptr;
  int *src_block = nullptr, *src_cc = nullptr;
  double *w = nullptr;
  int64_t nrows = 0;
};
struct GhostDev { // compact ghost CSR of one stencil kind on the device
  int64_t *grow = nullptr;    // [nirr+1] first row of every irregular block
  int64_t *rowptr = nullptr;
  int *dst = nullptr, *sb = nullptr, *sc = nullptr;
  double *w = nullptr;
};
struct FluxBuf { // where the face fluxes of the irregular blocks live: per irregular block (position in the irregular list)
  double *p;     // in a buffer of its own, or — distributed contexts — per block inside a field array, so that the
  int stride;    // whole-block halo pulls of the fields carry them across a rank boundary
  int by_block;
};
struct CoarseFace { // one coarse-fine face seen from the coarse side
  int coarse, face, fine[2]; // fine[half] = the fine block abutting that half of the face (-1: absent)
};

} // namespace cup2d

struct cup2d_amr;
// distributed contexts (cup2d_amr_create_ranks): refresh the halo slots of `field` from the owners (whole-block peer pulls,
// csrc/halo.cu) before a kernel reads neighbours; a no-op otherwise
extern "C" int amr_dist_refresh(cup2d_amr *a, int field);
// distributed contexts: v[0..n) summed over all ranks (identical result everywhere); a no-op otherwise
extern "C" int amr_dist_sum(cup2d_amr *a, double *v, int n);
// fast-kernel tables of a distributed context for its block range [b0, b1): slot_of[global block] = local slot or -1
int amr_fast_setup_dist(cup2d_amr *a, const std::vector<int32_t> &slot_of, int64_t b0, int64_t b1);

struct cup2d_amr {
  int64_t nb = 0;
  int device = 0;
  double h0 = 0, nu = 0;
  cup2d_amr_plan *plan = nullptr;
  cudaStream_t stream = nullptr;
  double *f[CUP2D_NFIELDS] = {};
  double *d_h = nullptr;            // cell size per block
  cup2d::Csr csr[4];                // kinds 0-2 at creation, 3 (chi lab of the tagging rule) on first use
  double *lab[4] = {};              // lab buffers per kind; a second kind-1 buffer for u_def
  double *lab_udef = nullptr;
  cup2d::CoarseFace *d_cf[2] = {};  // [0] x faces, [1] y faces
  int ncf[2] = {0, 0};
  double *d_part = nullptr;         // 2 doubles per block (partial maxima / sums)
  std::vector<double> h_part;
  double hmin = 0;
  cup2d_sim *poisson = nullptr;     // general-rows Poisson context over the same blocks (cup2d_amr_poisson_solve)
  // several GPUs (cup2d_amr_set_ranks): operators replicated on every rank, the Poisson solve distributed by block ranges
  int rank = 0, nranks = 1;
  std::vector<int64_t> rank_begin;
  bool dist = false;                // cup2d_amr_create_ranks: this context holds only its own block range (+ halo slots)
  int64_t gbegin = 0, nglobal = 0;  // distributed contexts: first own block in the global list, size of that list
  std::vector<int32_t> slot_of;     // distributed contexts: global block -> local slot (own blocks, then halo slots) or -1
  // fast paths (csrc/amr_fast.cu)
  bool fast = false;                // cup2d_amr_set_fast: the operator entry points dispatch to the fast kernels
  int *d_nbr4 = nullptr;            // [nb][4] W,E,S,N: same-level block, -1 wall, -2 coarser/finer
  int *d_irr_of = nullptr;          // [nb] position in the irregular list or -1
  int64_t nirr = 0;
  cup2d::GhostDev gt[3];            // compact ghost tables per stencil kind (cup2d_amr_plan_ghosts)
  double *d_faceflux = nullptr;     // [nirr][4 faces][8][2] face fluxes of the irregular blocks (single-rank contexts)
  // bodies (csrc/amr_penalize.cu): per-shape obstacle blocks, as cup2d_sim::Shape
  struct Shape { int nob = 0, cap = 0; int *d_ids = nullptr; double *d_X = nullptr, *d_udef = nullptr; };
  std::vector<Shape> shapes;
  std::vector<int32_t> h_ij;        // [nb][2] block index (i, j) at the block's own level (filled by cup2d_amr_create)
  int *d_ij = nullptr;              // the same on the device (first use)
  double *d_shape_part = nullptr;   // [cap][7] per-obstacle-block partial sums
  int shape_part_cap = 0;
  std::vector<double> h_shape_part;
  void free_shapes() {
    for (auto &sh : shapes) {
      cudaFree(sh.d_ids); cudaFree(sh.d_X); cudaFree(sh.d_udef);
    }
    shapes.clear();
    cudaFree(d_ij); cudaFree(d_shape_part);
    d_ij = nullptr, d_shape_part = nullptr, shape_part_cap = 0;
  }
};

