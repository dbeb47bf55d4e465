// Shared declarations of the multi-level device path (csrc/amr_ops.cu: table-gather baseline; csrc/amr_fast.cu: per-block
// lab loader on the WENO line core).  See amr_ops.cu for the status of this path.
#pragma once
#include <algorithm>
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
int cup2d_amr_create(int64_t nblocks, const int32_t *level_ij, int32_t bpdx, int32_t bpdy, double h0, double nu,
                     int32_t device, cup2d_amr **out);
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

// One shape's obstacle blocks on the device (cup2d_shape_set, cup2d_amr_shape_set; csrc/penalize.cu): the ids of the nob
// blocks its body touches, per block its chi X[8][8] and u_def[8][8][2]; room for cap blocks.  Kept here, not in sim.h, so
// that cup2d_amr::Shape below can extend it where only this header is seen.
struct Shape { int nob = 0, cap = 0; int *d_ids = nullptr; double *d_X = nullptr, *d_udef = nullptr; };
inline void shape_free(Shape &sh) { cudaFree(sh.d_ids); cudaFree(sh.d_X); cudaFree(sh.d_udef); }

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
// A scalar argument of a multi-level kernel (dt, a pressure mean): by value, as the blocking calls pass it, or read from
// device memory that an earlier kernel of the same enqueued step wrote (cup2d_amr_step_enqueue).  A kernel resolves it once,
// then computes exactly what it computes from a double; ByValue is passed and read like one.
struct ByValue {
  double v;
  __device__ __forceinline__ double get() const { return v; }
};
struct OnDevice {
  const double *p;
  __device__ __forceinline__ double get() const { return *p; }
};
// launch(ByValue{v}) or, with a device address, launch(OnDevice{p})
template <class F> inline int with_scalar(double v, const double *p, F &&launch) {
  return p ? launch(OnDevice{p}) : launch(ByValue{v});
}
// the record an enqueued step keeps on the device: its dt, the two h^2-weighted pressure means
enum { AMR_REC_DT = 0, AMR_REC_MEAN0 = 1, AMR_REC_MEAN1 = 2, AMR_REC_N = 4 };

// lab entries per block of the compact ghost kinds 0-3 and 6 (cup2d_amr_plan_ghosts: dst = irregular position * this + entry)
constexpr int GHOST_NCELL[7] = {14 * 14 * 2, 10 * 10 * 2, 10 * 10, 16 * 16, 0, 0, 16 * 16 * 2};

// h into a new device buffer of at least one element
template <class T> inline cudaError_t upload(T **d, const std::vector<T> &h) {
  const cudaError_t e = cudaMalloc(d, std::max<size_t>(h.size(), 1) * sizeof(T));
  if (e != cudaSuccess) return e;
  return cudaMemcpy(*d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice);
}

// The plan's tables on the host (csrc/amr_fast.cu), blocks named by their position in the whole list
struct PlanGhosts { // cup2d_amr_plan_ghosts of one kind
  std::vector<int64_t> rowptr;
  std::vector<int32_t> dst, sb, sc;
  std::vector<double> w;
};
int plan_ghosts(cup2d_amr *a, int which, PlanGhosts &g);
int plan_neighbours(cup2d_amr *a, std::vector<int32_t> &n8); // [nglobal][8], cup2d_amr_plan_neighbours
std::vector<int32_t> plan_irregular(cup2d_amr *a);
std::vector<int32_t> plan_faces(cup2d_amr *a);                // [faces][5], cup2d_amr_plan_faces

} // namespace cup2d

// the dt-dependent operators with dt by value (ddt = nullptr) or from the device record of an enqueued step (csrc/amr_fast.cu)
int amr_advect_rhs_fast(cup2d_amr *a, double dt, const double *ddt);
int amr_pressure_rhs_fast(cup2d_amr *a, double dt, int with_laplacian, const double *ddt);
int amr_pressure_gradient_fast(cup2d_amr *a, double dt, const double *ddt);

// the plan's block list, [n][3] (level, i, j), and its level-0 blocks per direction
const std::vector<int> &amr_plan_level_ij(const cup2d_amr_plan *p, int *bpdx, int *bpdy);
// full lab rows (as cup2d_amr_plan_stencil) of the blocks `blocks[0..nsub)` only, in that order (csrc/amr_regrid.cu)
int amr_plan_subset_rows(cup2d_amr_plan *p, int which, int64_t nsub, const int32_t *blocks, std::vector<int64_t> &rowptr,
                         std::vector<int32_t> &src_block, std::vector<int32_t> &src_cellcomp, std::vector<double> &weight);

struct cup2d_amr;
// adapt()'s tagging (cup2d_amr_adapt_tags) enqueued on the context's stream: the tagging field in tmp, the per-block L-inf in
// d_part[0..nb) (csrc/amr_ops.cu)
extern "C" int amr_adapt_tags_enqueue(cup2d_amr *a, double rtol, int level_max);
// the fast path's neighbour / irregular-block / compact ghost tables of kinds 0-2 (csrc/amr_fast.cu): amr_fast_tables builds
// them on first use on a single-rank context (a no-op on a distributed one), amr_fast_build builds them now
int amr_fast_tables(cup2d_amr *a);
int amr_fast_build(cup2d_amr *a);
// the compact ghost rows of stencil kind `which` of the context's irregular blocks into gt[which], every source by its slot
// (csrc/amr_fast.cu); CUP2D_EINVAL if a source is not a halo slot.  source_order: into gt_src[which] instead, each row's
// terms in the order of the full per-cell tables
int amr_ghost_rows(cup2d_amr *a, int which, bool source_order = false);
// the tables of the 16 x 16 chi / vel labs on first use (csrc/amr_fast.cu): the fast tables, d_nbr8 and gt[3]
int amr_lab16_tables(cup2d_amr *a);
// adapt()'s tagging on the fast kernels (csrc/amr_fast.cu): tmp and d_part as amr_adapt_tags_enqueue leaves them, from the
// fast tables, d_nbr8 and the compact rows of kinds 1 and 3; h_finest is the cell size of level level_max - 1
int amr_tags_fast(cup2d_amr *a, double rtol, double h_finest);
// the per-block (i, j) table on the device, built on first use (csrc/penalize.cu)
int amr_ensure_ij(cup2d_amr *a);
// distributed contexts (cup2d_amr_create_ranks): refresh the halo slots of `field` from the owners (whole-block peer pulls,
// csrc/halo.cu) before a kernel reads neighbours; a no-op otherwise
extern "C" int amr_dist_refresh(cup2d_amr *a, int field);
// distributed contexts: v[0..n) summed over all ranks (identical result everywhere); a no-op otherwise
extern "C" int amr_dist_sum(cup2d_amr *a, double *v, int n);
// distributed contexts on several ranks: the host array v[0..n) summed over all ranks in one launch and one host wait, the
// ranks' values added in rank order, so every rank gets the same bits; CUP2D_ECOMM if the ranks pass different n or a peer
// never arrives.  A no-op otherwise (one rank included).
extern "C" int amr_dist_sum_vec(cup2d_amr *a, double *v, int n);

struct cup2d_amr {
  int64_t nb = 0;
  int device = 0;
  double h0 = 0, nu = 0;
  cup2d_amr_plan *plan = nullptr;
  cudaStream_t stream = nullptr;
  double *f[CUP2D_NFIELDS] = {};
  double *d_h = nullptr;            // cell size per block
  cup2d::Csr csr[4];                // full per-cell tables of the baseline kernels (kind 3: the tagging rule's chi lab), each
                                    // on first use by a baseline-mode context; fast and distributed contexts never build them
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
  int64_t gbegin = 0, nglobal = 0;  // the context's blocks are [gbegin, gbegin + nb) of the plan's list of nglobal blocks
  std::vector<int32_t> slot_of;     // distributed contexts: global block -> local slot (own blocks, then halo slots) or -1
  int32_t slot(int64_t g) const { return dist ? slot_of[g] : (int32_t)g; } // where block g of the list lives here, or -1
  // fast paths (csrc/amr_fast.cu)
  bool fast = false;                // cup2d_amr_set_fast: the operator entry points dispatch to the fast kernels
  int *d_nbr4 = nullptr;            // [nb][4] W,E,S,N: same-level block, -1 wall, -2 coarser/finer
  int *d_irr_of = nullptr;          // [nb] position in the irregular list or -1
  int64_t nirr = 0;
  cup2d::GhostDev gt[7];            // compact ghost tables per stencil kind (amr_ghost_rows): 0-2 with the fast tables,
                                    // 3 (the 16 x 16 chi lab of tagging and forces) and 6 (the forces' vel lab) on first use
  cup2d::GhostDev gt_src[4];        // kinds 1 and 3 with each row's terms in the full tables' order (the tagging kernel)
  int *d_nbr8 = nullptr;            // [nb][8] cup2d_amr_plan_neighbours on the device (amr_lab16_tables, first use)
  double *d_faceflux = nullptr;     // [nirr][4 faces][8][2] face fluxes of the irregular blocks (single-rank contexts)
  // bodies (csrc/penalize.cu): per-shape obstacle blocks, a cup2d::Shape with
  // (d_dist, the signed distance, exists only for shapes placed by cup2d_amr_ongrid or given one by cup2d_amr_shape_set_dist;
  // ascending: the block ids are strictly ascending, recorded by cup2d_amr_shape_set, always true after cup2d_amr_ongrid)
  // (has_surface: cup2d_amr_surface has run on the shape as it stands; cup2d_amr_shape_set and cup2d_amr_ongrid clear it)
  struct Shape : cup2d::Shape { double *d_dist = nullptr; bool has_dist = false, ascending = true, has_surface = false; };
  std::vector<Shape> shapes;
  std::vector<int32_t> h_ij;        // [nb][2] block index (i, j) at the block's own level (filled by cup2d_amr_create)
  int *d_ij = nullptr;              // the same on the device (first use)
  double *d_shape_part = nullptr;   // [cap][7] per-obstacle-block partial sums
  int shape_part_cap = 0;
  std::vector<double> h_shape_part;
  // cup2d_amr_ongrid scratch (csrc/amr_ongrid.cu): staged midlines + segments, block masks, counts / offsets, per-block partials
  double *d_og_stage = nullptr, *d_og_part = nullptr;
  unsigned long long *d_og_mask = nullptr;
  int *d_og_cnt = nullptr;
  size_t og_stage_cap = 0, og_part_cap = 0, og_mask_cap = 0, og_cnt_cap = 0;
  bool og_timing = false, og_timed = false; // cup2d_amr_ongrid_timing: CUDA events (cudaEvent_t) around the kernels of the last call
  void *og_ev[12] = {};
  void (*og_release)(cup2d_amr *) = nullptr; // destroys og_ev (set with them, csrc/amr_ongrid.cu)
  // cup2d_amr_collide scratch (csrc/amr_collide.cu): staged shape / pair tables, per-pair matches, the 20 N sums
  unsigned char *d_co_stage = nullptr;
  int *d_co_match = nullptr;
  double *d_co_sums = nullptr;
  size_t co_stage_cap = 0, co_match_cap = 0, co_sums_cap = 0;
  // cup2d_amr_surface / cup2d_amr_forces (csrc/amr_forces.cu): per shape the surface points of its obstacle blocks, 64 slots
  // per block (slot k * 64 + j = point j of block k): (ix, iy), {dchidx, dchidy, D}, the 14 skin values; counts per block
  struct Surface { int cap = 0; int *d_ixy = nullptr, *d_cnt = nullptr; double *d_nrm = nullptr, *d_skin = nullptr; std::vector<int> cnt; };
  std::vector<Surface> surf;
  double *d_fo_part = nullptr;      // [obstacle blocks][19] per-block accumulators, then [nshapes][19] sums
  size_t fo_part_cap = 0;
  double *d_vsum = nullptr;         // distributed contexts: the values of amr_dist_sum_vec and its status word
  size_t vsum_cap = 0;
  // enqueued steps (cup2d_amr_step_enqueue / _pressure_enqueue, csrc/amr_ops.cu): the device record (AMR_REC_*), the events
  // that join the Poisson context's stream to this one, one executable graph per argument set (cudaGraphExec_t / cudaGraph_t)
  double *d_rec = nullptr;
  void *ev_fork = nullptr, *ev_join = nullptr;
  struct StepGraph { std::vector<unsigned long long> key; void *exec = nullptr, *graph = nullptr; };
  std::vector<StepGraph> graphs;
  bool use_graph = true;            // cup2d_amr_set_graph; stays with the handle across a regrid
  unsigned warmed = 0;              // bit (2 fast + pressure-only): that form has run directly once on this mesh
  bool step_pending = false;        // an enqueued step / pressure section whose result has not been read
  void free_shapes() {
    for (auto &sh : shapes) {
      cup2d::shape_free(sh);
      cudaFree(sh.d_dist);
    }
    shapes.clear();
    cudaFree(d_ij); cudaFree(d_shape_part);
    d_ij = nullptr, d_shape_part = nullptr, shape_part_cap = 0;
    cudaFree(d_og_stage); cudaFree(d_og_part); cudaFree(d_og_mask); cudaFree(d_og_cnt);
    d_og_stage = d_og_part = nullptr, d_og_mask = nullptr, d_og_cnt = nullptr;
    og_stage_cap = og_part_cap = og_mask_cap = og_cnt_cap = 0;
    cudaFree(d_co_stage); cudaFree(d_co_match); cudaFree(d_co_sums);
    d_co_stage = nullptr, d_co_match = nullptr, d_co_sums = nullptr;
    co_stage_cap = co_match_cap = co_sums_cap = 0;
    for (auto &q : surf) {
      cudaFree(q.d_ixy); cudaFree(q.d_cnt); cudaFree(q.d_nrm); cudaFree(q.d_skin);
    }
    surf.clear();
    cudaFree(d_fo_part);
    d_fo_part = nullptr, fo_part_cap = 0;
    if (og_release) og_release(this);
    og_release = nullptr;
    og_timing = og_timed = false;
  }
};

