// Internal state of one cup2d_sim (one process <-> one GPU <-> one contiguous SFC range of blocks).
#pragma once
#include "../../include/cup2d_b200.h"
#include "common.cuh"
#include "rows.cuh"
#include "amr.h" // the multi-level context, and the shape record both contexts keep
#include <mutex>
#include <string>
#include <vector>

#define CUP2D_REQUIRE(cond, msg)                                                                  \
  do {                                                                                            \
    if (!(cond)) {                                                                                \
      cup2d::set_error(msg);                                                                      \
      return CUP2D_EINVAL;                                                                        \
    }                                                                                             \
  } while (0)

namespace cup2d {

constexpr int TILE_B = 4;                // advect tile = 4x4 blocks = 32x32 cells
constexpr int TILE_SLOTS = 32;            // 16 interior + 4 W + 4 E + 4 S + 4 N
constexpr int MAX_RANKS = 8;
constexpr int RED_MAX_CTAS = 4096;        // upper bound on reduction grid size
constexpr int RED_SLOTS = 8;              // doubles per CTA partial

// Device-resident scalars of the Krylov recurrence (cuda.cu:24-34 BiCGSTABScalars, plus the host
// variables of cuda.cu:405-408 moved to the device so that no host sync is needed per iteration).
struct KrylovState {
  double alpha, omega, rho_prev, rho_curr; // recurrence scalars
  double beta;                             // beta for the next p-update
  double nr2, nrh2;                        // |r|^2, |rhat|^2 (breakdown test, cuda.cu:452-454)
  double rhat_nu;                          // rhat . nu
  double tr, tt;                           // t.r, t.t
  double err, err_init, err_opt;           // ||r||_inf now / initially / best
  double xsum;                             // sum of the returned iterate (pressure mean, main.cpp:7126-7148)
  double tol_abs, tol_rel;
  int max_restarts, max_iter;
  int iter;                                // completed iterations
  int restarts;
  int done;                                // 1: stop (converged / restart cap / max_iter)
  int restart_now;                         // 1: next p-update performs the restart of cuda.cu:457-477
  int cur, opt;                            // which of the 3 x buffers holds x / x_opt
  int x0_zero;                             // 1: the solve started from x0 = +0 (x of iteration 0 need not be read)
};

// dt-dependent factors of the current time step, device-resident (k_step_factors): a step captured in a CUDA graph
// reads them from here, so neither dt nor anything derived from it is baked into the graph
struct StepFactors {
  double dt, umax;
  double afac, dfac;   // advect-diffuse: -dt h, nu dt                     (main.cpp:5446-5447)
  double rhs_fac;      // Poisson right-hand side: 0.5 h / dt               (main.cpp:6119)
  double corr_fac;     // pressure correction: (-0.5 dt h) / h^2            (main.cpp:6028, 7182)
};

struct PeerBlob { // what every rank publishes to the others (cup2d_peer_export)
  cudaIpcMemHandle_t field[CUP2D_NFIELDS];
  cudaIpcMemHandle_t kz, kx[3], kzr;
  cudaIpcMemHandle_t mailbox;
  cudaIpcMemHandle_t halo_gid; // global ids of this rank's halo slots (read once by the peers at attach time)
  int64_t nloc, nhalo;
  int32_t rank, device;
};

// Constant memory and function attributes are per-DEVICE state: a call site that sets them up once keeps one of these and
// runs its setup once per device ordinal (one process may drive several devices).
struct PerDeviceOnce {
  std::mutex m;
  unsigned long long seen = 0;
  template <class F> int run(int device, F &&setup) {
    std::lock_guard<std::mutex> g(m);
    const unsigned long long bit = 1ull << (device & 63);
    if (seen & bit) return CUP2D_OK;
    const int rc = setup();
    if (rc == CUP2D_OK) seen |= bit;
    return rc;
  }
};

} // namespace cup2d

struct cup2d_sim {
  // topology
  int nbx = 0, nby = 0;
  int64_t nglobal = 0, gbegin = 0, nloc = 0, nhalo = 0, nslots = 0;
  int rank = 0, nranks = 1, device = 0;
  double h = 0, nu = 0, cfl = 0;
  std::vector<int32_t> ij;             // global (i,j) table
  std::vector<int64_t> rank_begin;
  std::vector<int32_t> halo_gid;       // global id of every halo slot (slot = nloc + k), sorted
  std::vector<int32_t> halo_owner;     // owning rank per halo slot
  std::vector<int> h_nbr, h_tiles, h_torg, h_halo_src; // host copies of the device tables
  bool poisson_only = false;           // created by cup2d_poisson_create: neighbour table only, no tiles
  bool plan_only = false;              // created by cup2d_plan_create: topology only, no CUDA state
  cudaStream_t stream = nullptr;
  // device tables
  int *d_nbr = nullptr;                // [nloc][4] slots of W,E,S,N neighbours, -1 = wall
  int *d_tiles = nullptr;              // [ntiles][TILE_SLOTS]
  int *d_tile_org = nullptr;           // [ntiles][2] tile origin in blocks
  int ntiles = 0;
  double *d_linf = nullptr;            // per-block L-inf of the tagging field (cup2d_adapt_tags)
  int *d_ij = nullptr;                 // (i,j) of the local blocks (cup2d_dump)
  // fields (dim*64*nslots doubles each)
  double *f[CUP2D_NFIELDS] = {};
  // Krylov vectors (64*nslots)
  double *kx[3] = {}, *kr = nullptr, *krhat = nullptr, *kp = nullptr, *knu = nullptr, *kt = nullptr,
         *kz = nullptr, *kzr = nullptr; // kz = M p, kzr = M r
  cup2d::KrylovState *d_state = nullptr, *h_state = nullptr;
  // reductions
  double *d_partials = nullptr;
  unsigned int *d_counter = nullptr;
  double *d_scal = nullptr, *h_scal = nullptr; // small scalar mailbox (umax, sums)
  cup2d::StepFactors *d_fac = nullptr, *h_fac = nullptr; // factors of the current step (device) / pinned read-back
  int num_sms = 0;
  // multi-GPU (peer memory over NVLink)
  bool peers_attached = false;
  void *peer_base[cup2d::MAX_RANKS][CUP2D_NFIELDS + 5] = {}; // fields, kz, kx[3], kzr
  int *d_halo_src = nullptr;           // [nhalo][2] = (owner rank, slot on owner)
  int *d_halo_gid = nullptr;           // [nhalo] global block id of every halo slot (exported to the peers)
  unsigned src_mask = 0, dst_mask = 0; // ranks this rank pulls halo blocks from / ranks that pull from this rank
  int *d_push_first = nullptr;         // [nloc] first entry of the block in d_push_ent, -1: no peer has it as a halo slot
  int2 *d_push_ent = nullptr;          // (peer rank, halo slot on that peer) ..., (-1,-1) ends a block's list
  int64_t n_push = 0;
  unsigned long long *d_mailbox = nullptr;       // this rank's flag/scalar mailbox (peer-writable)
  unsigned long long *peer_mailbox[cup2d::MAX_RANKS] = {};
  unsigned long long epoch = 0;
  cup2d::Comm comm = {};               // by-value kernel argument of every reducing kernel
  // general (non-stencil) Poisson rows: CSR side table (cup2d_poisson_create_general)
  int *d_irr_blk = nullptr, *d_irr_tab = nullptr, *d_irr_rowptr = nullptr, *d_irr_col = nullptr;
  double *d_irr_val = nullptr;
  int64_t n_irr_rows = 0;
  // bodies: per-shape obstacle blocks on the device (cup2d_shape_set)
  std::vector<cup2d::Shape> shapes;
  // host-buffer pipeline (cup2d_pipe_*): staging sets, copy streams, ordering events
  struct PipeSet { double *vel = nullptr, *pres = nullptr; cudaEvent_t in_done = nullptr, step_done = nullptr, out_done = nullptr; };
  PipeSet pipe[CUP2D_PIPE_SLOTS];
  cudaStream_t pipe_in = nullptr, pipe_out = nullptr;
  int64_t launches = 0;
  // optional per-kernel-class CUDA-event instrumentation (cup2d_profile_*)
  bool prof_on = false;
  struct ProfRec { int cls; cudaEvent_t a, b; };
  std::vector<ProfRec> prof;          // records since cup2d_profile_enable(1)
  std::vector<cudaEvent_t> prof_pool; // events are created once and reused: no cudaEventCreate inside a timed region
  size_t prof_pool_used = 0;
  // whole-step CUDA graphs (cup2d_step_enqueue): one executable graph per (buffer assignment, arguments)
  struct StepGraph { std::vector<unsigned long long> key; cudaGraphExec_t exec = nullptr; cudaGraph_t graph = nullptr; int64_t launches = 0; };
  std::vector<StepGraph> graphs;
  bool use_graph = true, warmed = false;
  cudaStream_t body_stream = nullptr;             // captures the body of the Krylov WHILE node
  unsigned long long cond_handle = 0;             // cudaGraphConditionalHandle of the loop being captured (0: none)
  bool step_pending = false;                      // a step was enqueued whose result has not been read
};

namespace cup2d {
enum KClass { KC_ADVECT = 0, KC_UMAX, KC_RHS, KC_CORRECT, KC_KINIT, KC_PUPDATE, KC_SPMV_NU, KC_XRUPDATE,
              KC_SPMV_T, KC_FINAL, KC_P_SPMV, KC_R_SPMV, KC_X_FINAL, KC_HALO, KC_VORT, KC_RHS_START, KC_COUNT };
// bracket one launch with events when profiling is on (no-op otherwise)
struct ProfScope {
  cup2d_sim *s;
  int idx = -1;
  ProfScope(cup2d_sim *sim, int cls) : s(sim) {
    if (!s->prof_on) return;
    cup2d_sim::ProfRec r;
    r.cls = cls;
    while (s->prof_pool.size() < s->prof_pool_used + 2) {
      cudaEvent_t e;
      cudaEventCreate(&e);
      s->prof_pool.push_back(e);
    }
    r.a = s->prof_pool[s->prof_pool_used++];
    r.b = s->prof_pool[s->prof_pool_used++];
    cudaEventRecord(r.a, s->stream);
    s->prof.push_back(r);
    idx = (int)s->prof.size() - 1;
  }
  ~ProfScope() {
    if (idx >= 0) cudaEventRecord(s->prof[idx].b, s->stream);
  }
};
int dim_of(int field);
inline IrrView irr_view(const cup2d_sim *s) {
  IrrView v;
  if (s->n_irr_rows > 0) {
    v.blk = s->d_irr_blk; v.tab = s->d_irr_tab; v.rowptr = s->d_irr_rowptr; v.col = s->d_irr_col; v.val = s->d_irr_val;
  }
  return v;
}
// operators (host-side launchers; all on s->stream)
int launch_advect(cup2d_sim *s, const double *in, const double *old, double *out, double coef,
                  double dt, bool raw, const StepFactors *dev = nullptr);
int launch_umax(cup2d_sim *s, double *umax_out);
int launch_umax_async(cup2d_sim *s);                      // umax -> d_scal[0], no host synchronisation
int launch_step_factors(cup2d_sim *s, double dt_host);    // d_fac from dt_host (> 0) or from d_scal[0] (the dt rule on the device)
int launch_pressure_rhs(cup2d_sim *s, double dt, bool has_udef); // tmp = b, pres = 0 (cup2d_pressure_rhs)
int pressure_rhs_inputs(cup2d_sim *s, bool has_udef);              // pold <- pres, halo refreshes of vel, tmpV, pold
int launch_pressure_correct(cup2d_sim *s, double dt, const StepFactors *dev = nullptr, bool pold_halo_current = false);
int launch_adapt_tags(cup2d_sim *s, double rtol, int chi_cells, double *linf_host);
int dump_fields(cup2d_sim *s, double time, const char *path);
int ensure_block_ij(cup2d_sim *s);
int shape_set(cup2d_sim *s, int shape, int nob, const int32_t *ids, const double *X, const double *udef);
void shapes_free(cup2d_sim *s);
int shape_integrals(cup2d_sim *s, int shape, double lambda, double dt, double cx, double cy, double *out);
int shape_penalize(cup2d_sim *s, int shape, double lambda, double dt, double cx, double cy, double us, double vs,
                   double omega);
int udef_assemble(cup2d_sim *s);
int poisson_solve(cup2d_sim *s, double tol_abs, double tol_rel, int max_restarts, int max_iter, int *iters, double *err);
int poisson_begin(cup2d_sim *s, double tol_abs, double tol_rel, int max_restarts, int max_iter);
// The right-hand side of a time step (vel, tmpV = u_def if has_udef, chi, pold; factor from dev) as the start of its solve
struct StepRhs {
  bool has_udef;
  const StepFactors *dev;
};
int poisson_begin_rhs(cup2d_sim *s, double tol_abs, double tol_rel, int max_restarts, int max_iter, const StepRhs &rhs);
int poisson_iterations(cup2d_sim *s, int n, cudaStream_t stream);
int poisson_result(cup2d_sim *s, int *iters, double *err);
// begin + iterations of an enqueued solve (csrc/api.cu): a WHILE node while capturing a tolerance-driven solve, else launches.
// rhs: start from a time step's right-hand side (poisson_begin_rhs); null: from b = tmp and x0 = pres (poisson_begin)
int poisson_enqueue(cup2d_sim *s, double tol_abs, double tol_rel, int max_restarts, int max_iter, bool capturing,
                    const StepRhs *rhs = nullptr);
int halo_exchange_ptr(cup2d_sim *s, double *base, int dim, int peer_index, bool done_barrier = true);
int halo_exchange_xopt(cup2d_sim *s); // halo of the x buffer KrylovState::opt names (chosen on the device)
int comm_check(cup2d_sim *s);         // CUP2D_ECOMM if a cross-GPU wait of this rank was given up
void swap_fields(cup2d_sim *s, int a, int b); // pointer swap, mirrored on the peer mappings
int poisson_create_general_ranks_ex(int64_t nblocks_global, int32_t rank, int32_t nranks, const int64_t *rank_begin,
                                    const int32_t *nbr, int64_t n_irr, const int32_t *irr_rows, const int32_t *irr_rowptr,
                                    const int32_t *irr_col, const double *irr_val, int64_t n_extra,
                                    const int32_t *extra_blocks, int32_t device, cup2d_sim **out);
} // namespace cup2d
