/* cup2d_b200 — C ABI of the CUDA-native (H100, sm_90a) CUP2D hot path (libcup2d_b200.so).
 *
 * Plain pointers and sizes only; no C++/torch types cross this boundary.  Every entry point
 * returns 0 on success and a negative CUP2D_E* code on failure; cup2d_last_error() gives the
 * message (the reference itself has no error convention: CUDA errors are swallowed, cuda.cu:358;
 * this library fails loudly instead).
 *
 * What each group replaces in the reference (slitvinov/CUP2D, file:line):
 *   grid / fields   Grid, Info, var.{vel,vold,tmpV,chi,pres,pold,tmp}     main.cpp:504-512, 2193-2201, 3264-3278, 6508-6541
 *   compute_dt      umax reduction + dt rule                              main.cpp:6579-6595
 *   advect_diffuse  computeA<VectorLab>(KernelAdvectDiffuse) + RK2 loops  main.cpp:5441-5503, 6607-6642, 162-208
 *   pressure_rhs    computeB<pressure_rhs> + pold/pres swap + pressure_rhs1  main.cpp:6105-6139, 6209-6230, 7011-7027
 *   poisson_solve   Solver::getVec + LocalSpMatDnVec::solve* (BiCGSTAB)   main.cpp:5998-6019, 7031-7118; cuda.cu:403-548
 *   pressure_correct mean removal + pressureCorrectionKernel + V update   main.cpp:6021-6043, 7120-7187
 *   halo exchange   sync1/Setup/pack/unpack_subregion                     main.cpp:1971-2142, 909-1380, 58-110
 *
 * Memory layout (kept from the reference so the host driver can hand blocks over unchanged):
 * a field is nblocks_local consecutive 8x8 blocks in the caller's block order (the reference's
 * Hilbert-sorted `infos[]`); cell (ix,iy) component c of block k is at
 *   k*dim*64 + dim*(8*iy+ix) + c        (dim = 2 for vel/vold/tmpV interleaved u,v; 1 otherwise)
 * exactly main.cpp:6517 + 5467-5468.  All arithmetic is FP64 (main.cpp:24 `typedef double Real`).
 */
#ifndef CUP2D_B200_H
#define CUP2D_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define CUP2D_BS 8 /* _BS_, reference Makefile:12 */

enum {
  CUP2D_OK = 0,
  CUP2D_EINVAL = -1,  /* bad argument / unsupported topology */
  CUP2D_ECUDA = -2,   /* CUDA runtime error (message in cup2d_last_error) */
  CUP2D_ENOGPU = -3,  /* no usable sm_90 device: there is NO CPU fallback */
  CUP2D_ESTATE = -4,  /* call made in the wrong state (e.g. multi-rank step before peers attached) */
  CUP2D_ECOMM = -5    /* a cross-GPU wait ran into its time limit (peer dead, or ranks issued different call sequences);
                         the reference aborts through MPI in that situation (SURVEY.md 8(b) error convention) */
};

/* field ids (var.* of main.cpp:3264-3278) */
enum {
  CUP2D_VEL = 0,  /* dim 2 */
  CUP2D_VOLD = 1, /* dim 2 */
  CUP2D_TMPV = 2, /* dim 2 : RK scratch, then sum of u_def (main.cpp:6980-7006) */
  CUP2D_CHI = 3,  /* dim 1 */
  CUP2D_PRES = 4, /* dim 1 */
  CUP2D_POLD = 5, /* dim 1 */
  CUP2D_TMP = 6,  /* dim 1 : Poisson right-hand side */
  CUP2D_NFIELDS = 7
};

typedef struct cup2d_sim cup2d_sim;

typedef struct {
  int32_t nbx, nby;          /* blocks per direction of the (uniform-level) grid: bpd << level */
  int64_t nblocks_global;    /* == nbx*nby */
  const int32_t *block_ij;   /* [2*nblocks_global]: (i,j) = Info::index of every block, in GLOBAL id
                                order (rank 0's infos[], then rank 1's, ... : main.cpp:6494-6504) */
  int32_t rank, nranks;      /* this process / number of processes (one per GPU) */
  const int64_t *rank_begin; /* [nranks+1]: rank r owns global block ids [rank_begin[r], rank_begin[r+1]) */
  double h;                  /* cell size (Info::h) */
  double nu;                 /* sim.nu */
  double cfl;                /* sim.CFL */
  int32_t device;            /* CUDA device ordinal for this process */
  int32_t reserved;
} cup2d_config;

/* ---- lifetime ---- */
int cup2d_create(const cup2d_config *cfg, cup2d_sim **out);
void cup2d_destroy(cup2d_sim *s);
const char *cup2d_last_error(void);
int cup2d_version(void);
int64_t cup2d_nblocks_local(const cup2d_sim *s);
int64_t cup2d_nblocks_halo(const cup2d_sim *s);

/* host helper mirroring SpaceCurve (main.cpp:342-446) for bpdx x bpdy base blocks at `level`:
 * writes (i,j) of all (bpdx<<level)*(bpdy<<level) blocks in the reference's Hilbert id order. */
int cup2d_block_order(int32_t bpdx, int32_t bpdy, int32_t level, int32_t *block_ij_out);

/* ---- fields: host <-> device in the reference block layout (local blocks only) ---- */
int cup2d_field_upload(cup2d_sim *s, int field, const double *host_blocks);
int cup2d_field_download(cup2d_sim *s, int field, double *host_blocks);
int cup2d_field_fill(cup2d_sim *s, int field, double value);
void *cup2d_field_device_ptr(cup2d_sim *s, int field); /* device pointer, same layout (+halo slots after) */
int cup2d_sync(cup2d_sim *s);                          /* cudaStreamSynchronize on the sim's stream */
void *cup2d_stream(cup2d_sim *s);                      /* cudaStream_t all work is launched on */

/* ---- operators; everything stays on the device ---- */
/* umax = max|vel| (all components), dt = min(0.25 h^2/(nu+0.25 h umax), cfl*h/(umax+1e-8)). main.cpp:6579-6595 */
int cup2d_compute_dt(cup2d_sim *s, double *umax_out, double *dt_out);
/* one fused RK stage: out = old + coef * K(in)/h^2, K = KernelAdvectDiffuse (main.cpp:5441-5503).
 * in/old/out are vector field ids; out must differ from in (old may equal in). */
int cup2d_advect_diffuse_stage(cup2d_sim *s, int in_field, int old_field, int out_field, double coef,
                               double dt);
/* raw K(vel) -> tmpV, undivided, exactly what the reference kernel writes (for operator parity tests). */
int cup2d_advect_diffuse_rhs(cup2d_sim *s, int in_field, int out_field, double dt);
/* vold = vel; vel = vold + 0.5 K(vel)/h^2; vel = vold + K(vel)/h^2.  main.cpp:6607-6642 */
int cup2d_advect_diffuse_rk2(cup2d_sim *s, double dt);
/* tmp = (0.5 h/dt)(div vel - chi div tmpV); pold = pres; pres = 0; tmp -= lap(pold).  main.cpp:7011-7027 */
int cup2d_pressure_rhs(cup2d_sim *s, double dt);
/* Solve A x = tmp (A = undivided 5-point Laplacian, Neumann walls), x0 = pres, result -> pres.
 * Block-Jacobi preconditioned BiCGSTAB with the reference's operation order, epsilons, restart and
 * stopping rules (cuda.cu:403-548).  max_iter: cuda.cu:438 hard-codes 1000.  iters/err may be NULL. */
int cup2d_poisson_solve(cup2d_sim *s, double tol_abs, double tol_rel, int max_restarts, int max_iter,
                        int *iters_out, double *err_out);
/* pres = pres - mean(pres); pres += pold - mean(pres); tmpV = -0.5 dt h grad(pres) (undivided);
 * vel += tmpV/h^2.  main.cpp:7120-7187 */
int cup2d_pressure_correct(cup2d_sim *s, double dt);
/* Regridding criterion from device-resident fields = the first two lines of adapt() and its per-block loop
 * (main.cpp:4659-4660, 4676-4680): tmp = KernelVorticity(vel) (main.cpp:3343-3366); if chi_cells > 0, GradChiOnTmp
 * (main.cpp:4631-4656): blocks with chi > 0 within chi_cells cells (reference: 4 on the finest level, else 2) get
 * their 4 centre cells set to 2*rtol; block_linf_out[k] = max|tmp| over local block k, `infos` order (host array of
 * cup2d_nblocks_local doubles, may be NULL).  The caller compares with Rtol / Ctol exactly as main.cpp:4681-4682.
 * Uses the Krylov scratch vector for the chi masks.  cup2d_vorticity_tag(s, out) == cup2d_adapt_tags(s, 0, 0, out). */
int cup2d_adapt_tags(cup2d_sim *s, double rtol, int chi_cells, double *block_linf_out);
int cup2d_vorticity_tag(cup2d_sim *s, double *block_linf_out);
/* dump() (main.cpp:3367-3467): writes <path>.xyz.raw, <path>.attr.raw (float32, cell quads and (u,v,0) in `infos`
 * order; every rank writes its own byte range) and, on the last rank, <path>.xdmf2 — byte-identical to the
 * reference's files (what post.py reads).  The narrowing to float32 happens on the device. */
int cup2d_dump(cup2d_sim *s, double time, const char *path);
/* ---- bodies: the penalisation phase on device-resident fields (main.cpp:6643-6681, 6944-7002) -------------------
 * A shape = the reference's per-shape obstacleBlocks (main.cpp:3283-3286, 4245-4263): nob local block ids (`infos`
 * order) with the shape's own chi[nob][8][8] and udef[nob][8][8][2].  Produced by the host body model every step. */
int cup2d_shape_set(cup2d_sim *s, int shape, int nob, const int32_t *block_ids, const double *chi, const double *udef);
/* main.cpp:6643-6688: out7 = {PM, PJ, PX, PY, UM, VM, AM}, summed over all ranks (every rank must call, also with
 * nob = 0).  The 3x3 solve for (u, v, omega) (6689-6703) stays on the host; the collision model (6704-6943) does too on
 * this uniform context, and runs on the device for multi-level contexts (cup2d_amr_collide). */
int cup2d_shape_integrals(cup2d_sim *s, int shape, double lambda, double dt, double cx, double cy, double *out7);
/* main.cpp:6944-6979: vel = alpha vel + (1-alpha)(us - omega*py + udef_x, vs + omega*px + udef_y) on the cells the
 * shape owns (its chi > 0 and not below the chi field), alpha = 1/(1+lambda*dt) where its chi > 0.5.  Call per shape
 * in the reference's order.  Bit-identical to the reference. */
int cup2d_penalize(cup2d_sim *s, int shape, double lambda, double dt, double cx, double cy, double us, double vs,
                   double omega);
/* main.cpp:6980-7002: tmpV = 0, then += udef of every shape (index order) where its chi is not below the chi field:
 * the u_def input of cup2d_pressure_rhs.  Bit-identical to the reference. */
int cup2d_udef_assemble(cup2d_sim *s);
/* One full time step of the hot path (no bodies): compute_dt (unless dt>0 is given), rk2, tmpV=0
 * (or kept if keep_udef), pressure_rhs, poisson_solve, pressure_correct.  Returns dt used. */
int cup2d_step(cup2d_sim *s, double dt_in, int keep_udef, double tol_abs, double tol_rel,
               int max_restarts, int max_iter, double *dt_out, int *iters_out, double *err_out);
/* The same step, asynchronously: cup2d_step_enqueue puts the whole step on the context's stream and returns without
 * waiting for the device; cup2d_step_result waits for it and returns dt, iteration count and residual
 * (cup2d_step == enqueue + result).  dt_in <= 0: the dt rule (main.cpp:6579-6595) runs on the device inside the step.
 * From the second step of a context on, the step is ONE cudaGraphLaunch of a graph captured once per buffer assignment
 * (vel/vold and pres/pold swap every step) and argument set; with tolerances the Krylov loop is a graph WHILE node whose
 * condition the device sets, so a tolerance-driven solve needs no host polling either.  Replaces the reference's
 * ~25 launches + 4 host synchronisations + 4 MPI_Allreduce per Krylov iteration (cuda.cu:403-548) and its per-operator
 * OpenMP loops (main.cpp:6607-6642, 7011-7027, 7120-7187).  Several steps may be enqueued before a result is read.
 * cup2d_set_graph(s, 0) makes every step use direct kernel launches (what profiling with cup2d_profile_enable does). */
int cup2d_step_enqueue(cup2d_sim *s, double dt_in, int keep_udef, double tol_abs, double tol_rel, int max_restarts,
                       int max_iter);
int cup2d_step_result(cup2d_sim *s, double *dt_out, int *iters_out, double *err_out);
int cup2d_set_graph(cup2d_sim *s, int on);

/* ---- host-buffer pipeline (single rank): independent steps whose inputs and results live in HOST memory ----
 * What the reference does around every solve is upload, compute, download, one after the other (cuda.cu:298-301,
 * 546-547).  Here the three legs of successive, independent steps overlap: a context owns CUP2D_PIPE_SLOTS staging sets
 * (vel + pres) and two copy streams, so that   upload(n+1) || step(n) || download(n-1)   run concurrently (PCIe is full
 * duplex; the copies take < 1 % of the HBM bandwidth the step uses).  Per slot the order is
 * upload -> step -> download [-> wait]; the calls only enqueue (cup2d_pipe_step blocks like cup2d_step does), the library
 * orders them with events, including reuse of a slot.  Host buffers must be page-locked for the copies to be asynchronous.
 * Results are bit-identical to cup2d_field_upload + cup2d_step + cup2d_field_download. */
#define CUP2D_PIPE_SLOTS 4
/* enqueue host -> staging set `slot` (vel: 128 doubles per block, pres: 64, block layout as cup2d_field_upload) */
int cup2d_pipe_upload(cup2d_sim *s, int slot, const double *vel_host, const double *pres_host);
/* cup2d_step on the contents of staging set `slot` (arguments as cup2d_step); the set then holds the step's vel and pres */
int cup2d_pipe_step(cup2d_sim *s, int slot, double dt_in, double tol_abs, double tol_rel, int max_restarts, int max_iter,
                    double *dt_out, int *iters_out, double *err_out);
/* enqueue staging set `slot` -> host */
int cup2d_pipe_download(cup2d_sim *s, int slot, double *vel_host, double *pres_host);
/* block until the last download of `slot` has landed in host memory */
int cup2d_pipe_wait(cup2d_sim *s, int slot);

/* ---- multi-GPU (one process per GPU; peers on the same NVSwitch node) ---- */
/* Size in bytes of the opaque per-rank handle blob exchanged by the launcher (torch.distributed). */
int cup2d_peer_blob_size(void);
/* Fill `blob` (cup2d_peer_blob_size() bytes) with this rank's CUDA IPC handles. */
int cup2d_peer_export(cup2d_sim *s, void *blob);
/* all_blobs = nranks blobs in rank order (all-gathered by the caller). Opens peer mappings. */
int cup2d_peer_attach(cup2d_sim *s, const void *all_blobs);
/* Explicit halo refresh of one field (normally implicit inside the operators). */
int cup2d_halo_exchange(cup2d_sim *s, int field);
/* Device address of `field` on rank `rank` as mapped into this process by cup2d_peer_attach (NULL before). */
void *cup2d_peer_field_ptr(cup2d_sim *s, int rank, int field);

/* ---- Poisson-only context (the LocalSpMatDnVec boundary, cuda.h:26-79) ---- */
/* nbr[4*k..4*k+3] = block indices of the W,E,S,N neighbours of block k on the same level, -1 = wall
 * (what the reference's COO rows main.cpp:7074-7107 encode on a uniform level).  The context supports
 * field upload/download of CUP2D_TMP (b) and CUP2D_PRES (x0 / x) and cup2d_poisson_solve; rows are
 * numbered block-major, row = 64*k + 8*iy + ix, exactly like Solver::CellIndexer (main.cpp:5753-5771). */
int cup2d_poisson_create(int64_t nblocks, const int32_t *nbr, int32_t device, cup2d_sim **out);
/* General variant: rows that are not the same-level stencil (the coarse-fine interpolation rows of
 * main.cpp:5915-5997 on AMR grids, or anything else) are given completely in CSR and override the
 * stencil for their cells: irr_rows[n_irr] sorted unique row indices, irr_rowptr[n_irr+1], irr_col/irr_val.
 * Faces covered by such rows must have nbr = -1.  With n_irr = 0 this is cup2d_poisson_create. */
int cup2d_poisson_create_general(int64_t nblocks, const int32_t *nbr, int64_t n_irr, const int32_t *irr_rows,
                                 const int32_t *irr_rowptr, const int32_t *irr_col, const double *irr_val,
                                 int32_t device, cup2d_sim **out);
/* The same matrix distributed over several ranks the way the reference distributes it (contiguous ranges of the block list,
 * main.cpp:6494-6504; rows of rank r offset by 64*rank_begin[r], 7040-7050; remote columns = the halo of cuda.cu:611-689):
 * nbr[4*nloc] = W,E,S,N of this rank's blocks as GLOBAL block ids, irr_rows = LOCAL rows 64*(block - rank_begin[rank]) + cell,
 * irr_col = GLOBAL columns 64*block + cell.  Remote blocks named by either table become halo slots refreshed by whole-block
 * peer pulls inside the solve; cup2d_peer_export / cup2d_peer_attach before the first cup2d_poisson_solve.  Fields are
 * uploaded / downloaded per rank (nloc blocks). */
int cup2d_poisson_create_general_ranks(int64_t nblocks_global, int32_t rank, int32_t nranks, const int64_t *rank_begin,
                                       const int32_t *nbr, int64_t n_irr, const int32_t *irr_rows,
                                       const int32_t *irr_rowptr, const int32_t *irr_col, const double *irr_val,
                                       int32_t device, cup2d_sim **out);

/* ---- host-side topology plan (no GPU needed; used by the CPU tests of the multi-rank logic) ---- */
/* Same config as cup2d_create, but builds only the host tables: SFC-range partition, halo plan
 * (which face-neighbour blocks this rank pulls from which owner), neighbour table, advect tiles.
 * The context accepts only cup2d_plan_table / cup2d_nblocks_* / cup2d_destroy. */
int cup2d_plan_create(const cup2d_config *cfg, cup2d_sim **out);
/* which: 0 halo global block ids [nhalo] (halo slot k = nblocks_local + k), 1 halo owner ranks [nhalo],
 * 2 halo source slots on the owner [nhalo], 3 neighbour slots W,E,S,N per local block [4*nblocks_local]
 * (-1 = wall), 4 advect tile slots [32*ntiles], 5 tile origins in blocks [2*ntiles].
 * Returns the number of int32 entries (out may be NULL to query). */
int64_t cup2d_plan_table(const cup2d_sim *s, int which, int32_t *out);

/* ---- instrumentation ---- */
/* number of kernels this library has launched since creation (bench.py's gpu_launches) */
int64_t cup2d_launch_count(const cup2d_sim *s);
/* per-kernel-class timing with CUDA events on the launching stream (bench.py's roofline leg).
 * enable(1) starts a fresh recording, enable(0) stops.  read() synchronises the stream and returns the
 * number of classes written: names[k*32..] (NUL-terminated), summed milliseconds and launch counts. */
int cup2d_profile_enable(cup2d_sim *s, int on);
int cup2d_profile_read(cup2d_sim *s, int max_entries, char *names, double *total_ms, int64_t *launches);

/* ---- multi-level (block-AMR) meshes: ghost-stencil plan, host-only (no GPU needed) --------------------------------
 * The reference assembles the ghost cells of a block next to coarser / finer blocks by interpolation and averaging
 * (BlockLab::load / post_load, main.cpp:2247-2933).  Every such ghost is a fixed linear combination of owned cells, so
 * the plan evaluates that assembly once per regrid on symbolic values and returns it as CSR tables for the tile loaders.
 * level_ij[k] = (level, i, j) of block k in `infos` order; bpdx, bpdy = level-0 blocks per direction. */
typedef struct cup2d_amr_plan cup2d_amr_plan;
int cup2d_amr_plan_create(int64_t nblocks, const int32_t *level_ij, int32_t bpdx, int32_t bpdy, cup2d_amr_plan **out);
void cup2d_amr_plan_destroy(cup2d_amr_plan *p);
/* which: 0 = velocity lab of the advect stencil {-3,-3,4,4,tensorial} (14x14x2 per block), 1 = velocity lab of the
 * +-1 stencil (10x10x2), 2 = scalar lab of the +-1 stencil (10x10), 3 = scalar lab {-4,-4,5,5,tensorial} (16x16), 4 / 5 =
 * vector / scalar labs of the +-1 stencil with corners, 6 = velocity lab {-4,-4,5,5,tensorial} of the force diagnostics
 * (16x16x2).  Rows = (block, iy, ix, comp) in that order; row r
 * is sum_e weight[e] * field[src_block[e]][src_cellcomp[e]] (cell*dim + comp of the source block).  A row without
 * entries is a lab cell the reference never writes (corner ghosts of the non-tensorial stencils).  Returns nnz; any
 * output pointer may be NULL (call once to size, once to fill; rowptr has nrows + 1 entries). */
int64_t cup2d_amr_plan_stencil(cup2d_amr_plan *p, int which, int64_t *rowptr, int32_t *src_block, int32_t *src_cellcomp,
                               double *weight);
/* Compact form for the device.  irregular = blocks that have a coarser or finer block among their 8 neighbours (all
 * other blocks get their ghosts from same-level copies and wall reflections alone).  ghosts: CSR over the ghost cells
 * (everything outside the 8x8 interior) of the irregular blocks only; dst[r] = ((position of the block in the irregular
 * list * ncell_lab + lab cell) * dim + comp) with the lab shapes of cup2d_amr_plan_stencil.  Returns nnz, *nrows rows.
 * Blocks are independent: built on several host threads. */
int64_t cup2d_amr_plan_irregular(cup2d_amr_plan *p, int32_t *blocks_out);
int64_t cup2d_amr_plan_ghosts(cup2d_amr_plan *p, int which, int64_t *nrows, int64_t *rowptr, int32_t *dst,
                              int32_t *src_block, int32_t *src_cellcomp, double *weight);
/* (cup2d_amr_plan_ghosts and cup2d_amr_plan_stats take the kinds 0-3 and 6) */
/* ghost tables are instantiated from a dictionary of local configurations (blocks with the same neighbourhood share one
 * symbolically evaluated pattern); after cup2d_amr_plan_ghosts(which): how many patterns, how many blocks bypassed it */
int cup2d_amr_plan_stats(cup2d_amr_plan *p, int which, int32_t *npatterns, int32_t *fallbacks);
/* out[k][8]: the 8 neighbour positions of block k in the order (-1,-1),(0,-1),(1,-1),(-1,0),(1,0),(-1,1),(0,1),(1,1):
 * >= 0 same-level block, -1 domain wall, -2 covered by a coarser block, -3 refined further (the regular-ghost fast path) */
int cup2d_amr_plan_neighbours(cup2d_amr_plan *p, int32_t *out);
/* Poisson matrix of the mesh in the form cup2d_poisson_create_general takes: nbr_out[4k..] = W,E,S,N same-level neighbour
 * of block k or -1 (wall, coarser, finer), and the rows whose stencil crosses a coarse-fine face, complete, in CSR —
 * the rows the reference's assembly loop pushes (main.cpp:7051-7113 with makeFlux / interpolate / D1 / D2,
 * main.cpp:5915-5997), values bitwise identical (same accumulation order).  Returns the number of such rows and *nnz_out;
 * call with irr_rows = NULL to size. */
int64_t cup2d_amr_plan_poisson(cup2d_amr_plan *p, int32_t *nbr_out, int64_t *nnz_out, int32_t *irr_rows,
                               int32_t *irr_rowptr, int32_t *irr_col, double *irr_val);
/* coarse-fine faces for the flux correction (prepare0, main.cpp:1683-1735): records of 5 int32 = (fine block, its face,
 * coarse block, its face, which half of the coarse face); faces 0 = x-, 1 = x+, 2 = y-, 3 = y+.  Returns the count. */
int64_t cup2d_amr_plan_faces(cup2d_amr_plan *p, int32_t *out);

/* ---- multi-level meshes on the device: first, correctness-oriented path (csrc/amr_ops.cu) --------------------------
 * Checked on the GPU by tests/test_gpu_amr.py.  One GPU.  Same field ids and block layout as the uniform-grid context, blocks in `infos` order. */
typedef struct cup2d_amr cup2d_amr;
int cup2d_amr_create(int64_t nblocks, const int32_t *level_ij, int32_t bpdx, int32_t bpdy, double h0, double nu,
                     int32_t device, cup2d_amr **out);
void cup2d_amr_destroy(cup2d_amr *a);
int cup2d_amr_field_upload(cup2d_amr *a, int field, const double *host);
int cup2d_amr_field_download(cup2d_amr *a, int field, double *host);
int cup2d_amr_sync(cup2d_amr *a);
/* tmpV = KernelAdvectDiffuse(vel), flux-corrected (main.cpp:6611-6617) */
int cup2d_amr_advect_diffuse_rhs(cup2d_amr *a, double dt);
/* same result through the per-block lab loader on the WENO line core of the uniform-grid kernel (csrc/amr_fast.cu) */
int cup2d_amr_advect_diffuse_rhs_fast(cup2d_amr *a, double dt);
int cup2d_amr_pressure_rhs_fast(cup2d_amr *a, double dt, int with_laplacian);
int cup2d_amr_pressure_gradient_fast(cup2d_amr *a, double dt);
int cup2d_amr_laplacian_fast(cup2d_amr *a, double dt);
/* on != 0: the operator entry points above, and with them cup2d_amr_step, run on the fast kernels */
int cup2d_amr_set_fast(cup2d_amr *a, int on);
/* tmp = pressure_rhs(vel, u_def = tmpV, chi), flux-corrected (main.cpp:7007-7013); with_laplacian != 0: then
 * tmp -= lap(pold), flux-corrected (main.cpp:7022-7027) */
int cup2d_amr_pressure_rhs(cup2d_amr *a, double dt, int with_laplacian);
/* tmpV = pressureCorrectionKernel(pres) (main.cpp:7174-7179; not flux-corrected in the reference either) */
int cup2d_amr_pressure_gradient(cup2d_amr *a, double dt);
/* the pieces of one time step without bodies (main.cpp:6576-7187), cell size per block:
 *   compute_dt        6579-6595 with h = the smallest cell of the mesh
 *   advect_diffuse_rk2 6607-6642
 *   poisson_rhs       7007-7027: tmp = pressure_rhs(vel, u_def = tmpV, chi); pold = pres; pres = 0; tmp -= lap(pold)
 *   poisson_solve     b = tmp, x0 = pres -> pres, on the general-rows solver with the rows of cup2d_amr_plan_poisson
 *   pressure_correct  7120-7187: pres = x - mean_h2(x); pres += pold - mean_h2(pres); vel += grad-term / h^2
 *   step              all of the above with u_def = 0 */
int cup2d_amr_compute_dt(cup2d_amr *a, double cfl, double *umax_out, double *dt_out);
int cup2d_amr_advect_diffuse_rk2(cup2d_amr *a, double dt);
int cup2d_amr_poisson_rhs(cup2d_amr *a, double dt);
int cup2d_amr_poisson_solve(cup2d_amr *a, double tol_abs, double tol_rel, int max_restarts, int max_iter, int *iters,
                            double *err);
int cup2d_amr_pressure_correct(cup2d_amr *a, double dt);
int cup2d_amr_step(cup2d_amr *a, double cfl, double dt_in, double tol_abs, double tol_rel, int max_restarts, int max_iter,
                   double *dt_out, int *iters, double *err);

/* Several GPUs (first form): every rank creates the context over the WHOLE mesh and computes the stencil operators
 * redundantly — bitwise the same on every rank — while the Poisson solve is distributed over the ranks by the block ranges
 * rank_begin[nranks+1] (cup2d_poisson_create_general_ranks) and its solution all-gathered over NVLink.  Call once, before the
 * first solve, then exchange the peer blobs exactly like cup2d_peer_export / cup2d_peer_attach. */
int cup2d_amr_set_ranks(cup2d_amr *a, int32_t rank, int32_t nranks, const int64_t *rank_begin);
/* Several GPUs (second form): the mesh itself is distributed.  Every rank passes the same whole block list; rank r then holds
 * only the blocks rank_begin[r] .. rank_begin[r+1] (the reference's partition, main.cpp:6494-6504) plus halo slots for every
 * remote block its tables name, and computes only its own blocks.  Its field arrays are those of the distributed Poisson
 * context, so halo refreshes are the whole-block peer pulls of the uniform path, the solve runs in place, the face fluxes of
 * fillcases cross a rank boundary inside a field array, and dt / the pressure means are all-reduced in a kernel.  Fast kernels
 * only; cup2d_amr_field_upload / _download move this rank's blocks.  Follow with cup2d_amr_peer_export / _attach. */
int cup2d_amr_create_ranks(int64_t nblocks, const int32_t *level_ij, int32_t bpdx, int32_t bpdy, double h0, double nu,
                           int32_t rank, int32_t nranks, const int64_t *rank_begin, int32_t device, cup2d_amr **out);
int cup2d_amr_peer_export(cup2d_amr *a, void *blob);
int cup2d_amr_peer_attach(cup2d_amr *a, const void *all_blobs);

/* adapt()'s tagging on a multi-level mesh (main.cpp:4676-4697; cf. cup2d_adapt_tags): block_linf_out[k] = L-inf over block
 * k of the field adapt() thresholds against Rtol / Ctol — the vorticity of vel (KernelVorticity, 3343-3366), with 2*rtol in
 * the four centre cells of every block whose chi lab (stencil {-4,-4,5,5,tensorial}, ghosts across level jumps included) is
 * positive within 4 cells (finest level, level_max - 1) or 2 cells (other levels) of it (GradChiOnTmp, 4631-4656).  The
 * field itself is left in tmp.  The decision is cup2d_amr_adapt_mesh, the field transfer cup2d_amr_regrid. */
int cup2d_amr_adapt_tags(cup2d_amr *a, double rtol, int level_max, double *block_linf_out);

/* dump() on a multi-level mesh (main.cpp:3367-3467; cf. cup2d_dump): path.xdmf2, path.xyz.raw, path.attr.raw — the
 * reference's three files, byte for byte, from the device-resident velocity. */
int cup2d_amr_dump(cup2d_amr *a, double time, const char *path);
/* adapt()'s refine / compress decision, host only, no GPU needed (main.cpp:4676-4860: thresholds, Refine at levelMax-1 and
 * Compress at level 0 dropped, the 2:1 pass from levelMax-1 down with the reference's in-place updates, sibling agreement),
 * then the new block list in the reference's order (fill_pos / Encode, main.cpp:1550-1553, 422-445).  block_linf = the
 * per-block L-inf of cup2d_amr_adapt_tags.  Returns the new block count; new_level_ij may be NULL to size it first. */
int64_t cup2d_amr_adapt_mesh(int64_t nblocks, const int32_t *level_ij, int32_t bpdx, int32_t bpdy, int32_t level_max,
                             const double *block_linf, double rtol, double ctol, int32_t *new_level_ij);
/* adapt()'s field transfer on the device (main.cpp:4902-5195; csrc/amr_regrid.cu): the context moves in place onto a mesh one
 * refine / compress step away.  Copies unchanged blocks, refines from the {-1,-1,2,2,tensorial} lab of the old mesh
 * (main.cpp:5012-5028), compresses by the reference's 4-cell average (5160-5164) for tmp, chi, vel, vold, pres, pold; tmpV is
 * zero afterwards.  Plan, tables, Poisson context and lab buffers are rebuilt for the new mesh; shapes are cleared (set them
 * again, as ongrid() does after adapt()).  CUP2D_EINVAL, context untouched, for a mesh that is not one step away;
 * CUP2D_ESTATE for contexts on several ranks.  The same block list is a no-op. */
int cup2d_amr_regrid(cup2d_amr *a, int64_t nblocks_new, const int32_t *new_level_ij);

/* Bodies on a multi-level mesh: the cup2d_shape_* calls (above) on the cup2d_amr context, with the cell size and the block
 * position taken per block (Info::h, Info::origin, main.cpp:695-696).  block_ids index the context's blocks; a shape's
 * arrays are copied before the call returns.  Sums to rounding (per-block partial sums added in block order), blend and
 * assembly bit-identical to the reference.  Same status as the rest of the multi-level device path. */
int cup2d_amr_shape_set(cup2d_amr *a, int shape, int nob, const int32_t *block_ids, const double *chi, const double *udef);
int cup2d_amr_shape_integrals(cup2d_amr *a, int shape, double lambda, double dt, double cx, double cy, double *out7);
int cup2d_amr_penalize(cup2d_amr *a, int shape, double lambda, double dt, double cx, double cy, double us, double vs,
                       double omega);
int cup2d_amr_udef_assemble(cup2d_amr *a);

/* ongrid() on a multi-level mesh (main.cpp:3991-4630; csrc/amr_ongrid.cu): the rasterisation of every body's midline into the
 * chi and tmp fields and into the shape's obstacle blocks, on the device.  The midline kinematics (main.cpp:4029-4207), the
 * 3x3 rigid-body solve stay with the caller; the collision model (cup2d_amr_collide), the surface normals (cup2d_amr_surface)
 * and the force diagnostics (cup2d_amr_forces) read the blocks on the device. */
typedef struct {
  int32_t nm, reserved;                /* midline points; nm >= 9 (Nsegments = (nm-1)/8 >= 1 dividing nm-1, main.cpp:4208-4210) */
  const double *rX, *rY, *norX, *norY; /* [nm] each: the shape-frame midline exactly as ongrid() holds it at main.cpp:4208 */
  const double *vX, *vY, *vNorX, *vNorY, *width;
  double center[2], orientation;       /* Shape::center, Shape::orientation (already advanced by main.cpp:3993-4007) */
  double center_of_mass[2];            /* Shape::centerOfMass before main.cpp:4485-4486 */
} cup2d_body;
/* main.cpp:4019-4024 + 4208-4556 for all shapes, in shape order: chi = 0 and tmp = -1 everywhere; the AreaSegment boxes
 * (3839-3878, 4216-4242; safe distance 4 h with h the smallest cell of the mesh) on the host, with the host libm's cos / sin;
 * the block scan (4243-4269), PutFishOnBlocks (4271-4463), PutChiOnGrid (3911-3969, 4469) and the rigid-motion removal
 * (4472-4556) on the device.  out[10*k..] = {Mass, COM_x, COM_y (4475-4483), new centerOfMass x, y (4485-4486), m, j, u, v, a
 * (4529-4531)}.  Leaves chi, tmp and each shape's obstacle blocks (ids in ascending block order, chi, dist, udef) on the device
 * for cup2d_amr_shape_integrals / _penalize / _udef_assemble; shapes k >= nshapes are dropped.  dist, tmp and u_def before the
 * correction are bit-identical to the reference; chi on blocks whose +-1 lab needs the ghost tables, and the sums, to rounding.
 * CUP2D_EINVAL (context untouched) for a body with nm < 9 or (nm-1) not a multiple of (nm-1)/8, a missing array or its center outside the domain (the reference
 * aborts, 4009-4013); CUP2D_ESTATE for contexts on several ranks.  1 <= nshapes <= 64. */
int cup2d_amr_ongrid(cup2d_amr *a, int nshapes, const cup2d_body *bodies, double *out);
/* download shape k's obstacle blocks (any pointer may be NULL; returns nob): ids[nob], chi[nob][64], dist[nob][64] (shapes placed
 * by cup2d_amr_ongrid or given by cup2d_amr_shape_set_dist), udef[nob][64][2] — what the host's forces and skins read */
int cup2d_amr_shape_get(cup2d_amr *a, int shape, int32_t *ids, double *chi, double *dist, double *udef);
/* CUDA-event timing of cup2d_amr_ongrid on the context's stream: timing(a, 1) creates the events and times every following call
 * (0 stops; a regrid clears it); times(a, ms8) gives the last timed call's milliseconds: {whole call on the stream (upload,
 * kernels and the host waits between them), scan, offsets, compact, fish, chi, moments, correct}, every kernel class summed
 * over the shapes */
int cup2d_amr_ongrid_timing(cup2d_amr *a, int on);
int cup2d_amr_ongrid_times(cup2d_amr *a, double *ms8);

/* The collision model on a multi-level mesh (main.cpp:6705-6943 with collision() / compute_j() at 209-291; csrc/amr_collide.cu),
 * on the obstacle blocks the device holds.  shape_set_dist uploads dist[nob][8][8] for a shape already set by
 * cup2d_amr_shape_set (recorded or host-built shapes), which cup2d_amr_shape_get then returns; a later shape_set drops it. */
int cup2d_amr_shape_set_dist(cup2d_amr *a, int shape, const double *dist);
typedef struct {
  double u, v, omega;       /* in: after the 3x3 solve (main.cpp:6699-6701); out: after the collision model (6937-6942) */
  double center_of_mass[2]; /* Shape::centerOfMass */
  double M, J, length;      /* Shape::M, Shape::J (cup2d_amr_ongrid's out[5], out[6]), Shape::length */
} cup2d_rigid;
/* Shapes 0 .. nshapes-1: over the cells of their common obstacle blocks where both chi are positive, each shape's sums of
 * 6733-6813 (its own chi, chi pos, chi velocity, chi grad dist, then the same of its partners) on the device, added in the
 * reference's order (partners in index order, blocks ascending, cells in row order), so bit-identical to the reference on one
 * rank; then on the host the pair loop of 6863-6943 (both centroid masses >= 2, centroids within `length`, approaching) with
 * the elastic impulse, which overwrites u, v, omega of both shapes of a pair.  Pairs are taken in (i ascending, j > i
 * ascending) order, each seeing what earlier pairs left: the reference's result on one OpenMP thread.  With more than two
 * shapes and several simultaneous collisions the reference's parallel loop has no defined order, and neither has its result.
 * sums20 (may be NULL) gets [nshapes][20] in the layout of 6814-6837 (the Z slots zero).  Fields and shape data are not
 * changed.  CUP2D_EINVAL for nshapes outside 1..64, a shape not set or one whose block ids are not strictly ascending
 * (cup2d_amr_ongrid leaves them ascending); CUP2D_ESTATE for a shape without dist or a context on several ranks.  On any
 * error `shapes` and the context are untouched. */
int cup2d_amr_collide(cup2d_amr *a, int nshapes, cup2d_rigid *shapes, double *sums20);

/* Surface normals and force diagnostics on a multi-level mesh (csrc/amr_forces.cu), on the obstacle blocks the device holds:
 * what a caller otherwise computes on the host from downloaded vel, pres and chi.  Bit-identical to the reference on one rank
 * where the labs involved are copies (no level jump); elsewhere the labs come from the plan's ghost rows, to rounding.
 * ComputeSurfaceNormals (main.cpp:3774-3828, as ongrid() calls it at 4470) on the chi and tmp fields as they stand, for shapes
 * 0 .. nshapes-1: each obstacle block's surface points (ix, iy, dchidx, dchidy, D) in the reference's push order.  Call it
 * after cup2d_amr_ongrid and before anything overwrites tmp (poisson_rhs, adapt_tags), as the reference does.  The reference
 * reads its lab rows there without their offset, so three cells per block read a corner ghost no rule writes; those hold
 * chi = 0 and tmp = -1, the reference's values while the bodies are away from the domain walls.  cup2d_amr_shape_set,
 * cup2d_amr_ongrid and cup2d_amr_regrid drop the points.  CUP2D_EINVAL for nshapes outside 1..64 or a shape not set;
 * CUP2D_ESTATE for contexts on several ranks. */
int cup2d_amr_surface(cup2d_amr *a, int nshapes);
/* shape k's surface points: block[n] (block id), ixy[n][2], normal[n][3] = {dchidx, dchidy, D}; skin[n][14] = x_s, y_s, p_s,
 * u_s, v_s, nx_s, ny_s, omega_s, uDef_s, vDef_s, fX_s, fY_s, fXv_s, fYv_s of the last cup2d_amr_forces call (zero before).
 * Any pointer may be NULL; returns n (CUP2D_EINVAL: no such shape, CUP2D_ESTATE: no points since the shape was last set). */
int64_t cup2d_amr_surface_get(cup2d_amr *a, int shape, int32_t *block, int32_t *ixy, double *normal, double *skin);
/* KernelComputeForces + main.cpp:7188-7284 from vel, pres, chi and each shape's u_def: out[23*k ..] = quantities[0..18] in the
 * order of 7233-7251 (circulation, perimeter, forcex, forcex_P, forcex_V, torque_P, drag, lift, Pout, PoutNew, PoutBnd, torque,
 * forcey, forcey_P, forcey_V, torque_V, thrust, defPowerBnd, defPower), then Pthrust, Pdrag, EffPDef, EffPDefBnd (7273-7280).
 * Reads u, v and center_of_mass of shapes[k] (cup2d_rigid, as cup2d_amr_collide leaves them).  Points, then blocks in
 * ascending id order, are added as the reference's serial chains.  Fields and shape data are not changed.  CUP2D_EINVAL for
 * nshapes outside 1..64, a shape not set or a NULL shapes / out; CUP2D_ESTATE for a shape whose surface points were dropped
 * or a context on several ranks.  On any error the context and out are untouched. */
int cup2d_amr_forces(cup2d_amr *a, int nshapes, const cup2d_rigid *shapes, double *out);

#ifdef __cplusplus
}
#endif
#endif
