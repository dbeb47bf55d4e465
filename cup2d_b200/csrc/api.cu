// C ABI of libcup2d_b200.so (include/cup2d_b200.h): context creation, topology tables, field
// transfer, the C++ host driver of one time step, and the NVLink peer-memory halo exchange.
#include "sim.h"
#include <algorithm>
#include <cstring>
#include <map>
#include <mutex>

namespace cup2d {

static thread_local std::string g_err;
void set_error(const std::string &msg) { g_err = msg; }
int dim_of(int field) { return (field == CUP2D_VEL || field == CUP2D_VOLD || field == CUP2D_TMPV) ? 2 : 1; }

// ---- space-filling curve: host restatement of SpaceCurve (main.cpp:342-446, init 6342-6376) ------
static long long hilbert_xy2d(int b, int x, int y) { // AxestoTranspose, main.cpp:347-359
  const int n = 1 << b;
  long long d = 0;
  for (int s = n / 2; s > 0; s /= 2) {
    const int rx = (x & s) > 0, ry = (y & s) > 0;
    d += (long long)s * s * ((3 * rx) ^ ry);
    if (ry == 0) { // rot, main.cpp:374-384
      if (rx == 1) {
        x = n - 1 - x;
        y = n - 1 - y;
      }
      std::swap(x, y);
    }
  }
  return d;
}
static void hilbert_d2xy(int b, long long d, int *xo, int *yo) { // TransposetoAxes, main.cpp:360-373
  const int n = 1 << b;
  int x = 0, y = 0;
  long long t = d;
  for (long long s = 1; s < n; s *= 2) {
    const long long rx = 1 & (t / 2), ry = 1 & (t ^ rx);
    if (ry == 0) {
      if (rx == 1) {
        x = (int)s - 1 - x;
        y = (int)s - 1 - y;
      }
      std::swap(x, y);
    }
    x += (int)(s * rx);
    y += (int)(s * ry);
    t /= 4;
  }
  *xo = x;
  *yo = y;
}

} // namespace cup2d

using namespace cup2d;

extern "C" {

const char *cup2d_last_error(void) { return g_err.c_str(); }
int cup2d_version(void) { return 100; }

int cup2d_block_order(int32_t bpdx, int32_t bpdy, int32_t level, int32_t *out) {
  CUP2D_REQUIRE(bpdx > 0 && bpdy > 0 && level >= 0 && out, "cup2d_block_order: bad arguments");
  // base curve over the bpdx x bpdy coarse blocks, compacted when the bounding 2^b square is not
  // filled (main.cpp:6342-6376)
  int base_level = 0;
  while ((1 << base_level) < std::max(bpdx, bpdy)) base_level++;
  std::vector<long long> zsave((size_t)bpdx * bpdy);
  bool regular = true;
  {
    const int n = 1 << base_level;
    std::vector<char> inside((size_t)n * n, 0);
    std::vector<long long> before((size_t)n * n + 1, 0);
    for (long long d = 0; d < (long long)n * n; d++) {
      int x, y;
      hilbert_d2xy(base_level, d, &x, &y);
      inside[d] = (x < bpdx && y < bpdy);
      before[d + 1] = before[d] + (inside[d] ? 0 : 1);
    }
    for (int j = 0; j < bpdy; j++)
      for (int i = 0; i < bpdx; i++) {
        long long idx = hilbert_xy2d(base_level, i, j);
        if (before[idx] > 0) regular = false;
        zsave[(size_t)j * bpdx + i] = idx - before[idx];
      }
  }
  const int nbx = bpdx << level, nby = bpdy << level;
  const long long aux = 1LL << level;
  std::vector<std::pair<long long, int>> keyed((size_t)nbx * nby);
  for (int j = 0; j < nby; j++)
    for (int i = 0; i < nbx; i++) {
      long long z;
      if (regular)
        z = hilbert_xy2d(level + base_level, i, j); // forward(), main.cpp:385-400
      else {
        const int I = (int)(i / aux), J = (int)(j / aux);
        z = hilbert_xy2d(level, (int)(i - I * aux), (int)(j - J * aux)) + zsave[(size_t)J * bpdx + I] * aux * aux;
      }
      keyed[(size_t)j * nbx + i] = {z, j * nbx + i};
    }
  std::sort(keyed.begin(), keyed.end());
  for (size_t k = 0; k < keyed.size(); k++) {
    out[2 * k] = keyed[k].second % nbx;
    out[2 * k + 1] = keyed[k].second / nbx;
  }
  return CUP2D_OK;
}

static int alloc_device_state(cup2d_sim *s);

static int build_tables(cup2d_sim *s) {
  const int nbx = s->nbx, nby = s->nby;
  const int64_t nloc = s->nloc, gb = s->gbegin, ge = s->gbegin + s->nloc;
  std::vector<int32_t> gid_of((size_t)nbx * nby, -1);
  for (int64_t g = 0; g < s->nglobal; g++) {
    const int i = s->ij[2 * g], j = s->ij[2 * g + 1];
    CUP2D_REQUIRE(i >= 0 && i < nbx && j >= 0 && j < nby, "cup2d_create: block index outside the grid");
    CUP2D_REQUIRE(gid_of[(size_t)j * nbx + i] < 0, "cup2d_create: duplicate block index");
    gid_of[(size_t)j * nbx + i] = (int32_t)g;
  }
  auto gid_at = [&](int i, int j) -> int32_t {
    if (i < 0 || i >= nbx || j < 0 || j >= nby) return -1;
    return gid_of[(size_t)j * nbx + i];
  };
  // halo = non-local face neighbours of local blocks (the hot-path stencils are cross-shaped)
  std::vector<int32_t> halo;
  static const int di[4] = {-1, 1, 0, 0}, dj[4] = {0, 0, -1, 1};
  for (int64_t g = gb; g < ge; g++) {
    const int i = s->ij[2 * g], j = s->ij[2 * g + 1];
    for (int k = 0; k < 4; k++) {
      const int32_t n = gid_at(i + di[k], j + dj[k]);
      if (n >= 0 && (n < gb || n >= ge)) halo.push_back(n);
    }
  }
  std::sort(halo.begin(), halo.end());
  halo.erase(std::unique(halo.begin(), halo.end()), halo.end());
  s->halo_gid = halo;
  s->nhalo = (int64_t)halo.size();
  s->nslots = nloc + s->nhalo;
  s->halo_owner.resize(halo.size());
  for (size_t k = 0; k < halo.size(); k++) {
    int r = 0;
    while (!(halo[k] >= s->rank_begin[r] && halo[k] < s->rank_begin[r + 1])) r++;
    s->halo_owner[k] = r;
  }
  auto slot_of = [&](int32_t g) -> int {
    if (g < 0) return -1;
    if (g >= gb && g < ge) return (int)(g - gb);
    auto it = std::lower_bound(halo.begin(), halo.end(), g);
    if (it != halo.end() && *it == g) return (int)(nloc + (it - halo.begin()));
    return -1;
  };
  // per-block neighbour table W,E,S,N
  std::vector<int> nbr((size_t)nloc * 4);
  for (int64_t g = gb; g < ge; g++) {
    const int i = s->ij[2 * g], j = s->ij[2 * g + 1];
    for (int k = 0; k < 4; k++) nbr[(size_t)(g - gb) * 4 + k] = slot_of(gid_at(i + di[k], j + dj[k]));
  }
  // advect tiles: aligned 4x4 block groups that contain at least one local block, in SFC order of
  // first appearance (keeps neighbouring tiles close in launch order => L2 reuse of ring blocks)
  std::map<std::pair<int, int>, int> tile_id;
  std::vector<std::pair<int, int>> tiles;
  for (int64_t g = gb; g < ge; g++) {
    std::pair<int, int> key(s->ij[2 * g] / TILE_B, s->ij[2 * g + 1] / TILE_B);
    if (tile_id.emplace(key, (int)tiles.size()).second) tiles.push_back(key);
  }
  s->ntiles = (int)tiles.size();
  std::vector<int> tslots((size_t)s->ntiles * TILE_SLOTS), torg((size_t)s->ntiles * 2);
  for (int t = 0; t < s->ntiles; t++) {
    const int bi0 = tiles[t].first * TILE_B, bj0 = tiles[t].second * TILE_B;
    torg[2 * t] = bi0;
    torg[2 * t + 1] = bj0;
    int *ts = &tslots[(size_t)t * TILE_SLOTS];
    for (int by = 0; by < 4; by++)
      for (int bx = 0; bx < 4; bx++) ts[by * 4 + bx] = slot_of(gid_at(bi0 + bx, bj0 + by));
    for (int k = 0; k < 4; k++) {
      ts[16 + k] = slot_of(gid_at(bi0 - 1, bj0 + k)); // W
      ts[20 + k] = slot_of(gid_at(bi0 + 4, bj0 + k)); // E
      ts[24 + k] = slot_of(gid_at(bi0 + k, bj0 - 1)); // S
      ts[28 + k] = slot_of(gid_at(bi0 + k, bj0 + 4)); // N
    }
  }
  s->h_nbr = nbr;
  s->h_tiles = tslots;
  s->h_torg = torg;
  // halo source table: (owner rank, slot on the owner)
  s->h_halo_src.assign((size_t)s->nhalo * 2, 0);
  for (int64_t k = 0; k < s->nhalo; k++) {
    s->h_halo_src[2 * k] = s->halo_owner[k];
    s->h_halo_src[2 * k + 1] = (int)(halo[k] - s->rank_begin[s->halo_owner[k]]);
  }
  return CUP2D_OK;
}

static int upload_tables(cup2d_sim *s) {
  auto up = [](int **d, const std::vector<int> &h) -> cudaError_t {
    cudaError_t e = cudaMalloc(d, std::max<size_t>(h.size(), 4) * sizeof(int));
    if (e != cudaSuccess) return e;
    return cudaMemcpy(*d, h.data(), h.size() * sizeof(int), cudaMemcpyHostToDevice);
  };
  CUP2D_CUDA(up(&s->d_nbr, s->h_nbr));
  CUP2D_CUDA(up(&s->d_tiles, s->h_tiles));
  CUP2D_CUDA(up(&s->d_tile_org, s->h_torg));
  if (s->nhalo > 0) CUP2D_CUDA(up(&s->d_halo_src, s->h_halo_src));
  return CUP2D_OK;
}

// fills the topology part of a context from a config (no CUDA calls)
static int init_topology(const cup2d_config *cfg, cup2d_sim **out) {
  CUP2D_REQUIRE(cfg && out, "cup2d_create: null argument");
  CUP2D_REQUIRE(cfg->nbx > 0 && cfg->nby > 0 && cfg->nblocks_global == (int64_t)cfg->nbx * cfg->nby,
                "cup2d_create: nblocks_global must equal nbx*nby (uniform level)");
  CUP2D_REQUIRE(cfg->nranks >= 1 && cfg->nranks <= MAX_RANKS && cfg->rank >= 0 && cfg->rank < cfg->nranks,
                "cup2d_create: bad rank/nranks (1..8 ranks)");
  CUP2D_REQUIRE(cfg->block_ij && cfg->rank_begin, "cup2d_create: missing tables");
  CUP2D_REQUIRE(cfg->h > 0, "cup2d_create: h must be positive");
  CUP2D_REQUIRE(cfg->nblocks_global * 64 < (1LL << 31), "cup2d_create: more than 2^31 cells per field");
  cup2d_sim *s = new cup2d_sim;
  s->nbx = cfg->nbx;
  s->nby = cfg->nby;
  s->nglobal = cfg->nblocks_global;
  s->rank = cfg->rank;
  s->nranks = cfg->nranks;
  s->device = cfg->device;
  s->h = cfg->h;
  s->nu = cfg->nu;
  s->cfl = cfg->cfl;
  s->ij.assign(cfg->block_ij, cfg->block_ij + 2 * cfg->nblocks_global);
  s->rank_begin.assign(cfg->rank_begin, cfg->rank_begin + cfg->nranks + 1);
  bool ok = s->rank_begin[0] == 0 && s->rank_begin[cfg->nranks] == s->nglobal;
  for (int r = 0; ok && r < cfg->nranks; r++) ok = s->rank_begin[r + 1] > s->rank_begin[r];
  if (!ok) {
    delete s;
    set_error("cup2d_create: rank_begin must be increasing and span [0, nblocks_global] (every rank owns blocks)");
    return CUP2D_EINVAL;
  }
  s->gbegin = s->rank_begin[s->rank];
  s->nloc = s->rank_begin[s->rank + 1] - s->gbegin;
  int rc = build_tables(s);
  if (rc) {
    delete s;
    return rc;
  }
  *out = s;
  return CUP2D_OK;
}

int cup2d_plan_create(const cup2d_config *cfg, cup2d_sim **out) {
  cup2d_sim *s = nullptr;
  int rc = init_topology(cfg, &s);
  if (rc) return rc;
  s->plan_only = true;
  *out = s;
  return CUP2D_OK;
}

int64_t cup2d_plan_table(const cup2d_sim *s, int which, int32_t *out) {
  if (!s) return CUP2D_EINVAL;
  const std::vector<int> *v = nullptr;
  std::vector<int> tmp;
  switch (which) {
  case 0: tmp.assign(s->halo_gid.begin(), s->halo_gid.end()); v = &tmp; break;
  case 1: tmp.assign(s->halo_owner.begin(), s->halo_owner.end()); v = &tmp; break;
  case 2: tmp.resize(s->nhalo); for (int64_t k = 0; k < s->nhalo; k++) tmp[k] = s->h_halo_src[2 * k + 1]; v = &tmp; break;
  case 3: v = &s->h_nbr; break;
  case 4: v = &s->h_tiles; break;
  case 5: v = &s->h_torg; break;
  default: set_error("cup2d_plan_table: unknown table"); return CUP2D_EINVAL;
  }
  if (out) memcpy(out, v->data(), v->size() * sizeof(int));
  return (int64_t)v->size();
}

int cup2d_create(const cup2d_config *cfg, cup2d_sim **out) {
  CUP2D_REQUIRE(cfg && out, "cup2d_create: null argument");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    set_error("cup2d_create: no CUDA device visible; this library has no CPU fallback");
    return CUP2D_ENOGPU;
  }
  CUP2D_REQUIRE(cfg->device >= 0 && cfg->device < ndev, "cup2d_create: bad device ordinal");
  CUP2D_CUDA(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  CUP2D_CUDA(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9 || prop.minor != 0) {
    set_error(std::string("cup2d_create: device '") + prop.name + "' is not sm_90 (compiled for sm_90a only)");
    return CUP2D_ENOGPU;
  }
  cup2d_sim *s = nullptr;
  int rc = init_topology(cfg, &s);
  if (rc) return rc;
  s->num_sms = prop.multiProcessorCount;
  rc = alloc_device_state(s);
  if (rc) {
    cup2d_destroy(s);
    return rc;
  }
  *out = s;
  return CUP2D_OK;
}

// Poisson-only context from a bare block neighbour table (what the LocalSpMatDnVec adapter derives from
// the reference's COO pushes, dropin/local_spmat_adapter.cpp): no (i,j) geometry, no advect tiles.
int cup2d_poisson_create(int64_t nblocks, const int32_t *nbr, int32_t device, cup2d_sim **out) {
  CUP2D_REQUIRE(nblocks > 0 && nbr && out, "cup2d_poisson_create: bad arguments");
  CUP2D_REQUIRE(nblocks * 64 < (1LL << 31), "cup2d_poisson_create: more than 2^31 rows");
  for (int64_t k = 0; k < 4 * nblocks; k++)
    CUP2D_REQUIRE(nbr[k] >= -1 && nbr[k] < nblocks, "cup2d_poisson_create: neighbour slot out of range");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    set_error("cup2d_poisson_create: no CUDA device visible; this library has no CPU fallback");
    return CUP2D_ENOGPU;
  }
  CUP2D_REQUIRE(device >= 0 && device < ndev, "cup2d_poisson_create: bad device ordinal");
  CUP2D_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  CUP2D_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    set_error(std::string("cup2d_poisson_create: device '") + prop.name + "' is not sm_90");
    return CUP2D_ENOGPU;
  }
  cup2d_sim *s = new cup2d_sim;
  s->nglobal = s->nloc = s->nslots = nblocks;
  s->device = device;
  s->h = 1.0;
  s->poisson_only = true;
  s->rank_begin = {0, nblocks};
  s->h_nbr.assign(nbr, nbr + 4 * nblocks);
  s->num_sms = prop.multiProcessorCount;
  int rc = alloc_device_state(s);
  if (rc) {
    cup2d_destroy(s);
    return rc;
  }
  *out = s;
  return CUP2D_OK;
}

// general rows of a Poisson-only context: irr_rows (sorted, unique) index LOCAL rows 64*block + cell, irr_col index the
// context's vector slots (local blocks, then halo slots)
static int install_general_rows(cup2d_sim *s, int64_t n_irr, const int32_t *irr_rows, const int32_t *irr_rowptr,
                                const int32_t *irr_col, const double *irr_val) {
  std::vector<int> blk(s->nloc, -1), tab;
  int nirrblk = 0;
  for (int64_t k = 0; k < n_irr; k++) {
    const int r = irr_rows[k];
    CUP2D_REQUIRE(r >= 0 && r < s->nloc * 64 && (k == 0 || irr_rows[k - 1] < r),
                  "cup2d_poisson_create_general: irr_rows must be sorted, unique, in range");
    const int b = r / 64;
    if (blk[b] < 0) {
      blk[b] = nirrblk++;
      tab.resize((size_t)nirrblk * 64, -1);
    }
    tab[(size_t)blk[b] * 64 + r % 64] = (int)k;
  }
  const int nnz = irr_rowptr[n_irr];
  for (int j = 0; j < nnz; j++)
    CUP2D_REQUIRE(irr_col[j] >= 0 && irr_col[j] < s->nslots * 64, "cup2d_poisson_create_general: column out of range");
  auto up = [](void **d, const void *h, size_t bytes) -> cudaError_t {
    cudaError_t e = cudaMalloc(d, bytes ? bytes : 8);
    if (e != cudaSuccess) return e;
    return cudaMemcpy(*d, h, bytes, cudaMemcpyHostToDevice);
  };
  CUP2D_CUDA(up((void **)&s->d_irr_blk, blk.data(), blk.size() * sizeof(int)));
  CUP2D_CUDA(up((void **)&s->d_irr_tab, tab.data(), tab.size() * sizeof(int)));
  CUP2D_CUDA(up((void **)&s->d_irr_rowptr, irr_rowptr, (size_t)(n_irr + 1) * sizeof(int)));
  CUP2D_CUDA(up((void **)&s->d_irr_col, irr_col, (size_t)nnz * sizeof(int)));
  CUP2D_CUDA(up((void **)&s->d_irr_val, irr_val, (size_t)nnz * sizeof(double)));
  s->n_irr_rows = n_irr;
  return CUP2D_OK;
}

// Poisson-only context whose matrix is "same-level stencil from nbr[] + general CSR rows that override
// it".  irr_rows (sorted, unique) are row indices 64*block + 8*iy + ix; their complete rows are given
// in CSR (rowptr has n_irr+1 entries).  nbr faces that are covered by general rows must be -1.
int cup2d_poisson_create_general(int64_t nblocks, const int32_t *nbr, int64_t n_irr, const int32_t *irr_rows,
                                 const int32_t *irr_rowptr, const int32_t *irr_col, const double *irr_val,
                                 int32_t device, cup2d_sim **out) {
  int rc = cup2d_poisson_create(nblocks, nbr, device, out);
  if (rc || n_irr <= 0) return rc;
  cup2d_sim *s = *out;
  auto bail = [&](const char *msg) {
    set_error(msg);
    cup2d_destroy(s);
    *out = nullptr;
    return CUP2D_EINVAL;
  };
  if (!irr_rows || !irr_rowptr || !irr_col || !irr_val) return bail("cup2d_poisson_create_general: null table");
  if ((rc = install_general_rows(s, n_irr, irr_rows, irr_rowptr, irr_col, irr_val))) { // no half-built context escapes
    cup2d_destroy(s);
    *out = nullptr;
    return rc;
  }
  return CUP2D_OK;
}

// The same on several ranks (one process per GPU): rank r owns the contiguous range rank_begin[r] .. rank_begin[r+1] of the
// global block list.  nbr = W,E,S,N of the LOCAL blocks as GLOBAL block ids (-1: wall or covered by general rows);
// irr_rows = LOCAL row indices 64*(block - rank_begin[rank]) + cell; irr_col = GLOBAL column indices 64*block + cell.
// Every remote block these tables name becomes a halo slot of this rank (refreshed by whole-block peer pulls like the
// face neighbours of the uniform path), the tables are renumbered to slots, and the Krylov kernels run unchanged.
// cup2d_peer_export / cup2d_peer_attach must follow before the first solve.
int cup2d_poisson_create_general_ranks(int64_t nblocks_global, int32_t rank, int32_t nranks, const int64_t *rank_begin,
                                       const int32_t *nbr, int64_t n_irr, const int32_t *irr_rows,
                                       const int32_t *irr_rowptr, const int32_t *irr_col, const double *irr_val,
                                       int32_t device, cup2d_sim **out) {
  return poisson_create_general_ranks_ex(nblocks_global, rank, nranks, rank_begin, nbr, n_irr, irr_rows, irr_rowptr, irr_col,
                                         irr_val, 0, nullptr, device, out);
}
} // extern "C"
// + n_extra further remote blocks that must be halo slots of this rank (the stencil tables of a distributed multi-level
// context name blocks the Poisson rows do not)
int cup2d::poisson_create_general_ranks_ex(int64_t nblocks_global, int32_t rank, int32_t nranks, const int64_t *rank_begin,
                                           const int32_t *nbr, int64_t n_irr, const int32_t *irr_rows,
                                           const int32_t *irr_rowptr, const int32_t *irr_col, const double *irr_val,
                                           int64_t n_extra, const int32_t *extra_blocks, int32_t device, cup2d_sim **out) {
  CUP2D_REQUIRE(out && nbr && rank_begin && nblocks_global > 0, "cup2d_poisson_create_general_ranks: bad arguments");
  CUP2D_REQUIRE(nranks >= 1 && nranks <= MAX_RANKS && rank >= 0 && rank < nranks, "cup2d_poisson_create_general_ranks: bad rank/nranks (1..8 ranks)");
  CUP2D_REQUIRE(nblocks_global * 64 < (1LL << 31), "cup2d_poisson_create_general_ranks: more than 2^31 rows");
  CUP2D_REQUIRE(n_irr == 0 || (irr_rows && irr_rowptr && irr_col && irr_val), "cup2d_poisson_create_general_ranks: null table");
  bool ok = rank_begin[0] == 0 && rank_begin[nranks] == nblocks_global;
  for (int r = 0; ok && r < nranks; r++) ok = rank_begin[r + 1] > rank_begin[r];
  CUP2D_REQUIRE(ok, "cup2d_poisson_create_general_ranks: rank_begin must be increasing and span [0, nblocks_global]");
  const int64_t gb = rank_begin[rank], ge = rank_begin[rank + 1], nloc = ge - gb;
  const int64_t nnz = n_irr > 0 ? irr_rowptr[n_irr] : 0;
  std::vector<int32_t> halo;
  for (int64_t k = 0; k < 4 * nloc; k++) {
    CUP2D_REQUIRE(nbr[k] >= -1 && nbr[k] < nblocks_global, "cup2d_poisson_create_general_ranks: neighbour id out of range");
    if (nbr[k] >= 0 && (nbr[k] < gb || nbr[k] >= ge)) halo.push_back(nbr[k]);
  }
  for (int64_t j = 0; j < nnz; j++) {
    CUP2D_REQUIRE(irr_col[j] >= 0 && irr_col[j] < nblocks_global * 64, "cup2d_poisson_create_general_ranks: column out of range");
    const int32_t g = irr_col[j] / 64;
    if (g < gb || g >= ge) halo.push_back(g);
  }
  for (int64_t k = 0; k < n_extra; k++) {
    CUP2D_REQUIRE(extra_blocks[k] >= 0 && extra_blocks[k] < nblocks_global, "cup2d_poisson_create_general_ranks: extra block out of range");
    if (extra_blocks[k] < gb || extra_blocks[k] >= ge) halo.push_back(extra_blocks[k]);
  }
  std::sort(halo.begin(), halo.end());
  halo.erase(std::unique(halo.begin(), halo.end()), halo.end());
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    set_error("cup2d_poisson_create_general_ranks: no CUDA device visible; this library has no CPU fallback");
    return CUP2D_ENOGPU;
  }
  CUP2D_REQUIRE(device >= 0 && device < ndev, "cup2d_poisson_create_general_ranks: bad device ordinal");
  CUP2D_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  CUP2D_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    set_error(std::string("cup2d_poisson_create_general_ranks: device '") + prop.name + "' is not sm_90");
    return CUP2D_ENOGPU;
  }
  cup2d_sim *s = new cup2d_sim;
  s->nglobal = nblocks_global;
  s->rank = rank;
  s->nranks = nranks;
  s->device = device;
  s->h = 1.0;
  s->poisson_only = true;
  s->rank_begin.assign(rank_begin, rank_begin + nranks + 1);
  s->gbegin = gb;
  s->nloc = nloc;
  s->halo_gid = halo;
  s->nhalo = (int64_t)halo.size();
  s->nslots = nloc + s->nhalo;
  s->halo_owner.resize(halo.size());
  s->h_halo_src.assign(2 * halo.size(), 0);
  for (size_t k = 0; k < halo.size(); k++) {
    int r = 0;
    while (!(halo[k] >= rank_begin[r] && halo[k] < rank_begin[r + 1])) r++;
    s->halo_owner[k] = r;
    s->h_halo_src[2 * k] = r;
    s->h_halo_src[2 * k + 1] = (int)(halo[k] - rank_begin[r]);
  }
  auto slot_of = [&](int32_t g) -> int {
    if (g < 0) return -1;
    if (g >= gb && g < ge) return (int)(g - gb);
    return (int)(nloc + (std::lower_bound(halo.begin(), halo.end(), g) - halo.begin()));
  };
  s->h_nbr.resize(4 * nloc);
  for (int64_t k = 0; k < 4 * nloc; k++) s->h_nbr[k] = slot_of(nbr[k]);
  s->num_sms = prop.multiProcessorCount;
  int rc = alloc_device_state(s);
  if (!rc && n_irr > 0) {
    std::vector<int32_t> col(nnz);
    for (int64_t j = 0; j < nnz; j++) col[j] = slot_of(irr_col[j] / 64) * 64 + irr_col[j] % 64;
    rc = install_general_rows(s, n_irr, irr_rows, irr_rowptr, col.data(), irr_val);
  }
  if (rc) {
    cup2d_destroy(s);
    return rc;
  }
  *out = s;
  return CUP2D_OK;
}
extern "C" {

static int alloc_device_state(cup2d_sim *s) {
  int rc = upload_tables(s);
  if (rc) return rc;
  CUP2D_CUDA(cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking));
  for (int f = 0; f < CUP2D_NFIELDS; f++) {
    const size_t bytes = (size_t)s->nslots * 64 * dim_of(f) * sizeof(double);
    CUP2D_CUDA(cudaMalloc(&s->f[f], bytes));
    CUP2D_CUDA(cudaMemset(s->f[f], 0, bytes));
  }
  const size_t vb = (size_t)s->nslots * 64 * sizeof(double);
  double **kv[] = {&s->kx[0], &s->kx[1], &s->kx[2], &s->kr, &s->krhat, &s->kp, &s->knu, &s->kt, &s->kz, &s->kzr};
  for (auto p : kv) {
    CUP2D_CUDA(cudaMalloc(p, vb));
    CUP2D_CUDA(cudaMemset(*p, 0, vb));
  }
  CUP2D_CUDA(cudaMalloc(&s->d_state, sizeof(KrylovState)));
  CUP2D_CUDA(cudaMemset(s->d_state, 0, sizeof(KrylovState)));
  CUP2D_CUDA(cudaMallocHost(&s->h_state, sizeof(KrylovState)));
  memset(s->h_state, 0, sizeof(KrylovState));
  CUP2D_CUDA(cudaMalloc(&s->d_partials, (size_t)RED_MAX_CTAS * RED_SLOTS * sizeof(double)));
  CUP2D_CUDA(cudaMalloc(&s->d_counter, sizeof(unsigned int)));
  CUP2D_CUDA(cudaMemset(s->d_counter, 0, sizeof(unsigned int)));
  CUP2D_CUDA(cudaMalloc(&s->d_scal, 16 * sizeof(double)));
  CUP2D_CUDA(cudaMallocHost(&s->h_scal, 16 * sizeof(double)));
  CUP2D_CUDA(cudaMalloc(&s->d_fac, sizeof(StepFactors)));
  CUP2D_CUDA(cudaMemset(s->d_fac, 0, sizeof(StepFactors)));
  CUP2D_CUDA(cudaMallocHost(&s->h_fac, sizeof(StepFactors)));
  memset(s->h_fac, 0, sizeof(StepFactors));
  CUP2D_CUDA(cudaMalloc(&s->d_mailbox, 4096));
  CUP2D_CUDA(cudaMemset(s->d_mailbox, 0, 4096));
  s->comm.rank = s->rank;
  s->comm.nranks = 1; // raised to nranks by cup2d_peer_attach
  s->comm.timeout_ns = 30ull * 1000000000ull; // bound of every cross-GPU wait (CUP2D_COMM_TIMEOUT_MS overrides at attach)
  {
    std::vector<int> gid(s->halo_gid.begin(), s->halo_gid.end());
    CUP2D_CUDA(cudaMalloc(&s->d_halo_gid, std::max<size_t>(gid.size(), 4) * sizeof(int)));
    if (!gid.empty()) CUP2D_CUDA(cudaMemcpy(s->d_halo_gid, gid.data(), gid.size() * sizeof(int), cudaMemcpyHostToDevice));
  }
  s->comm.mb[s->rank] = s->d_mailbox;
  CUP2D_CUDA(cudaDeviceSynchronize());
  return CUP2D_OK;
}

void cup2d_destroy(cup2d_sim *s) {
  if (!s) return;
  if (s->plan_only) {
    delete s;
    return;
  }
  cudaSetDevice(s->device);
  if (s->stream) cudaStreamSynchronize(s->stream);
  if (s->peers_attached) {
    for (int r = 0; r < s->nranks; r++) {
      if (r == s->rank) continue;
      for (auto p : s->peer_base[r])
        if (p) cudaIpcCloseMemHandle(p);
      if (s->peer_mailbox[r]) cudaIpcCloseMemHandle(s->peer_mailbox[r]);
    }
  }
  for (auto &ps : s->pipe) {
    cudaFree(ps.vel); cudaFree(ps.pres);
    if (ps.in_done) cudaEventDestroy(ps.in_done);
    if (ps.step_done) cudaEventDestroy(ps.step_done);
    if (ps.out_done) cudaEventDestroy(ps.out_done);
  }
  if (s->pipe_in) cudaStreamDestroy(s->pipe_in);
  if (s->pipe_out) cudaStreamDestroy(s->pipe_out);
  for (auto p : s->f) cudaFree(p);
  for (auto p : s->kx) cudaFree(p);
  cudaFree(s->kr); cudaFree(s->krhat); cudaFree(s->kp); cudaFree(s->knu); cudaFree(s->kt); cudaFree(s->kz); cudaFree(s->kzr);
  cudaFree(s->d_nbr); cudaFree(s->d_tiles); cudaFree(s->d_tile_org); cudaFree(s->d_halo_src); shapes_free(s);
  cudaFree(s->d_linf); cudaFree(s->d_ij);
  cudaFree(s->d_state); cudaFree(s->d_partials); cudaFree(s->d_counter); cudaFree(s->d_scal);
  cudaFree(s->d_mailbox);
  cudaFree(s->d_halo_gid); cudaFree(s->d_push_first); cudaFree(s->d_push_ent);
  cudaFree(s->d_irr_blk); cudaFree(s->d_irr_tab); cudaFree(s->d_irr_rowptr); cudaFree(s->d_irr_col); cudaFree(s->d_irr_val);
  if (s->h_state) cudaFreeHost(s->h_state);
  if (s->h_scal) cudaFreeHost(s->h_scal);
  cudaFree(s->d_fac);
  if (s->h_fac) cudaFreeHost(s->h_fac);
  for (auto &g : s->graphs) {
    if (g.exec) cudaGraphExecDestroy(g.exec);
    if (g.graph) cudaGraphDestroy(g.graph);
  }
  if (s->body_stream) cudaStreamDestroy(s->body_stream);
  for (auto e : s->prof_pool) cudaEventDestroy(e);
  if (s->stream) cudaStreamDestroy(s->stream);
  delete s;
}

int64_t cup2d_nblocks_local(const cup2d_sim *s) { return s ? s->nloc : 0; }
int64_t cup2d_nblocks_halo(const cup2d_sim *s) { return s ? s->nhalo : 0; }
int64_t cup2d_launch_count(const cup2d_sim *s) { return s ? s->launches : 0; }

static const char *kclass_name[KC_COUNT] = {"advect_stage_kernel", "umax_kernel", "pressure_rhs_kernel",
    "pressure_correct_kernel", "k_init", "k_pupdate", "k_spmv<0>", "k_r_update", "k_spmv<1>", "k_final",
    "k_p_spmv", "k_r_spmv", "k_x_final", "halo_pull_kernel", "vorticity_tag_kernel", "pressure_rhs_start_kernel"};
int cup2d_profile_enable(cup2d_sim *s, int on) {
  if (!s) return CUP2D_EINVAL;
  s->prof.clear(); // the events stay in the pool and are reused
  s->prof_pool_used = 0;
  s->prof_on = on != 0;
  return CUP2D_OK;
}
int cup2d_profile_read(cup2d_sim *s, int max_entries, char *names, double *total_ms, int64_t *launches) {
  if (!s || !names || !total_ms || !launches) return CUP2D_EINVAL;
  if (cudaStreamSynchronize(s->stream) != cudaSuccess) return CUP2D_ECUDA;
  double ms[KC_COUNT] = {};
  int64_t n[KC_COUNT] = {};
  for (auto &r : s->prof) {
    float t = 0;
    if (cudaEventElapsedTime(&t, r.a, r.b) == cudaSuccess) { ms[r.cls] += t; n[r.cls]++; }
  }
  int k = 0;
  for (int c = 0; c < KC_COUNT && k < max_entries; c++) {
    if (!n[c]) continue;
    strncpy(names + 32 * k, kclass_name[c], 31);
    names[32 * k + 31] = 0;
    total_ms[k] = ms[c];
    launches[k] = n[c];
    k++;
  }
  return k;
}
void *cup2d_stream(cup2d_sim *s) { return s ? (void *)s->stream : nullptr; }

#define CHECK_SIM(s) CUP2D_REQUIRE((s) != nullptr && !(s)->plan_only, "null or plan-only cup2d_sim (plan-only contexts have no device state)")
#define CHECK_FIELD(f) CUP2D_REQUIRE((f) >= 0 && (f) < CUP2D_NFIELDS, "bad field id")

int cup2d_field_upload(cup2d_sim *s, int field, const double *host) {
  CHECK_SIM(s); CHECK_FIELD(field);
  CUP2D_REQUIRE(host, "null host pointer");
  CUP2D_CUDA(cudaSetDevice(s->device));
  CUP2D_CUDA(cudaMemcpyAsync(s->f[field], host, (size_t)s->nloc * 64 * dim_of(field) * sizeof(double),
                             cudaMemcpyHostToDevice, s->stream));
  return CUP2D_OK;
}
int cup2d_field_download(cup2d_sim *s, int field, double *host) {
  CHECK_SIM(s); CHECK_FIELD(field);
  CUP2D_REQUIRE(host, "null host pointer");
  CUP2D_CUDA(cudaSetDevice(s->device));
  CUP2D_CUDA(cudaMemcpyAsync(host, s->f[field], (size_t)s->nloc * 64 * dim_of(field) * sizeof(double),
                             cudaMemcpyDeviceToHost, s->stream));
  CUP2D_CUDA(cudaStreamSynchronize(s->stream));
  return CUP2D_OK;
}
int cup2d_field_fill(cup2d_sim *s, int field, double value) {
  CHECK_SIM(s); CHECK_FIELD(field);
  CUP2D_REQUIRE(value == 0.0, "cup2d_field_fill: only 0 is supported");
  CUP2D_CUDA(cudaMemsetAsync(s->f[field], 0, (size_t)s->nslots * 64 * dim_of(field) * sizeof(double), s->stream));
  return CUP2D_OK;
}
void *cup2d_field_device_ptr(cup2d_sim *s, int field) {
  if (!s || field < 0 || field >= CUP2D_NFIELDS) return nullptr;
  return s->f[field];
}
int cup2d_sync(cup2d_sim *s) {
  CHECK_SIM(s);
  CUP2D_CUDA(cudaStreamSynchronize(s->stream));
  return comm_check(s); // CUP2D_ECOMM if a cross-GPU wait of this rank was given up
}

static int need_peers(cup2d_sim *s) {
  if (s->nranks > 1 && !s->peers_attached) {
    set_error("multi-rank operator called before cup2d_peer_attach");
    return CUP2D_ESTATE;
  }
  return CUP2D_OK;
}

int cup2d_compute_dt(cup2d_sim *s, double *umax_out, double *dt_out) {
  CHECK_SIM(s);
  CUP2D_CUDA(cudaSetDevice(s->device));
  double umax = 0;
  int rc = launch_umax(s, &umax);
  if (rc) return rc;
  // umax is already global: the reduction's finalizer all-reduces over the peers (common.cuh)
  const double h = s->h;
  const double dt_diff = 0.25 * h * h / (s->nu + 0.25 * h * umax); // main.cpp:6593
  const double dt_adv = h / (umax + 1e-8);                          // main.cpp:6594
  if (umax_out) *umax_out = umax;
  if (dt_out) *dt_out = std::min(dt_diff, s->cfl * dt_adv);
  return CUP2D_OK;
}

int cup2d_advect_diffuse_stage(cup2d_sim *s, int in_f, int old_f, int out_f, double coef, double dt) {
  CHECK_SIM(s);
  CUP2D_REQUIRE(in_f >= 0 && in_f < 3 && old_f >= 0 && old_f < 3 && out_f >= 0 && out_f < 3, "advect: vector field ids only");
  CUP2D_REQUIRE(out_f != in_f, "advect: out must differ from in (halo cells of in are read by other tiles)");
  CUP2D_REQUIRE(!s->poisson_only, "advect: Poisson-only context (cup2d_poisson_create) has no grid geometry");
  CUP2D_CUDA(cudaSetDevice(s->device));
  int rc = need_peers(s);
  if (rc) return rc;
  if (s->nranks > 1 && (rc = halo_exchange_ptr(s, s->f[in_f], 2, in_f))) return rc;
  return launch_advect(s, s->f[in_f], s->f[old_f], s->f[out_f], coef, dt, false);
}
int cup2d_advect_diffuse_rhs(cup2d_sim *s, int in_f, int out_f, double dt) {
  CHECK_SIM(s);
  CUP2D_REQUIRE(in_f >= 0 && in_f < 3 && out_f >= 0 && out_f < 3 && in_f != out_f, "advect_rhs: bad field ids");
  CUP2D_REQUIRE(!s->poisson_only, "advect: Poisson-only context (cup2d_poisson_create) has no grid geometry");
  CUP2D_CUDA(cudaSetDevice(s->device));
  int rc = need_peers(s);
  if (rc) return rc;
  if (s->nranks > 1 && (rc = halo_exchange_ptr(s, s->f[in_f], 2, in_f))) return rc;
  return launch_advect(s, s->f[in_f], s->f[in_f], s->f[out_f], 1.0, dt, true);
}
static int rk2(cup2d_sim *s, double dt, const StepFactors *dev);
int cup2d_advect_diffuse_rk2(cup2d_sim *s, double dt) {
  CHECK_SIM(s);
  CUP2D_REQUIRE(!s->poisson_only, "advect: Poisson-only context (cup2d_poisson_create) has no grid geometry");
  CUP2D_CUDA(cudaSetDevice(s->device));
  int rc = need_peers(s);
  if (rc) return rc;
  return rk2(s, dt, nullptr);
}
static int rk2(cup2d_sim *s, double dt, const StepFactors *dev) {
  int rc;
  // vold <- vel is a pointer swap (main.cpp:6607-6610 copies); stage 1 reads vold, writes tmpV-as-V1;
  // stage 2 reads V1, adds to vold, writes vel.  No copy kernel: 80 B/cell/step -> 64 B/cell/step.
  swap_fields(s, CUP2D_VEL, CUP2D_VOLD);
  if (s->nranks > 1) {
    if ((rc = halo_exchange_ptr(s, s->f[CUP2D_VOLD], 2, CUP2D_VOLD))) return rc;
  }
  if ((rc = launch_advect(s, s->f[CUP2D_VOLD], s->f[CUP2D_VOLD], s->f[CUP2D_TMPV], 0.5, dt, false, dev))) return rc;
  if (s->nranks > 1) {
    if ((rc = halo_exchange_ptr(s, s->f[CUP2D_TMPV], 2, CUP2D_TMPV))) return rc;
  }
  return launch_advect(s, s->f[CUP2D_TMPV], s->f[CUP2D_VOLD], s->f[CUP2D_VEL], 1.0, dt, false, dev);
}
int cup2d_pressure_rhs(cup2d_sim *s, double dt) {
  CHECK_SIM(s);
  CUP2D_REQUIRE(dt > 0, "pressure_rhs: dt must be positive");
  CUP2D_CUDA(cudaSetDevice(s->device));
  int rc = need_peers(s);
  if (rc) return rc;
  return launch_pressure_rhs(s, dt, true);
}
int cup2d_poisson_solve(cup2d_sim *s, double tol_abs, double tol_rel, int max_restarts, int max_iter,
                        int *iters, double *err) {
  CHECK_SIM(s);
  CUP2D_CUDA(cudaSetDevice(s->device));
  int rc = need_peers(s);
  if (rc) return rc;
  rc = poisson_solve(s, tol_abs, tol_rel, max_restarts, max_iter, iters, err);
  if (rc) return rc;
  CUP2D_CUDA(cudaMemcpyAsync(s->f[CUP2D_PRES], s->kx[s->h_state->opt], (size_t)s->nloc * 64 * sizeof(double),
                             cudaMemcpyDeviceToDevice, s->stream));
  return CUP2D_OK;
}
int cup2d_adapt_tags(cup2d_sim *s, double rtol, int chi_cells, double *block_linf_out) {
  CHECK_SIM(s);
  CUP2D_REQUIRE(!s->poisson_only, "adapt_tags: a Poisson-only context has no velocity field");
  CUP2D_REQUIRE(chi_cells >= 0 && chi_cells <= CUP2D_BS, "adapt_tags: chi_cells must be 0..8 (the reference uses 2 or 4)");
  CUP2D_CUDA(cudaSetDevice(s->device));
  int rc = need_peers(s);
  if (rc) return rc;
  return launch_adapt_tags(s, rtol, chi_cells, block_linf_out);
}
int cup2d_vorticity_tag(cup2d_sim *s, double *block_linf_out) { return cup2d_adapt_tags(s, 0.0, 0, block_linf_out); }
int cup2d_dump(cup2d_sim *s, double time, const char *path) {
  CHECK_SIM(s);
  CUP2D_REQUIRE(!s->poisson_only && path && *path, "dump: bad arguments");
  CUP2D_CUDA(cudaSetDevice(s->device));
  return dump_fields(s, time, path);
}
#define CHECK_SHAPE(s, shape, must_exist)                                                         \
  CUP2D_REQUIRE(!s->poisson_only, "shape call on a Poisson-only context");                        \
  CUP2D_REQUIRE(shape >= 0 && shape < 64, "shape index out of range (0..63)");                    \
  CUP2D_REQUIRE(!(must_exist) || shape < (int)s->shapes.size(), "shape has not been set (cup2d_shape_set)")
int cup2d_shape_set(cup2d_sim *s, int shape, int nob, const int32_t *block_ids, const double *chi,
                    const double *udef) {
  CHECK_SIM(s);
  CHECK_SHAPE(s, shape, false);
  CUP2D_REQUIRE(nob >= 0 && (nob == 0 || (block_ids && chi && udef)), "cup2d_shape_set: bad arguments");
  for (int k = 0; k < nob; k++)
    CUP2D_REQUIRE(block_ids[k] >= 0 && block_ids[k] < s->nloc, "cup2d_shape_set: block id outside the local range");
  CUP2D_CUDA(cudaSetDevice(s->device));
  return shape_set(s, shape, nob, block_ids, chi, udef);
}
int cup2d_shape_integrals(cup2d_sim *s, int shape, double lambda, double dt, double cx, double cy, double *out7) {
  CHECK_SIM(s);
  CHECK_SHAPE(s, shape, true);
  CUP2D_REQUIRE(out7, "cup2d_shape_integrals: null output");
  CUP2D_CUDA(cudaSetDevice(s->device));
  int rc = need_peers(s);
  if (rc) return rc;
  return shape_integrals(s, shape, lambda, dt, cx, cy, out7);
}
int cup2d_penalize(cup2d_sim *s, int shape, double lambda, double dt, double cx, double cy, double us, double vs,
                   double omega) {
  CHECK_SIM(s);
  CHECK_SHAPE(s, shape, true);
  CUP2D_CUDA(cudaSetDevice(s->device));
  return shape_penalize(s, shape, lambda, dt, cx, cy, us, vs, omega);
}
int cup2d_udef_assemble(cup2d_sim *s) {
  CHECK_SIM(s);
  CUP2D_REQUIRE(!s->poisson_only, "udef_assemble on a Poisson-only context");
  CUP2D_CUDA(cudaSetDevice(s->device));
  return udef_assemble(s);
}
int cup2d_pressure_correct(cup2d_sim *s, double dt) {
  CHECK_SIM(s);
  CUP2D_CUDA(cudaSetDevice(s->device));
  int rc = need_peers(s);
  if (rc) return rc;
  return launch_pressure_correct(s, dt);
}

} // extern "C"

namespace cup2d {

// The Krylov solve of an enqueued step on s->stream (b = tmp and x0 = pres, or b formed from the step's right-hand side and
// x0 = 0; the iterate stays in the Krylov buffers, KrylovState::opt names the best one).  Fixed work is queued at once; a tolerance-driven solve is, while `capturing`, a WHILE node whose
// body is one iteration, and otherwise host-polled in batches of 8 (the only host waits, in direct launches only).
int poisson_enqueue(cup2d_sim *s, double tol_abs, double tol_rel, int max_restarts, int max_iter, bool capturing,
                    const StepRhs *rhs) {
  const bool tol = tol_abs > 0 || tol_rel > 0;
#ifndef CUP2D_FULL_EMU
  cudaGraph_t cap_graph = nullptr;
  if (capturing && tol && max_iter > 0) {
    // tolerance-driven solve inside a graph: a WHILE node whose body is one iteration.  Its condition starts at 1 on
    // every launch; the last CTA of the starting kernel and of every k_final / k_x_final sets it to !done
    // (cudaGraphSetConditional).
    cudaStreamCaptureStatus st;
    CUP2D_CUDA(cudaStreamGetCaptureInfo(s->stream, &st, nullptr, &cap_graph, nullptr, nullptr));
    cudaGraphConditionalHandle handle;
    CUP2D_CUDA(cudaGraphConditionalHandleCreate(&handle, cap_graph, 1, cudaGraphCondAssignDefault));
    s->cond_handle = (unsigned long long)handle;
  }
#endif
  int rc = rhs ? poisson_begin_rhs(s, tol_abs, tol_rel, max_restarts, max_iter, *rhs)
               : poisson_begin(s, tol_abs, tol_rel, max_restarts, max_iter);
  if (rc) {
    s->cond_handle = 0;
    return rc;
  }
  if (max_iter > 0) {
    if (!tol) {
      if ((rc = poisson_iterations(s, max_iter, s->stream))) return rc;
    } else if (capturing) {
#ifndef CUP2D_FULL_EMU
      cudaStreamCaptureStatus st;
      const cudaGraphNode_t *deps = nullptr;
      size_t ndeps = 0;
      cudaError_t e = cudaStreamGetCaptureInfo(s->stream, &st, nullptr, &cap_graph, &deps, &ndeps);
      cudaGraphNodeParams np = {cudaGraphNodeTypeConditional};
      np.type = cudaGraphNodeTypeConditional;
      np.conditional.handle = (cudaGraphConditionalHandle)s->cond_handle;
      np.conditional.type = cudaGraphCondTypeWhile;
      np.conditional.size = 1;
      cudaGraphNode_t loop = nullptr;
      if (e == cudaSuccess) e = cudaGraphAddNode(&loop, cap_graph, deps, ndeps, &np);
      if (e == cudaSuccess && !s->body_stream) e = cudaStreamCreateWithFlags(&s->body_stream, cudaStreamNonBlocking);
      if (e == cudaSuccess)
        e = cudaStreamBeginCaptureToGraph(s->body_stream, np.conditional.phGraph_out[0], nullptr, nullptr, 0, cudaStreamCaptureModeRelaxed);
      if (e != cudaSuccess) {
        s->cond_handle = 0;
        CUP2D_CUDA(e);
      }
      rc = poisson_iterations(s, 1, s->body_stream);
      s->cond_handle = 0;
      cudaGraph_t body = nullptr;
      e = cudaStreamEndCapture(s->body_stream, &body);
      if (rc) return rc;
      CUP2D_CUDA(e);
      CUP2D_CUDA(cudaStreamUpdateCaptureDependencies(s->stream, &loop, 1, cudaStreamSetCaptureDependencies));
#endif
    } else {
      // direct launches (profiling, first step of a context): the host looks at the `done` flag every 8 iterations
      int launched = 0;
      while (launched < max_iter) {
        const int batch = max_iter - launched < 8 ? max_iter - launched : 8;
        if ((rc = poisson_iterations(s, batch, s->stream))) return rc;
        launched += batch;
        if ((rc = poisson_result(s, nullptr, nullptr))) return rc;
        if (s->h_state->done) break;
      }
    }
  }
  return CUP2D_OK;
}

} // namespace cup2d

extern "C" {

// ---- one time step, enqueued without any host synchronisation --------------------------------------------------------
// The body: [umax + dt rule on the device] -> RK2 -> Poisson right-hand side -> BiCGSTAB -> correction.  Every dt-dependent
// kernel reads the device-resident StepFactors, the correction picks the best Krylov iterate through the device-side state,
// cross-GPU epochs are device counters: nothing in the body depends on a host value that changes from step to step, so the
// body can be captured ONCE per buffer assignment into a CUDA graph and replayed with a single cudaGraphLaunch (the
// reference needs ~25 launches + 4 host synchronisations per Krylov iteration, cuda.cu:403-548).  A tolerance-driven solve
// is a WHILE node whose condition the last CTA of the iteration's final kernel sets (cudaGraphSetConditional): the data-
// dependent loop runs on the device too.
static int step_body(cup2d_sim *s, bool dev_dt, int keep_udef, double tol_abs, double tol_rel, int max_restarts, int max_iter,
                     bool capturing) {
  int rc;
  if (dev_dt) {
    if ((rc = launch_umax_async(s))) return rc;
    if ((rc = launch_step_factors(s, 0.0))) return rc;
  }
  if ((rc = rk2(s, 0.0, s->d_fac))) return rc;
  // keep_udef = 0: no bodies, the sum of u_def is identically zero (main.cpp:6980-6983), so the RHS
  // kernel skips the chi*div(u_def) term instead of reading a zeroed field (tmpV keeps RK scratch).
  // keep_udef = 1: the caller uploaded chi and the summed u_def into tmpV after the RK2 stages.
  // The solve starts in the kernel that forms the right-hand side (x0 = 0): neither b nor x0 goes through tmp / pres, so
  // after a step tmp does not hold b (cup2d_pressure_rhs still writes it there).
  const StepRhs rhs{keep_udef != 0, s->d_fac};
  if ((rc = poisson_enqueue(s, tol_abs, tol_rel, max_restarts, max_iter, capturing, &rhs))) return rc;
  return launch_pressure_correct(s, 1.0, s->d_fac, true);
}

int cup2d_set_graph(cup2d_sim *s, int on) {
  CHECK_SIM(s);
  s->use_graph = on != 0;
  return CUP2D_OK;
}

int cup2d_step_enqueue(cup2d_sim *s, double dt_in, int keep_udef, double tol_abs, double tol_rel, int max_restarts,
                       int max_iter) {
  CHECK_SIM(s);
  CUP2D_REQUIRE(!s->poisson_only, "cup2d_step: Poisson-only context");
  CUP2D_CUDA(cudaSetDevice(s->device));
  int rc = need_peers(s);
  if (rc) return rc;
  const bool dev_dt = !(dt_in > 0);
  if (!dev_dt && (rc = launch_step_factors(s, dt_in))) return rc; // by-value dt: outside the graph
  s->step_pending = true;
  bool graph = s->use_graph && !s->prof_on && s->warmed;
#ifdef CUP2D_FULL_EMU
  graph = false;
#endif
  if (!graph) {
    s->warmed = true; // the first step of a context runs directly: one-time tables and kernel attributes are set up in it
    return step_body(s, dev_dt, keep_udef, tol_abs, tol_rel, max_restarts, max_iter, false);
  }
#ifndef CUP2D_FULL_EMU
  // one executable graph per assignment of buffers to roles (the body swaps vel<->vold and pres<->pold, so successive
  // steps alternate between two assignments; the host-buffer pipeline adds its staging sets) and per argument set
  std::vector<unsigned long long> key;
  for (int f = 0; f < CUP2D_NFIELDS; f++) key.push_back((unsigned long long)(uintptr_t)s->f[f]);
  auto bits = [](double v) { unsigned long long u; memcpy(&u, &v, 8); return u; };
  key.insert(key.end(), {(unsigned long long)dev_dt, (unsigned long long)(keep_udef != 0), bits(tol_abs), bits(tol_rel),
                         (unsigned long long)max_restarts, (unsigned long long)max_iter, (unsigned long long)s->n_irr_rows});
  cup2d_sim::StepGraph *hit = nullptr;
  for (auto &g : s->graphs)
    if (g.key == key) hit = &g;
  if (!hit) {
    if (s->graphs.size() >= 32) { // a caller cycling through many buffer sets: drop the oldest
      cudaGraphExecDestroy(s->graphs.front().exec);
      cudaGraphDestroy(s->graphs.front().graph);
      s->graphs.erase(s->graphs.begin());
    }
    const int64_t l0 = s->launches;
    double *f0[CUP2D_NFIELDS];
    void *pb0[MAX_RANKS][CUP2D_NFIELDS + 5];
    memcpy(f0, s->f, sizeof f0);
    memcpy(pb0, s->peer_base, sizeof pb0);
    CUP2D_CUDA(cudaStreamBeginCapture(s->stream, cudaStreamCaptureModeRelaxed));
    rc = step_body(s, dev_dt, keep_udef, tol_abs, tol_rel, max_restarts, max_iter, true);
    cudaGraph_t g = nullptr;
    const cudaError_t e = cudaStreamEndCapture(s->stream, &g);
    // capturing applied the body's buffer swaps to the context; undo them, the launch below applies them again
    memcpy(s->f, f0, sizeof f0);
    memcpy(s->peer_base, pb0, sizeof pb0);
    const int64_t nl = s->launches - l0;
    s->launches = l0;
    if (rc) {
      if (g) cudaGraphDestroy(g);
      return rc;
    }
    CUP2D_CUDA(e);
    cup2d_sim::StepGraph sg;
    sg.key = key;
    sg.graph = g;
    sg.launches = nl;
    CUP2D_CUDA(cudaGraphInstantiate(&sg.exec, g, 0));
    s->graphs.push_back(sg);
    hit = &s->graphs.back();
  }
  CUP2D_CUDA(cudaGraphLaunch(hit->exec, s->stream));
  s->launches += hit->launches;
  // the buffer swaps the body makes on the host side (rk2: vel <-> vold; right-hand side: pres <-> pold)
  swap_fields(s, CUP2D_VEL, CUP2D_VOLD);
  swap_fields(s, CUP2D_PRES, CUP2D_POLD);
#endif
  return CUP2D_OK;
}

int cup2d_step_result(cup2d_sim *s, double *dt_out, int *iters_out, double *err_out) {
  CHECK_SIM(s);
  CUP2D_CUDA(cudaSetDevice(s->device));
  CUP2D_CUDA(cudaMemcpyAsync(s->h_fac, s->d_fac, sizeof(StepFactors), cudaMemcpyDeviceToHost, s->stream));
  const int rc = poisson_result(s, iters_out, err_out); // synchronises the stream
  if (dt_out) *dt_out = s->h_fac->dt;
  s->step_pending = false;
  return rc;
}

int cup2d_step(cup2d_sim *s, double dt_in, int keep_udef, double tol_abs, double tol_rel,
               int max_restarts, int max_iter, double *dt_out, int *iters_out, double *err_out) {
  const int rc = cup2d_step_enqueue(s, dt_in, keep_udef, tol_abs, tol_rel, max_restarts, max_iter);
  if (rc) return rc;
  return cup2d_step_result(s, dt_out, iters_out, err_out);
}

/* ---- host-buffer pipeline: upload(n+1) || step(n) || download(n-1) on three streams (include/cup2d_b200.h) ---- */
static int pipe_slot(cup2d_sim *s, int slot) {
  CHECK_SIM(s);
  CUP2D_REQUIRE(slot >= 0 && slot < CUP2D_PIPE_SLOTS, "cup2d_pipe: slot out of range");
  CUP2D_REQUIRE(s->nranks == 1 && !s->poisson_only, "cup2d_pipe: single-rank contexts with a grid only (peer mappings are tied to the field buffers)");
  CUP2D_CUDA(cudaSetDevice(s->device));
  if (!s->pipe_in) {
    CUP2D_CUDA(cudaStreamCreateWithFlags(&s->pipe_in, cudaStreamNonBlocking));
    CUP2D_CUDA(cudaStreamCreateWithFlags(&s->pipe_out, cudaStreamNonBlocking));
  }
  cup2d_sim::PipeSet &ps = s->pipe[slot];
  if (!ps.vel) {
    CUP2D_CUDA(cudaMalloc(&ps.vel, (size_t)s->nslots * 128 * sizeof(double)));
    CUP2D_CUDA(cudaMalloc(&ps.pres, (size_t)s->nslots * 64 * sizeof(double)));
    CUP2D_CUDA(cudaEventCreateWithFlags(&ps.in_done, cudaEventDisableTiming));
    CUP2D_CUDA(cudaEventCreateWithFlags(&ps.step_done, cudaEventDisableTiming));
    CUP2D_CUDA(cudaEventCreateWithFlags(&ps.out_done, cudaEventDisableTiming));
  }
  return CUP2D_OK;
}
int cup2d_pipe_upload(cup2d_sim *s, int slot, const double *vel_host, const double *pres_host) {
  int rc = pipe_slot(s, slot);
  if (rc) return rc;
  CUP2D_REQUIRE(vel_host && pres_host, "cup2d_pipe_upload: null host pointer");
  cup2d_sim::PipeSet &ps = s->pipe[slot];
  // the set may still be written by a step or read by a download enqueued earlier (a never-recorded event does not block)
  CUP2D_CUDA(cudaStreamWaitEvent(s->pipe_in, ps.step_done, 0));
  CUP2D_CUDA(cudaStreamWaitEvent(s->pipe_in, ps.out_done, 0));
  CUP2D_CUDA(cudaMemcpyAsync(ps.vel, vel_host, (size_t)s->nloc * 128 * sizeof(double), cudaMemcpyHostToDevice, s->pipe_in));
  CUP2D_CUDA(cudaMemcpyAsync(ps.pres, pres_host, (size_t)s->nloc * 64 * sizeof(double), cudaMemcpyHostToDevice, s->pipe_in));
  CUP2D_CUDA(cudaEventRecord(ps.in_done, s->pipe_in));
  return CUP2D_OK;
}
int cup2d_pipe_step(cup2d_sim *s, int slot, double dt_in, double tol_abs, double tol_rel, int max_restarts, int max_iter,
                    double *dt_out, int *iters_out, double *err_out) {
  int rc = pipe_slot(s, slot);
  if (rc) return rc;
  cup2d_sim::PipeSet &ps = s->pipe[slot];
  CUP2D_CUDA(cudaStreamWaitEvent(s->stream, ps.in_done, 0));
  CUP2D_CUDA(cudaStreamWaitEvent(s->stream, ps.out_done, 0)); // a download of this set's previous contents
  // The context trades its vel / pres buffers for the set's for the duration of the step and trades back afterwards: the
  // step swaps buffers internally (vold <-> vel, pold <-> pres), so what comes back to the set are the buffers that hold
  // the RESULT, whichever they are, and the context keeps the same number of buffers it had.  Work enqueued on s->stream by
  // later steps never touches a buffer a set owns, so a download can run beside the next step.
  std::swap(s->f[CUP2D_VEL], ps.vel);
  std::swap(s->f[CUP2D_PRES], ps.pres);
  rc = cup2d_step(s, dt_in, 0, tol_abs, tol_rel, max_restarts, max_iter, dt_out, iters_out, err_out);
  std::swap(s->f[CUP2D_VEL], ps.vel);
  std::swap(s->f[CUP2D_PRES], ps.pres);
  if (rc) return rc;
  CUP2D_CUDA(cudaEventRecord(ps.step_done, s->stream));
  return CUP2D_OK;
}
int cup2d_pipe_download(cup2d_sim *s, int slot, double *vel_host, double *pres_host) {
  int rc = pipe_slot(s, slot);
  if (rc) return rc;
  CUP2D_REQUIRE(vel_host && pres_host, "cup2d_pipe_download: null host pointer");
  cup2d_sim::PipeSet &ps = s->pipe[slot];
  CUP2D_CUDA(cudaStreamWaitEvent(s->pipe_out, ps.in_done, 0));
  CUP2D_CUDA(cudaStreamWaitEvent(s->pipe_out, ps.step_done, 0));
  CUP2D_CUDA(cudaMemcpyAsync(vel_host, ps.vel, (size_t)s->nloc * 128 * sizeof(double), cudaMemcpyDeviceToHost, s->pipe_out));
  CUP2D_CUDA(cudaMemcpyAsync(pres_host, ps.pres, (size_t)s->nloc * 64 * sizeof(double), cudaMemcpyDeviceToHost, s->pipe_out));
  CUP2D_CUDA(cudaEventRecord(ps.out_done, s->pipe_out));
  return CUP2D_OK;
}
int cup2d_pipe_wait(cup2d_sim *s, int slot) {
  int rc = pipe_slot(s, slot);
  if (rc) return rc;
  CUP2D_CUDA(cudaEventSynchronize(s->pipe[slot].out_done));
  return CUP2D_OK;
}

} // extern "C"
