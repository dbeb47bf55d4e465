// Glue for running the reference's OWN time loop with its hot path on libcup2d_b200.so (INTEGRATION.md section 2 as code).
//
// The reference keeps every field as one malloc'ed array per block (Grid::infos[i].block).  This header is force-included
// in front of the reference translation unit; the two code fragments patched_loop_rk2.inc / patched_loop_pressure.inc are
// spliced over main.cpp:6607-6642 (RK2 advect-diffuse) and main.cpp:7007-7187 (Poisson right-hand side, solve, correction)
// by line number at build time (oracle/Makefile, target ref_patched) — no reference source is stored in this repository.
// Everything between the two ranges (penalisation, rigid-body solve, collisions, u_def assembly: main.cpp:6643-7006) keeps
// running on the host on host fields, so this first form ships vel / chi / u_def / pres across PCIe twice per step; the
// device-resident form replaces those host phases with the cup2d_shape_* calls.  One uniform level only (cup2d_create).
// The multi-level forms use the cup2d_amr_* part below; the device form (amr_device_*.inc) keeps one context for the whole run
// and regrids it in place (regrid_amr), so that after its initial upload no field crosses PCIe (field_bytes counts them).
#pragma once
#include "cup2d_b200.h"
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

namespace b200 {
inline cup2d_sim *ctx = nullptr;
inline std::vector<double> stage;
inline uint64_t field_bytes = 0; // field bytes moved between host and device by the upload / download helpers below

inline void check(int rc, const char *what) {
  if (rc) {
    fprintf(stderr, "cup2d_b200: %s failed (%d): %s\n", what, rc, cup2d_last_error());
    abort();
  }
}
// create the device context from the reference's own block list the first time it is needed
template <class Sim, class GridT> void ensure(const Sim &sim, GridT *grid) {
  if (ctx) return;
  const auto &infos = grid->infos;
  const int level = infos[0].level;
  std::vector<int32_t> ij(2 * infos.size());
  for (size_t i = 0; i < infos.size(); i++) {
    if (infos[i].level != level) {
      fprintf(stderr, "cup2d_b200 loop glue: the mesh is not on one level (block %zu)\n", i);
      abort();
    }
    ij[2 * i] = infos[i].index[0];
    ij[2 * i + 1] = infos[i].index[1];
  }
  int64_t rank_begin[2] = {0, (int64_t)infos.size()};
  cup2d_config cfg;
  memset(&cfg, 0, sizeof cfg);
  cfg.nbx = sim.bpdx << level;
  cfg.nby = sim.bpdy << level;
  cfg.nblocks_global = (int64_t)infos.size();
  cfg.block_ij = ij.data();
  cfg.rank = 0;
  cfg.nranks = 1;
  cfg.rank_begin = rank_begin;
  cfg.h = infos[0].h;
  cfg.nu = sim.nu;
  cfg.cfl = sim.CFL;
  cfg.device = 0;
  check(cup2d_create(&cfg, &ctx), "cup2d_create");
}
template <class GridT> void upload(int field, GridT *grid, int dim) {
  const auto &infos = grid->infos;
  const size_t n = (size_t)dim * CUP2D_BS * CUP2D_BS;
  stage.resize(infos.size() * n);
  for (size_t i = 0; i < infos.size(); i++) memcpy(stage.data() + i * n, infos[i].block, n * sizeof(double));
  check(cup2d_field_upload(ctx, field, stage.data()), "cup2d_field_upload");
  field_bytes += stage.size() * sizeof(double);
}
template <class GridT> void download(int field, GridT *grid, int dim) {
  auto &infos = grid->infos;
  const size_t n = (size_t)dim * CUP2D_BS * CUP2D_BS;
  stage.resize(infos.size() * n);
  check(cup2d_field_download(ctx, field, stage.data()), "cup2d_field_download");
  field_bytes += stage.size() * sizeof(double);
  for (size_t i = 0; i < infos.size(); i++) memcpy(infos[i].block, stage.data() + i * n, n * sizeof(double));
}
// hand one shape's obstacle blocks (main.cpp:3283-3286: per block its own chi and u_def) to the device
template <class ShapeT> void shape_set(int k, const ShapeT &shape) {
  std::vector<int32_t> ids;
  std::vector<double> X, U;
  const auto &ob = shape->obstacleBlocks;
  for (size_t i = 0; i < ob.size(); i++) {
    if (!ob[i]) continue;
    ids.push_back((int32_t)i);
    const double *c = (const double *)ob[i]->chi, *u = (const double *)ob[i]->udef;
    X.insert(X.end(), c, c + CUP2D_BS * CUP2D_BS);
    U.insert(U.end(), u, u + 2 * CUP2D_BS * CUP2D_BS);
  }
  check(cup2d_shape_set(ctx, k, (int)ids.size(), ids.data(), X.data(), U.data()), "cup2d_shape_set");
}
// ---- multi-level meshes: the same glue on the cup2d_amr context, re-created whenever adapt() changed the mesh ----------
inline cup2d_amr *amr = nullptr;
inline std::vector<int32_t> amr_mesh;
template <class Sim, class GridT> void ensure_amr(const Sim &sim, GridT *grid) {
  const auto &infos = grid->infos;
  std::vector<int32_t> mesh(3 * infos.size());
  for (size_t i = 0; i < infos.size(); i++) {
    mesh[3 * i] = infos[i].level;
    mesh[3 * i + 1] = infos[i].index[0];
    mesh[3 * i + 2] = infos[i].index[1];
  }
  if (amr && mesh == amr_mesh) return;
  if (amr) cup2d_amr_destroy(amr);
  amr = nullptr;
  check(cup2d_amr_create((int64_t)infos.size(), mesh.data(), sim.bpdx, sim.bpdy, sim.h0, sim.nu, 0, &amr), "cup2d_amr_create");
  if (const char *e = getenv("CUP2D_B200_AMR_FAST")) check(cup2d_amr_set_fast(amr, atoi(e)), "cup2d_amr_set_fast");
  amr_mesh.swap(mesh);
}
// the device form (dropin/amr_device_*.inc) keeps ONE context for the whole run: adapt()'s new mesh is applied in place with
// adapt()'s field transfer on the device (cup2d_amr_regrid, a no-op when the mesh did not change)
template <class GridT> void regrid_amr(GridT *grid) {
  const auto &infos = grid->infos;
  std::vector<int32_t> mesh(3 * infos.size());
  for (size_t i = 0; i < infos.size(); i++) {
    mesh[3 * i] = infos[i].level;
    mesh[3 * i + 1] = infos[i].index[0];
    mesh[3 * i + 2] = infos[i].index[1];
  }
  if (mesh == amr_mesh) return;
  check(cup2d_amr_regrid(amr, (int64_t)infos.size(), mesh.data()), "cup2d_amr_regrid");
  amr_mesh.swap(mesh);
}
template <class GridT> void amr_upload(int field, GridT *grid, int dim) {
  const auto &infos = grid->infos;
  const size_t n = (size_t)dim * CUP2D_BS * CUP2D_BS;
  stage.resize(infos.size() * n);
  for (size_t i = 0; i < infos.size(); i++) memcpy(stage.data() + i * n, infos[i].block, n * sizeof(double));
  check(cup2d_amr_field_upload(amr, field, stage.data()), "cup2d_amr_field_upload");
  field_bytes += stage.size() * sizeof(double);
}
template <class GridT> void amr_download(int field, GridT *grid, int dim) {
  auto &infos = grid->infos;
  const size_t n = (size_t)dim * CUP2D_BS * CUP2D_BS;
  stage.resize(infos.size() * n);
  check(cup2d_amr_field_download(amr, field, stage.data()), "cup2d_amr_field_download");
  field_bytes += stage.size() * sizeof(double);
  for (size_t i = 0; i < infos.size(); i++) memcpy(infos[i].block, stage.data() + i * n, n * sizeof(double));
}
template <class ShapeT> void amr_shape_set(int k, const ShapeT &shape) {
  std::vector<int32_t> ids;
  std::vector<double> X, U;
  const auto &ob = shape->obstacleBlocks;
  for (size_t i = 0; i < ob.size(); i++) {
    if (!ob[i]) continue;
    ids.push_back((int32_t)i);
    const double *c = (const double *)ob[i]->chi, *u = (const double *)ob[i]->udef;
    X.insert(X.end(), c, c + CUP2D_BS * CUP2D_BS);
    U.insert(U.end(), u, u + 2 * CUP2D_BS * CUP2D_BS);
  }
  check(cup2d_amr_shape_set(amr, k, (int)ids.size(), ids.data(), X.data(), U.data()), "cup2d_amr_shape_set");
  field_bytes += (X.size() + U.size()) * sizeof(double);
}
// the device form: the context is created at the first ongrid() (main.cpp:6543) from the initial block list, and the initial
// velocity and pressure are its only field upload; from then on every field lives on the device
template <class Sim, class GridT, class PresT> void ensure_amr_device(const Sim &sim, GridT *vel, PresT *pres) {
  if (amr) return;
  ensure_amr(sim, vel);
  amr_upload(CUP2D_VEL, vel, 2);
  amr_upload(CUP2D_PRES, pres, 1);
}
inline bool device_tags() { // adapt()'s tagging field from the device (default) or from the reference's own host sweeps
  const char *e = getenv("CUP2D_B200_AMR_TAGS");
  return !e || atoi(e) != 0;
}
inline int max_iter() { // cuda.cu:438 hard-codes 1000; the test harness may lower it
  const char *e = getenv("CUP2D_B200_MAX_ITER");
  return e ? atoi(e) : 1000;
}
} // namespace b200
