// TEST INFRASTRUCTURE — generator of tests/golden/amrforces_*.npz (tests/golden/make_forces_golden.py), never shipped.
//
// Includes the UNMODIFIED reference translation unit (/root/reference/main.cpp, only `main` renamed) and runs its run.sh case.
// The surface normals (ComputeSurfaceNormals, main.cpp:3774-3828, called from ongrid() at 4470) and the force diagnostics
// (KernelComputeForces, 5573-5746, and the reductions of 7188-7284) are observed through the MPI_Allreduce hook of
// oracle/shim/mpi.h, with no source patch:
//   the first MPI_SUM of count 3 of an ongrid() (4483, after the normals): the mesh, chi, tmp and per shape the obstacle ids
//   and every obstacle block's surface list;
//   every MPI_SUM of count 19 (7252), one per shape: vel, pres, chi and the reference's own labs of the obstacle blocks (at the
//   first), per shape u, v, centerOfMass, ids, chi, udef, the 14 skin arrays, the per-block accumulators and the buffer;
//   the first hook after the count-19 one of shape k: Pthrust, Pdrag, EffPDef, EffPDefBnd of shape k (7273-7280).
//
//   ref_forces levelMax first count out.bin     records the time steps first .. first + count - 1
//   record stream [tag, n, n doubles]; every step starts with tag 1 = {step, nshapes, h0, bpdx, bpdy, nu}
//     2: mesh (level, i, j)   3: chi at ongrid   4: tmp at ongrid   5: vel   6: pres   7: chi at the forces
//     8: the blocks whose labs follow (every shape's obstacle blocks, ascending)
//     9: VectorLab of vel, stencil {-4,-4,5,5,tensorial} (16*16*2 per block)   10: ScalarLab of chi, same stencil (16*16)
//     per shape k (tag + 100 k): 20 ids at ongrid   21 surface points per block   22 (ix, iy, dchidx, dchidy, delta) rows
//       30 {u, v, cmx, cmy}   31 ids   32 chi   33 udef   34 skin [n][14]   35 per-block accumulators [nob][19]
//       36 the 19-value buffer   37 Pthrust, Pdrag, EffPDef, EffPDefBnd
#define CUP2D_REF_HOOK_TU 1
#define main ref_main
#include "main.cpp" // resolved with -I/root/reference
#undef main

namespace {
int g_first = 0, g_count = 0, g_n3 = 0, g_n19 = 0, g_derived = -1;
bool g_armed = true;
FILE *g_fout = nullptr;

void put(double tag, const std::vector<double> &v) {
  const double hdr[2] = {tag, (double)v.size()};
  fwrite(hdr, sizeof(double), 2, g_fout);
  fwrite(v.data(), sizeof(double), v.size(), g_fout);
}
void put_blocks(double tag, Grid *g, int dim) {
  std::vector<double> v;
  for (auto &info : g->infos) v.insert(v.end(), info.block, info.block + dim * _BS_ * _BS_);
  put(tag, v);
}
template <class F> void put_obstacles(double tag, Shape *s, F f) {
  std::vector<double> v;
  for (size_t id = 0; id < s->obstacleBlocks.size(); id++)
    if (s->obstacleBlocks[id]) f(*s->obstacleBlocks[id], v, id);
  put(tag, v);
}
template <class LabT, int DIM> struct DumpLab { // a "kernel" that only copies the assembled lab out
  Stencil stencil;
  std::vector<double> *out;
  int nm;
  DumpLab(Stencil st, std::vector<double> *o) : stencil(st), out(o), nm(_BS_ + st.ex - st.sx - 1) {}
  void operator()(LabT *lab, const Info *info) const {
    const size_t n = (size_t)nm * nm * DIM;
    memcpy(out->data() + (size_t)info->id * n, lab->m, n * sizeof(double));
  }
};
bool recording() { return sim.step >= g_first && sim.step < g_first + g_count; }

void on_normals() { // ongrid() of a recorded step, after ComputeSurfaceNormals
  const size_t ns = sim.shapes.size();
  put(1, {(double)sim.step, (double)ns, sim.h0, (double)sim.bpdx, (double)sim.bpdy, sim.nu});
  std::vector<double> mesh;
  for (auto &info : var.chi->infos) { mesh.push_back(info.level); mesh.push_back(info.index[0]); mesh.push_back(info.index[1]); }
  put(2, mesh);
  put_blocks(3, var.chi, 1);
  put_blocks(4, var.tmp, 1);
  for (size_t k = 0; k < ns; k++) {
    Shape *s = sim.shapes[k];
    const double b = 100.0 * k;
    put_obstacles(b + 20, s, [](Obstacle &, std::vector<double> &v, size_t id) { v.push_back((double)id); });
    put_obstacles(b + 21, s, [](Obstacle &o, std::vector<double> &v, size_t) { v.push_back((double)o.n_surfPoints); });
    put_obstacles(b + 22, s, [](Obstacle &o, std::vector<double> &v, size_t) {
      for (auto &p : o.surface) v.insert(v.end(), {(double)p.ix, (double)p.iy, p.dchidx, p.dchidy, p.delta});
    });
  }
}

void on_fields() { // the first count-19 sum of a recorded step: fields and the reference's labs of the obstacle blocks
  put_blocks(5, var.vel, 2);
  put_blocks(6, var.pres, 1);
  put_blocks(7, var.chi, 1);
  const size_t nb = var.vel->infos.size();
  std::vector<char> ob(nb, 0);
  for (Shape *s : sim.shapes)
    for (size_t id = 0; id < s->obstacleBlocks.size(); id++)
      if (s->obstacleBlocks[id]) ob[id] = 1;
  std::vector<double> ids;
  for (size_t id = 0; id < nb; id++)
    if (ob[id]) ids.push_back((double)id);
  put(8, ids);
  g_armed = false; // the lab loads below are not part of the time step
  std::vector<double> lab(nb * 16 * 16 * 2), sel;
  computeA<VectorLab>(DumpLab<VectorLab, 2>(Stencil{-4, -4, 5, 5, true}, &lab), var.vel, 2);
  for (double id : ids) sel.insert(sel.end(), lab.begin() + (size_t)id * 512, lab.begin() + (size_t)id * 512 + 512);
  put(9, sel);
  sel.clear();
  computeA<ScalarLab>(DumpLab<ScalarLab, 1>(Stencil{-4, -4, 5, 5, true}, &lab), var.chi, 1);
  for (double id : ids) sel.insert(sel.end(), lab.begin() + (size_t)id * 256, lab.begin() + (size_t)id * 256 + 256);
  put(10, sel);
  g_armed = true;
}

void on_forces(int k, const double *buf) {
  if (k == 0) on_fields();
  Shape *s = sim.shapes[k];
  const double b = 100.0 * k;
  put(b + 30, {s->u, s->v, s->centerOfMass[0], s->centerOfMass[1]});
  put_obstacles(b + 31, s, [](Obstacle &, std::vector<double> &v, size_t id) { v.push_back((double)id); });
  put_obstacles(b + 32, s, [](Obstacle &o, std::vector<double> &v, size_t) { v.insert(v.end(), &o.chi[0][0], &o.chi[0][0] + 64); });
  put_obstacles(b + 33, s, [](Obstacle &o, std::vector<double> &v, size_t) { v.insert(v.end(), &o.udef[0][0][0], &o.udef[0][0][0] + 128); });
  put_obstacles(b + 34, s, [](Obstacle &o, std::vector<double> &v, size_t) {
    for (size_t q = 0; q < o.n_surfPoints; q++)
      v.insert(v.end(), {o.x_s[q], o.y_s[q], o.p_s[q], o.u_s[q], o.v_s[q], o.nx_s[q], o.ny_s[q], o.omega_s[q], o.uDef_s[q],
                         o.vDef_s[q], o.fX_s[q], o.fY_s[q], o.fXv_s[q], o.fYv_s[q]});
  });
  put_obstacles(b + 35, s, [](Obstacle &o, std::vector<double> &v, size_t) { // in the order of quantities[19] (7233-7251)
    v.insert(v.end(), {o.circulation, o.perimeter, o.forcex, o.forcex_P, o.forcex_V, o.torque_P, o.drag, o.lift, o.Pout,
                       o.PoutNew, o.PoutBnd, o.torque, o.forcey, o.forcey_P, o.forcey_V, o.torque_V, o.thrust, o.defPowerBnd,
                       o.defPower});
  });
  put(b + 36, std::vector<double>(buf, buf + 19));
}

void on_derived(int k) {
  Shape *s = sim.shapes[k];
  put(100.0 * k + 37, {s->Pthrust, s->Pdrag, s->EffPDef, s->EffPDefBnd});
}
} // namespace

void cup2d_ref_hook(int op, void *buf, int count) {
  if (!g_armed) return;
  const int ns = (int)sim.shapes.size();
  if (g_derived >= 0) { // the loop body after the sum of shape g_derived has run
    on_derived(g_derived);
    const bool last = g_derived == ns - 1;
    g_derived = -1;
    if (last && sim.step >= g_first + g_count) {
      fclose(g_fout);
      exit(0);
    }
  }
  if (op == MPI_SUM && count == 3) {
    if (g_n3++ % ns == 0 && recording()) on_normals();
  } else if (op == MPI_SUM && count == 19) {
    const int k = g_n19++ % ns;
    if (recording()) {
      on_forces(k, (const double *)buf);
      g_derived = k;
    }
  }
}

extern int cup2d_ref_force_iters;

int main(int argc, char **argv) {
  if (argc != 5) {
    fprintf(stderr, "usage: ref_forces levelMax first count out.bin\n");
    return 2;
  }
  g_first = atoi(argv[2]);
  g_count = atoi(argv[3]);
  g_fout = fopen(argv[4], "wb");
  cup2d_ref_force_iters = 5;
  // run.sh:1-22 verbatim except levelMax (argument) and tdump 0 (no output files)
  const char *args[] = {"ref_main", "-AdaptSteps", "20", "-bpdx", "2", "-bpdy", "1", "-CFL", "0.5", "-Ctol", "1",
                        "-extent", "4", "-lambda", "1e7", "-levelMax", argv[1], "-levelStart", "5",
                        "-maxPoissonIterations", "1000", "-maxPoissonRestarts", "0", "-nu", "0.00004",
                        "-poissonTol", "1e-3", "-poissonTolRel", "1e-2", "-Rtol", "2", "-tdump", "0", "-tend", "10.0",
                        "-shapes", "angle=0 L=0.2 xpos=1.8 ypos=0.8\n angle=180 L=0.2 xpos=1.6 ypos=0.8"};
  return ref_main(sizeof args / sizeof *args, (char **)args);
}
