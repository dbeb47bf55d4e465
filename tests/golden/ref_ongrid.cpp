// TEST INFRASTRUCTURE — generator of tests/golden/amrongrid_*.npz (tests/golden/make_ongrid_golden.py), never shipped.
//
// Includes the UNMODIFIED reference translation unit (/root/reference/main.cpp, only `main` renamed) and runs its run.sh case.
// ongrid() (main.cpp:3991-4630) is observed through the MPI_Allreduce hook of oracle/shim/mpi.h, with no source patch:
//   MPI_MIN, count 1, while some shape's obstacleBlocks is empty (main.cpp:4215; shape k is the first shape with an empty
//   list, cleared at 4028 and refilled at 4245 — the dt reduction of 6583 sees every list filled): the midline of shape k as
//   ongrid() holds it at 4208, its center, orientation and centerOfMass;
//   the next nshapes MPI_SUM of count 3 (4483): the chi and tmp fields (first shape), then per shape the obstacle blocks (ids,
//   dist, chi, udef before the correction) and the per-block Mass / COM_x / COM_y;
//   the next nshapes MPI_SUM of count 7 (4520): the seven sums;
//   the first hook after that (end of ongrid): per shape the corrected udef, centerOfMass, M and J.
//
//   ref_ongrid levelMax first count out.bin       records ongrid calls first .. first+count-1 (0 = the first of the setup)
//   record stream [tag, n, n doubles]; every call starts with tag 1 = {call index, nshapes, h0, extent x, extent y, bpdx, bpdy}
//     2: mesh (level, i, j)                       per shape k (tag + 100 k):
//     3: chi field   4: tmp field                   10: {Nm, center x, y, orientation, centerOfMass x, y}
//                                                   11..19: rX rY norX norY vX vY vNorX vNorY width
//                                                   20: obstacle ids   21: dist   22: chi   23: udef (pre)   24: Mass/COM per block
//                                                   25: com[3]   26: the seven sums   27: udef (corrected)
//                                                   28: {centerOfMass x, y after 4485-4486, M, J}
#define CUP2D_REF_HOOK_TU 1
#define main ref_main
#include "main.cpp" // resolved with -I/root/reference
#undef main

namespace {
int g_first = 0, g_count = 0, g_call = -1;
int g_nsum3 = 0, g_nsum7 = 0;
bool g_in = false, g_rec = false;
FILE *g_fout = nullptr;

void put(double tag, const std::vector<double> &v) {
  const double hdr[2] = {tag, (double)v.size()};
  fwrite(hdr, sizeof(double), 2, g_fout);
  fwrite(v.data(), sizeof(double), v.size(), g_fout);
}
void put_blocks(double tag, Grid *g) {
  std::vector<double> v;
  for (auto &info : g->infos) v.insert(v.end(), info.block, info.block + _BS_ * _BS_);
  put(tag, v);
}
template <class F> void put_obstacles(double tag, Shape *s, F f) {
  std::vector<double> v;
  for (size_t id = 0; id < s->obstacleBlocks.size(); id++)
    if (s->obstacleBlocks[id]) f(*s->obstacleBlocks[id], v, id);
  put(tag, v);
}
int first_empty() {
  for (size_t k = 0; k < sim.shapes.size(); k++)
    if (sim.shapes[k]->obstacleBlocks.empty()) return (int)k;
  return -1;
}

void on_min() {
  const int k = first_empty();
  if (k < 0) return; // the dt reduction of the time loop
  if (k == 0) {
    g_call++;
    g_in = true;
    g_nsum3 = g_nsum7 = 0;
    g_rec = g_call >= g_first && g_call < g_first + g_count;
    if (g_rec) {
      put(1, {(double)g_call, (double)sim.shapes.size(), sim.h0, sim.extents[0], sim.extents[1], (double)sim.bpdx, (double)sim.bpdy});
      std::vector<double> mesh;
      for (auto &info : var.tmp->infos) { mesh.push_back(info.level); mesh.push_back(info.index[0]); mesh.push_back(info.index[1]); }
      put(2, mesh);
    }
  }
  if (!g_rec) return;
  Shape *s = sim.shapes[k];
  const double b = 100.0 * k;
  put(b + 10, {(double)s->Nm, s->center[0], s->center[1], s->orientation, s->centerOfMass[0], s->centerOfMass[1]});
  Real *arr[9] = {s->rX, s->rY, s->norX, s->norY, s->vX, s->vY, s->vNorX, s->vNorY, s->width};
  for (int q = 0; q < 9; q++) put(b + 11 + q, std::vector<double>(arr[q], arr[q] + s->Nm));
}

void on_sum3(double *com) {
  const int k = g_nsum3++;
  if (!g_rec) return;
  if (k == 0) {
    put_blocks(3, var.chi);
    put_blocks(4, var.tmp);
  }
  Shape *s = sim.shapes[k];
  const double b = 100.0 * k;
  put_obstacles(b + 20, s, [](Obstacle &, std::vector<double> &v, size_t id) { v.push_back((double)id); });
  put_obstacles(b + 21, s, [](Obstacle &o, std::vector<double> &v, size_t) { v.insert(v.end(), &o.dist[0][0], &o.dist[0][0] + 64); });
  put_obstacles(b + 22, s, [](Obstacle &o, std::vector<double> &v, size_t) { v.insert(v.end(), &o.chi[0][0], &o.chi[0][0] + 64); });
  put_obstacles(b + 23, s, [](Obstacle &o, std::vector<double> &v, size_t) { v.insert(v.end(), &o.udef[0][0][0], &o.udef[0][0][0] + 128); });
  put_obstacles(b + 24, s, [](Obstacle &o, std::vector<double> &v, size_t) { v.push_back(o.Mass); v.push_back(o.COM_x); v.push_back(o.COM_y); });
  put(b + 25, {com[0], com[1], com[2]});
}

void on_sum7(double *q) {
  const int k = g_nsum7++;
  if (g_rec) put(100.0 * k + 26, std::vector<double>(q, q + 7));
}

void on_end() {
  g_in = false;
  if (!g_rec) return;
  for (size_t k = 0; k < sim.shapes.size(); k++) {
    Shape *s = sim.shapes[k];
    put_obstacles(100.0 * k + 27, s, [](Obstacle &o, std::vector<double> &v, size_t) { v.insert(v.end(), &o.udef[0][0][0], &o.udef[0][0][0] + 128); });
    put(100.0 * k + 28, {s->centerOfMass[0], s->centerOfMass[1], s->M, s->J});
  }
  if (g_call + 1 >= g_first + g_count) {
    fclose(g_fout);
    exit(0);
  }
}
} // namespace

void cup2d_ref_hook(int op, void *buf, int count) {
  const int ns = (int)sim.shapes.size();
  if (g_in && g_nsum7 == ns) { on_end(); }
  if (op == MPI_MIN && count == 1) on_min();
  else if (g_in && op == MPI_SUM && count == 3 && g_nsum3 < ns) on_sum3((double *)buf);
  else if (g_in && op == MPI_SUM && count == 7 && g_nsum3 == ns && g_nsum7 < ns) on_sum7((double *)buf);
}

extern int cup2d_ref_force_iters;

int main(int argc, char **argv) {
  if (argc != 5) {
    fprintf(stderr, "usage: ref_ongrid levelMax first count out.bin\n");
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
