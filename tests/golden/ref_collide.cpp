// TEST INFRASTRUCTURE — generator of tests/golden/amrcollide_*.npz (tests/golden/make_collide_golden.py), never shipped.
//
// Includes the UNMODIFIED reference translation unit (/root/reference/main.cpp, only `main` renamed) and runs its run.sh case
// with the shapes given on the command line.  The collision model (main.cpp:6705-6943) is observed through the MPI_Allreduce
// hook of oracle/shim/mpi.h, with no source patch:
//   MPI_SUM of count 20 N (6838): the mesh, per shape its obstacle blocks (ids, chi, dist, udef as they are at that point),
//   (u, v, omega) after the 3x3 solve, centerOfMass, M, J and length, and the all-reduced buffer;
//   the first hook after that (the pair loop of 6863-6943 has run): per shape (u, v, omega).
//
//   ref_collide levelMax count out.bin shapes      records the first `count` collision calls of the time loop
//   record stream [tag, n, n doubles]; every call starts with tag 1 = {call index, nshapes, h0, bpdx, bpdy}
//     2: mesh (level, i, j)                         per shape k (tag + 100 k):
//     30: the 20 N buffer                             10: {u, v, omega, centerOfMass x, y, M, J, length}
//     31: (u, v, omega) of every shape after          20: obstacle ids   21: chi   22: dist   23: udef
#define CUP2D_REF_HOOK_TU 1
#define main ref_main
#include "main.cpp" // resolved with -I/root/reference
#undef main

namespace {
int g_count = 0, g_call = 0;
bool g_after = false;
FILE *g_fout = nullptr;

void put(double tag, const std::vector<double> &v) {
  const double hdr[2] = {tag, (double)v.size()};
  fwrite(hdr, sizeof(double), 2, g_fout);
  fwrite(v.data(), sizeof(double), v.size(), g_fout);
}
template <class F> void put_obstacles(double tag, Shape *s, F f) {
  std::vector<double> v;
  for (size_t id = 0; id < s->obstacleBlocks.size(); id++)
    if (s->obstacleBlocks[id]) f(*s->obstacleBlocks[id], v, id);
  put(tag, v);
}

void on_sums(const double *buf, int count) {
  const size_t ns = sim.shapes.size();
  put(1, {(double)g_call, (double)ns, sim.h0, (double)sim.bpdx, (double)sim.bpdy});
  std::vector<double> mesh;
  for (auto &info : var.chi->infos) { mesh.push_back(info.level); mesh.push_back(info.index[0]); mesh.push_back(info.index[1]); }
  put(2, mesh);
  for (size_t k = 0; k < ns; k++) {
    Shape *s = sim.shapes[k];
    const double b = 100.0 * k;
    put(b + 10, {s->u, s->v, s->omega, s->centerOfMass[0], s->centerOfMass[1], s->M, s->J, s->length});
    put_obstacles(b + 20, s, [](Obstacle &, std::vector<double> &v, size_t id) { v.push_back((double)id); });
    put_obstacles(b + 21, s, [](Obstacle &o, std::vector<double> &v, size_t) { v.insert(v.end(), &o.chi[0][0], &o.chi[0][0] + 64); });
    put_obstacles(b + 22, s, [](Obstacle &o, std::vector<double> &v, size_t) { v.insert(v.end(), &o.dist[0][0], &o.dist[0][0] + 64); });
    put_obstacles(b + 23, s, [](Obstacle &o, std::vector<double> &v, size_t) { v.insert(v.end(), &o.udef[0][0][0], &o.udef[0][0][0] + 128); });
  }
  put(30, std::vector<double>(buf, buf + count));
  g_after = true;
}

void on_after() {
  g_after = false;
  std::vector<double> v;
  for (Shape *s : sim.shapes) v.insert(v.end(), {s->u, s->v, s->omega});
  put(31, v);
  if (++g_call >= g_count) {
    fclose(g_fout);
    exit(0);
  }
}
} // namespace

void cup2d_ref_hook(int op, void *buf, int count) {
  if (g_after) on_after();
  else if (op == MPI_SUM && count == 20 * (int)sim.shapes.size()) on_sums((const double *)buf, count);
}

extern int cup2d_ref_force_iters;

int main(int argc, char **argv) {
  if (argc != 5) {
    fprintf(stderr, "usage: ref_collide levelMax count out.bin shapes\n");
    return 2;
  }
  g_count = atoi(argv[2]);
  g_fout = fopen(argv[3], "wb");
  cup2d_ref_force_iters = 5;
  // run.sh:1-22 verbatim except levelMax (argument), tdump 0 (no output files) and the shapes (argument)
  const char *args[] = {"ref_main", "-AdaptSteps", "20", "-bpdx", "2", "-bpdy", "1", "-CFL", "0.5", "-Ctol", "1",
                        "-extent", "4", "-lambda", "1e7", "-levelMax", argv[1], "-levelStart", "5",
                        "-maxPoissonIterations", "1000", "-maxPoissonRestarts", "0", "-nu", "0.00004",
                        "-poissonTol", "1e-3", "-poissonTolRel", "1e-2", "-Rtol", "2", "-tdump", "0", "-tend", "10.0",
                        "-shapes", argv[4]};
  return ref_main(sizeof args / sizeof *args, (char **)args);
}
