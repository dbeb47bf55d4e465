// TEST INFRASTRUCTURE — generator of tests/golden/amrregrid_*.npz (tests/golden/make_regrid_golden.py), never shipped.
//
// Includes the UNMODIFIED reference translation unit (/root/reference/main.cpp, only `main` renamed), runs its run.sh case
// for nsteps steps and then, at the dt reduction of the next step (main.cpp:6592, through the hook of oracle/shim/mpi.h),
// records the reference's own adapt() (main.cpp:4657-5260) on that state:
//
//   ref_aregrid levelMax nsteps rq cq out.bin
//     vel and pres seeded (smooth part + per-cell noise), vold = vel, pold = pres, chi stays the fishes'; Rtol / Ctol midway
//     between the two per-block L-inf values of adapt()'s tagging field around the quantiles rq / cq; then adapt().
//     record stream [tag, n, n doubles]:
//     10: Rtol, Ctol, levelMax, h0, bpdx, bpdy   11: mesh (level, i, j)   12: vel   16: vold   13: pres   17: pold   14: chi
//     18: tmp (the tagging field)   42: per-block L-inf of tmp
//     24: VectorLab of vel, stencil {-1,-1,2,2,tensorial} (10*10*2/block)   25: ScalarLab of pres, same stencil (10*10/block)
//     after adapt(): 50: new mesh (infos order)   51: vel   52: vold   53: pres   54: pold   55: chi   56: tmp
#define CUP2D_REF_HOOK_TU 1
#define main ref_main
#include "main.cpp" // resolved with -I/root/reference
#undef main

namespace {
int g_calls = 0, g_nsteps = 0;
double g_rq = 0, g_cq = 0;
std::string g_out;
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
void put_mesh(double tag, Grid *g) {
  std::vector<double> mesh;
  for (auto &info : g->infos) { mesh.push_back(info.level); mesh.push_back(info.index[0]); mesh.push_back(info.index[1]); }
  put(tag, mesh);
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
double seeded(int level, int i, int j, int ix, int iy, int comp, double x, double y) {
  // smooth part + a deterministic per-cell perturbation (so that an indexing error cannot hide behind smoothness)
  unsigned long long k = (((((unsigned long long)level * 4099 + i) * 4099 + j) * 67 + ix) * 67 + iy) * 7 + comp;
  k ^= k >> 33; k *= 0xff51afd7ed558ccdULL; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ULL; k ^= k >> 33;
  const double noise = (double)(k >> 11) / 9007199254740992.0 - 0.5;
  const double s = comp == 0 ? sin(1.3 * x + 0.4) * cos(2.1 * y) : comp == 1 ? cos(0.9 * x) * sin(1.7 * y + 0.2)
                 : comp == 2 ? cos(1.1 * x - 0.3) * cos(0.8 * y) : comp == 3 ? 0.5 + 0.5 * sin(2.0 * x) * sin(1.5 * y)
                 : comp == 4 ? 0.3 * sin(3 * x + y) : 0.2 * cos(2 * y - x);
  return s + 0.05 * noise;
}
void seed_grid(Grid *g, int dim, int comp0) {
  for (auto &info : g->infos)
    for (int iy = 0; iy < _BS_; iy++)
      for (int ix = 0; ix < _BS_; ix++)
        for (int c = 0; c < dim; c++)
          info.block[dim * (_BS_ * iy + ix) + c] =
              seeded(info.level, info.index[0], info.index[1], ix, iy, comp0 + c, info.origin[0] + info.h * (ix + 0.5),
                     info.origin[1] + info.h * (iy + 0.5));
}
std::vector<double> block_linf(Grid *g) {
  std::vector<double> v;
  for (auto &info : g->infos) {
    double m = 0.0;
    for (int j = 0; j < _BS_ * _BS_; j++) m = std::max(m, std::fabs(info.block[j]));
    v.push_back(m);
  }
  return v;
}
double threshold(std::vector<double> v, double q) { // midway between two neighbouring values: no block sits at a threshold
  std::sort(v.begin(), v.end());
  const size_t k = std::min(v.size() - 2, (size_t)(q * (double)v.size()));
  return 0.5 * (v[k] + v[k + 1]);
}

void do_aregrid() {
  g_fout = fopen(g_out.c_str(), "wb");
  seed_grid(var.vel, 2, 0);
  seed_grid(var.vold, 2, 0); // vold = vel and pold = pres: the fixture then stores each once
  seed_grid(var.pres, 1, 2);
  seed_grid(var.pold, 1, 2);
  // the tagging field adapt() computes first (main.cpp:4659-4660); its per-block L-inf depends on Rtol only on the blocks of
  // the chi rule (2 Rtol, above Rtol whatever it is), so the thresholds can be taken before Rtol is set
  computeA<VectorLab>(KernelVorticity(), var.vel, 2);
  computeA<ScalarLab>(GradChiOnTmp(), var.chi, 1);
  const std::vector<double> linf0 = block_linf(var.tmp);
  sim.Rtol = threshold(linf0, g_rq);
  sim.Ctol = threshold(linf0, g_cq);
  computeA<VectorLab>(KernelVorticity(), var.vel, 2);
  computeA<ScalarLab>(GradChiOnTmp(), var.chi, 1);
  put(10, {sim.Rtol, sim.Ctol, (double)sim.levelMax, sim.h0, (double)sim.bpdx, (double)sim.bpdy});
  put_mesh(11, var.vel);
  put_blocks(12, var.vel, 2);
  put_blocks(16, var.vold, 2);
  put_blocks(13, var.pres, 1);
  put_blocks(17, var.pold, 1);
  put_blocks(14, var.chi, 1);
  put_blocks(18, var.tmp, 1);
  put(42, block_linf(var.tmp));
  const size_t nb = var.vel->infos.size();
  {
    std::vector<double> lab(nb * 10 * 10 * 2);
    computeA<VectorLab>(DumpLab<VectorLab, 2>(Stencil{-1, -1, 2, 2, true}, &lab), var.vel, 2);
    put(24, lab);
  }
  {
    std::vector<double> lab(nb * 10 * 10);
    computeA<ScalarLab>(DumpLab<ScalarLab, 1>(Stencil{-1, -1, 2, 2, true}, &lab), var.pres, 1);
    put(25, lab);
  }
  adapt();
  put_mesh(50, var.vel);
  put_blocks(51, var.vel, 2);
  put_blocks(52, var.vold, 2);
  put_blocks(53, var.pres, 1);
  put_blocks(54, var.pold, 1);
  put_blocks(55, var.chi, 1);
  put_blocks(56, var.tmp, 1);
  fclose(g_fout);
}
} // namespace

void cup2d_ref_hook(int op, void *, int count) {
  if (op != MPI_MAX || count != 1) return;
  if (g_calls++ < g_nsteps) return; // let the reference run nsteps steps first
  do_aregrid();
  exit(0);
}

extern int cup2d_ref_force_iters;

int main(int argc, char **argv) {
  if (argc != 6) {
    fprintf(stderr, "usage: ref_aregrid levelMax nsteps rq cq out.bin\n");
    return 2;
  }
  g_nsteps = atoi(argv[2]);
  g_rq = atof(argv[3]);
  g_cq = atof(argv[4]);
  g_out = argv[5];
  cup2d_ref_force_iters = 5;
  // run.sh:1-22 verbatim except levelMax (argument) and tdump 0 (no output files)
  const char *args[] = {"ref_main", "-AdaptSteps", "20", "-bpdx", "2", "-bpdy", "1", "-CFL", "0.5", "-Ctol", "1",
                        "-extent", "4", "-lambda", "1e7", "-levelMax", argv[1], "-levelStart", "5",
                        "-maxPoissonIterations", "1000", "-maxPoissonRestarts", "0", "-nu", "0.00004",
                        "-poissonTol", "1e-3", "-poissonTolRel", "1e-2", "-Rtol", "2", "-tdump", "0", "-tend", "10.0",
                        "-shapes", "angle=0 L=0.2 xpos=1.8 ypos=0.8\n angle=180 L=0.2 xpos=1.6 ypos=0.8"};
  return ref_main(sizeof args / sizeof *args, (char **)args);
}
