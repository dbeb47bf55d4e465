// TEST INFRASTRUCTURE (oracle) — not part of the product path.
//
// Step recorder for the reference's multi-level fish loop, around the UNMODIFIED reference translation unit (only `main` is
// renamed by a macro) or one of the drop-in forms spliced from it (oracle/amrdevice.mk).  Like ref_harness.cpp it takes
// control through the MPI_Allreduce hook of oracle/shim/mpi.h; it records, it never seeds.
//
//   ref_afish afish levelMax nsteps kiter out.bin
//        the reference's run.sh case (2 fish, regridding; shapes from CUP2D_REF_SHAPES if set, dump interval from
//        CUP2D_REF_TDUMP, default 0), recorded at the dt reduction of every step (main.cpp:6592), steps 0 .. nsteps-1:
//        double header {dt, nblocks, nshapes, field bytes the drop-in glue moved since the first dt reduction (0 without the
//        glue), wall seconds since then, sim.time}, (level,i,j) as doubles, vel blocks (128 per block), pres blocks (64),
//        then per shape 33 doubles: centerOfMass[2], orientation, u, v, omega, M, J, the 19 force quantities of
//        main.cpp:7254-7272 (of the step that just ended), u v omega at the collision reduction (main.cpp:6838, before the
//        pair loop) and after the pair loop (at main.cpp:7138; nothing changes them until the next step's 3x3 solve, so
//        where that reduction does not run, at the dt reduction).  kiter fixes the CPU solver's iteration count.
//        The device form (CUP2D_PATCHED_MAIN 5) reads vel and pres from the device, outside the glue's byte counter: its host
//        copies are stale.
#define CUP2D_REF_HOOK_TU 1
#define main ref_main
#if defined(CUP2D_PATCHED_MAIN) && CUP2D_PATCHED_MAIN == 5
#include "main_amrdevice.cpp" // oracle/_ref/: multi-level with every field on the device (oracle/amrdevice.mk)
#elif defined(CUP2D_PATCHED_MAIN) && CUP2D_PATCHED_MAIN == 4
#include "main_afish_amrresident.cpp" // oracle/_ref/: the multi-level device-resident form (oracle/amrdevice.mk)
#elif defined(CUP2D_PATCHED_MAIN)
#error "ref_afish: no recorder for this drop-in form"
#else
#include "main.cpp" // resolved with -I/root/reference
#endif
#undef main
#include <chrono>

extern int cup2d_ref_force_iters;

namespace {
int g_nsteps = 0, g_calls = 0;
std::string g_out;
FILE *g_fout = nullptr;
std::vector<double> g_coll_before, g_coll_after;
unsigned long long g_bytes0 = 0;
double g_t0 = 0;

double now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
unsigned long long glue_field_bytes() {
#ifdef CUP2D_PATCHED_MAIN
  return b200::field_bytes;
#else
  return 0;
#endif
}
} // namespace

void cup2d_ref_hook(int op, void *buf, int count) {
  (void)buf;
  const size_t S = sim.shapes.size();
  if (op == MPI_SUM && count == (int)(20 * S)) { // main.cpp:6838
    g_coll_before.clear();
    for (auto &sh : sim.shapes) g_coll_before.insert(g_coll_before.end(), {sh->u, sh->v, sh->omega});
    g_coll_after.clear();
    return;
  }
  if (op == MPI_SUM && count == 2 && !g_coll_before.empty() && g_coll_after.empty()) { // main.cpp:7138
    for (auto &sh : sim.shapes) g_coll_after.insert(g_coll_after.end(), {sh->u, sh->v, sh->omega});
    return;
  }
  if (op != MPI_MAX || count != 1) return;
  const int call = g_calls++;
  if (call == 0) {
    g_fout = fopen(g_out.c_str(), "wb");
    if (!g_fout) {
      fprintf(stderr, "ref_afish: cannot write %s\n", g_out.c_str());
      exit(2);
    }
    g_bytes0 = glue_field_bytes();
    g_t0 = now();
    return;
  }
  if (g_coll_after.empty())
    for (auto &sh : sim.shapes) g_coll_after.insert(g_coll_after.end(), {sh->u, sh->v, sh->omega});
  const size_t nb = var.vel->infos.size();
  std::vector<double> r = {sim.dt, (double)nb, (double)S, (double)(glue_field_bytes() - g_bytes0), now() - g_t0, sim.time};
  for (auto &info : var.vel->infos) r.insert(r.end(), {(double)info.level, (double)info.index[0], (double)info.index[1]});
  std::vector<double> vel(nb * 2 * _BS_ * _BS_), pres(nb * _BS_ * _BS_);
#if defined(CUP2D_PATCHED_MAIN) && CUP2D_PATCHED_MAIN == 5
  b200::check(cup2d_amr_field_download(b200::amr, CUP2D_VEL, vel.data()), "cup2d_amr_field_download");
  b200::check(cup2d_amr_field_download(b200::amr, CUP2D_PRES, pres.data()), "cup2d_amr_field_download");
#else
  for (size_t i = 0; i < nb; i++) {
    memcpy(&vel[i * 2 * _BS_ * _BS_], var.vel->infos[i].block, 2 * _BS_ * _BS_ * sizeof(double));
    memcpy(&pres[i * _BS_ * _BS_], var.pres->infos[i].block, _BS_ * _BS_ * sizeof(double));
  }
#endif
  r.insert(r.end(), vel.begin(), vel.end());
  r.insert(r.end(), pres.begin(), pres.end());
  for (size_t k = 0; k < S; k++) {
    const auto &sh = sim.shapes[k];
    r.insert(r.end(), {sh->centerOfMass[0], sh->centerOfMass[1], sh->orientation, sh->u, sh->v, sh->omega, sh->M, sh->J,
                       sh->circulation, sh->perimeter, sh->forcex, sh->forcex_P, sh->forcex_V, sh->torque_P, sh->drag, sh->lift,
                       sh->Pout, sh->PoutNew, sh->PoutBnd, sh->torque, sh->forcey, sh->forcey_P, sh->forcey_V, sh->torque_V,
                       sh->thrust, sh->defPowerBnd, sh->defPower});
    for (int q = 0; q < 3; q++) r.push_back(g_coll_before.size() == 3 * S ? g_coll_before[3 * k + q] : 0.0);
    for (int q = 0; q < 3; q++) r.push_back(g_coll_after[3 * k + q]);
  }
  fwrite(r.data(), sizeof(double), r.size(), g_fout);
  g_coll_before.clear();
  g_coll_after.clear();
  if (call == g_nsteps) {
    fclose(g_fout);
    exit(0);
  }
}

int main(int argc, char **argv) {
  if (argc != 6 || std::string(argv[1]) != "afish") {
    fprintf(stderr, "usage: ref_afish afish levelMax nsteps kiter out.bin\n");
    return 2;
  }
  g_nsteps = atoi(argv[3]);
  cup2d_ref_force_iters = atoi(argv[4]);
  g_out = argv[5];
  // run.sh:1-22 verbatim except levelMax (argument), tdump and shapes (environment)
  const char *args[] = {"ref_main", "-AdaptSteps", "20", "-bpdx", "2", "-bpdy", "1", "-CFL", "0.5", "-Ctol", "1",
                        "-extent", "4", "-lambda", "1e7", "-levelMax", argv[2], "-levelStart", "5",
                        "-maxPoissonIterations", "1000", "-maxPoissonRestarts", "0", "-nu", "0.00004",
                        "-poissonTol", "1e-3", "-poissonTolRel", "1e-2", "-Rtol", "2",
                        "-tdump", getenv("CUP2D_REF_TDUMP") ? getenv("CUP2D_REF_TDUMP") : "0", "-tend", "10.0",
                        "-shapes", getenv("CUP2D_REF_SHAPES") ? getenv("CUP2D_REF_SHAPES")
                                                              : "angle=0 L=0.2 xpos=1.8 ypos=0.8\n angle=180 L=0.2 xpos=1.6 ypos=0.8"};
  return ref_main(sizeof args / sizeof *args, (char **)args);
}
