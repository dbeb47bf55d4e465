// TEST INFRASTRUCTURE — sanitizer run of cup2d_amr_surface / _forces (tests/test_amr_forces.py, CUP2D_TEST_SANITIZERS=1).  Linked
// against the emulated product sources built with -fsanitize=thread or -fsanitize=address,alignment,bounds (every CUDA thread
// an OS thread, every device buffer its own exact-size allocation filled with 0xFF bytes).  A level-2 mesh of 16 blocks with
// one block refined (a level jump) carries two overlapping bent bodies placed by cup2d_amr_ongrid, with smooth vel and pres;
// the normals are taken once and the force diagnostics twice (the second call reuses the tables and scratch buffers), and
// the 23 numbers per shape and every point's normal and skin are checked to be finite.
#include "../../include/cup2d_b200.h"
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CHECK(x)                                                                                  \
  do {                                                                                            \
    int _rc = (x);                                                                                \
    if (_rc) {                                                                                    \
      fprintf(stderr, "%s -> %d: %s\n", #x, _rc, cup2d_last_error());                             \
      return 1;                                                                                   \
    }                                                                                             \
  } while (0)

struct Midline {
  std::vector<double> a[9]; // rX rY norX norY vX vY vNorX vNorY width
};

static Midline midline(int nm, double length, double bend) {
  Midline m;
  for (auto &v : m.a) v.resize(nm);
  for (int i = 0; i < nm; i++) {
    const double t = (double)i / (nm - 1), s = t * length;
    const double x = s - 0.5 * length, y = bend * length * std::sin(2 * M_PI * t) * t;
    const double dy = bend * length * (2 * M_PI / length * std::cos(2 * M_PI * t) * t + std::sin(2 * M_PI * t) / length);
    const double n = std::sqrt(1 + dy * dy);
    m.a[0][i] = x, m.a[1][i] = y, m.a[2][i] = -dy / n, m.a[3][i] = 1 / n;
    m.a[4][i] = -0.05 * std::cos(2 * M_PI * t), m.a[5][i] = 0.2 * std::sin(2 * M_PI * t) * t;
    m.a[6][i] = 0.1 * std::cos(3 * t), m.a[7][i] = -0.1 * std::sin(2 * t);
    m.a[8][i] = 0.08 * length * std::sqrt(t * (1 - t)) + 1e-3 * length;
  }
  return m;
}

int main() {
  const int L = 2, n = 16;
  std::vector<int32_t> ij(2 * n), lij;
  CHECK(cup2d_block_order(1, 1, L, ij.data()));
  for (int k = 0; k < n; k++) {
    const int i = ij[2 * k], j = ij[2 * k + 1];
    if (i == 1 && j == 1)
      for (int c = 0; c < 4; c++) lij.insert(lij.end(), {L + 1, 2 * i + (c & 1), 2 * j + (c >> 1)});
    else
      lij.insert(lij.end(), {L, i, j});
  }
  const int64_t nb = (int64_t)lij.size() / 3;
  cup2d_amr *a = nullptr;
  CHECK(cup2d_amr_create(nb, lij.data(), 1, 1, 1.0 / 32, 1e-3, 0, &a)); // domain [0, 0.25]^2
  const Midline m[2] = {midline(41, 0.12, 0.05), midline(33, 0.09, -0.08)};
  const double centre[2][2] = {{0.09, 0.095}, {0.1, 0.11}}, angle[2] = {0.4, 2.2};
  cup2d_body b[2];
  for (int s = 0; s < 2; s++) {
    b[s].nm = (int32_t)m[s].a[0].size(), b[s].reserved = 0;
    b[s].rX = m[s].a[0].data(), b[s].rY = m[s].a[1].data(), b[s].norX = m[s].a[2].data(), b[s].norY = m[s].a[3].data();
    b[s].vX = m[s].a[4].data(), b[s].vY = m[s].a[5].data(), b[s].vNorX = m[s].a[6].data(), b[s].vNorY = m[s].a[7].data();
    b[s].width = m[s].a[8].data();
    b[s].center[0] = centre[s][0], b[s].center[1] = centre[s][1], b[s].orientation = angle[s];
    b[s].center_of_mass[0] = centre[s][0] + 0.001, b[s].center_of_mass[1] = centre[s][1];
  }
  double out[20];
  CHECK(cup2d_amr_ongrid(a, 2, b, out));
  std::vector<double> vel((size_t)nb * 128), pres((size_t)nb * 64);
  for (int64_t k = 0; k < nb; k++) {
    const double h = 1.0 / 32 / (1 << lij[3 * k]);
    for (int c = 0; c < 64; c++) {
      const double x = (lij[3 * k + 1] * 8 + (c & 7) + 0.5) * h, y = (lij[3 * k + 2] * 8 + (c >> 3) + 0.5) * h;
      vel[(size_t)k * 128 + 2 * c] = std::sin(20 * x) * std::cos(17 * y), vel[(size_t)k * 128 + 2 * c + 1] = std::cos(13 * x) + y;
      pres[(size_t)k * 64 + c] = std::cos(19 * x - 0.2) * std::cos(11 * y);
    }
  }
  CHECK(cup2d_amr_field_upload(a, 0, vel.data()));
  CHECK(cup2d_amr_field_upload(a, 4, pres.data()));
  CHECK(cup2d_amr_surface(a, 2));
  cup2d_rigid r[2];
  for (int s = 0; s < 2; s++) {
    r[s].u = s ? -0.3 : 0.3, r[s].v = s ? 0.1 : -0.1, r[s].omega = 0;
    r[s].center_of_mass[0] = out[10 * s + 3], r[s].center_of_mass[1] = out[10 * s + 4];
    r[s].M = out[10 * s + 5], r[s].J = out[10 * s + 6], r[s].length = 0.12;
  }
  for (int rep = 0; rep < 2; rep++) {
    double f[46];
    CHECK(cup2d_amr_forces(a, 2, r, f));
    for (double v : f)
      if (!std::isfinite(v)) return 4;
    int64_t npts[2];
    for (int s = 0; s < 2; s++) {
      npts[s] = cup2d_amr_surface_get(a, s, nullptr, nullptr, nullptr, nullptr);
      if (npts[s] <= 0) return 5;
      std::vector<int32_t> blk(npts[s]), ixy(2 * npts[s]);
      std::vector<double> nrm(3 * npts[s]), skin(14 * npts[s]);
      if (cup2d_amr_surface_get(a, s, blk.data(), ixy.data(), nrm.data(), skin.data()) != npts[s]) return 6;
      for (double v : nrm)
        if (!std::isfinite(v)) return 7;
      for (double v : skin)
        if (!std::isfinite(v)) return 8;
    }
    printf("forces call %d: points %lld %lld, forcex %.6e %.6e, torque %.6e %.6e\n", rep, (long long)npts[0], (long long)npts[1], f[2],
           f[25], f[11], f[34]);
  }
  cup2d_amr_destroy(a);
  return 0;
}
