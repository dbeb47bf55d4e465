// TEST INFRASTRUCTURE — sanitizer run of a regrid (tests/test_amr_regrid.py, CUP2D_TEST_SANITIZERS=1).  Linked against the
// emulated product sources built with -fsanitize=thread or -fsanitize=address,alignment,bounds (every CUDA thread an OS
// thread, every device buffer its own exact-size allocation filled with 0xFF bytes).  A uniform level-2 mesh of 16 blocks
// takes a step (so that the old mesh's tables, lab buffers and Poisson context exist), is regridded with one block refined
// and one sibling group compressed, and takes a step on the new mesh with the baseline and the fast kernels.
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

int main() {
  const int L = 2, n = 16;
  std::vector<int32_t> ij(2 * n), lij;
  CHECK(cup2d_block_order(1, 1, L, ij.data()));
  for (int k = 0; k < n; k++) lij.insert(lij.end(), {L, ij[2 * k], ij[2 * k + 1]});
  cup2d_amr *a = nullptr;
  CHECK(cup2d_amr_create(n, lij.data(), 1, 1, 1.0 / 32, 1e-3, 0, &a));
  std::vector<double> f2(n * 128), f1(n * 64);
  for (size_t i = 0; i < f2.size(); i++) f2[i] = std::sin(0.29 * i) * 0.7;
  for (size_t i = 0; i < f1.size(); i++) f1[i] = std::cos(0.13 * i);
  for (int fld : {CUP2D_VEL, CUP2D_VOLD, CUP2D_TMPV}) CHECK(cup2d_amr_field_upload(a, fld, f2.data()));
  for (int fld : {CUP2D_PRES, CUP2D_POLD, CUP2D_CHI, CUP2D_TMP}) CHECK(cup2d_amr_field_upload(a, fld, f1.data()));
  double dt, err;
  int it;
  CHECK(cup2d_amr_step(a, 0.5, 0.0, 0.0, 0.0, 0, 3, &dt, &it, &err));
  // (2, 0, 0) refined, the group (2, 2..3, 2..3) compressed into (1, 1, 1)
  std::vector<int32_t> nl;
  for (int k = 0; k < n; k++) {
    const int i = lij[3 * k + 1], j = lij[3 * k + 2];
    if (i == 0 && j == 0)
      for (int c = 0; c < 4; c++) nl.insert(nl.end(), {L + 1, c & 1, c >> 1});
    else if (i >= 2 && j >= 2) {
      if (i == 2 && j == 2) nl.insert(nl.end(), {L - 1, 1, 1});
    } else
      nl.insert(nl.end(), {L, i, j});
  }
  const int64_t nn = (int64_t)nl.size() / 3;
  CHECK(cup2d_amr_regrid(a, nn, nl.data()));
  std::vector<double> v(nn * 128), t(nn * 128);
  CHECK(cup2d_amr_field_download(a, CUP2D_VEL, v.data()));
  CHECK(cup2d_amr_field_download(a, CUP2D_TMPV, t.data()));
  for (size_t i = 0; i < v.size(); i++)
    if (!std::isfinite(v[i]) || t[i] != 0.0) return 4;
  for (int fast = 0; fast < 2; fast++) {
    CHECK(cup2d_amr_set_fast(a, fast));
    CHECK(cup2d_amr_step(a, 0.5, 0.0, 0.0, 0.0, 0, 3, &dt, &it, &err));
    if (!std::isfinite(dt) || !std::isfinite(err)) return 3;
    printf("regrid step (fast=%d): %lld -> %lld blocks dt %.3e iters %d err %.3e\n", fast, (long long)n, (long long)nn, dt, it, err);
  }
  cup2d_amr_destroy(a);
  return 0;
}
