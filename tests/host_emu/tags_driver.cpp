// TEST INFRASTRUCTURE — adapt()'s tagging on fast and distributed contexts builds none of the full per-cell tables
// (tests/test_amr_tags_fast_emulation.py; with CUP2D_TEST_SANITIZERS=1 also under ThreadSanitizer / AddressSanitizer).
// Linked against the emulated product sources; it reads the context's internals through the product's own headers.  A
// two-level mesh (a level-2 unit square with one block refined): a baseline context builds the kind-1 and kind-3 tables
// when it tags (the check below can see them); a fast context and a one-rank distributed context tag, adapt and tag again
// on the new mesh without them.
#include "sim.h"
#include "amr.h"
#include <cmath>
#include <cstdio>
#include <vector>

#define CHECK(x)                                                                                  \
  do {                                                                                            \
    int _rc = (x);                                                                                \
    if (_rc) {                                                                                    \
      fprintf(stderr, "%s -> %d: %s\n", #x, _rc, cup2d_last_error());                             \
      return 1;                                                                                   \
    }                                                                                             \
  } while (0)

static bool full_tables(const cup2d_amr *a) {
  return a->csr[1].rowptr || a->csr[3].rowptr || a->lab[1] || a->lab[3];
}

static int tag_adapt_tag(cup2d_amr *a, const char *what) {
  const int64_t n = a->nb;
  std::vector<double> f2(n * 128), f1(n * 64), linf(n);
  for (size_t i = 0; i < f2.size(); i++) f2[i] = std::sin(0.29 * i) * 0.7;
  for (size_t i = 0; i < f1.size(); i++) f1[i] = i % 97 == 0 ? 0.8 : 0.0; // chi: a few positive cells
  CHECK(cup2d_amr_field_upload(a, CUP2D_VEL, f2.data()));
  CHECK(cup2d_amr_field_upload(a, CUP2D_CHI, f1.data()));
  CHECK(cup2d_amr_adapt_tags(a, 20.0, 4, linf.data()));
  int32_t changed = 0;
  int64_t nn = 0;
  CHECK(cup2d_amr_adapt(a, nullptr, 20.0, 1.0, 4, &nn, &changed));
  if (!changed) return 5;
  linf.resize(a->nb);
  CHECK(cup2d_amr_adapt_tags(a, 20.0, 4, linf.data()));
  for (double v : linf)
    if (!std::isfinite(v)) return 4;
  if (full_tables(a)) {
    fprintf(stderr, "%s: full tables built\n", what);
    return 6;
  }
  printf("%s: %lld -> %lld blocks, no full tables\n", what, (long long)n, (long long)nn);
  return 0;
}

int main() {
  const int L = 2, n = 16;
  std::vector<int32_t> ij(2 * n), lij;
  CHECK(cup2d_block_order(1, 1, L, ij.data()));
  for (int k = 0; k < n; k++) {
    const int i = ij[2 * k], j = ij[2 * k + 1];
    if (i == 1 && j == 1)
      for (int c = 0; c < 4; c++) lij.insert(lij.end(), {L + 1, 2 + (c & 1), 2 + (c >> 1)});
    else
      lij.insert(lij.end(), {L, i, j});
  }
  const int64_t nb = (int64_t)lij.size() / 3;
  { // the baseline builds them: the check can see them
    cup2d_amr *a = nullptr;
    CHECK(cup2d_amr_create(nb, lij.data(), 1, 1, 1.0 / 32, 1e-3, 0, &a));
    std::vector<double> z(nb * 128, 0.0), linf(nb);
    CHECK(cup2d_amr_field_upload(a, CUP2D_VEL, z.data()));
    CHECK(cup2d_amr_field_upload(a, CUP2D_CHI, z.data()));
    CHECK(cup2d_amr_adapt_tags(a, 1.0, 4, linf.data()));
    if (!a->csr[1].rowptr || !a->csr[3].rowptr) return 7;
    cup2d_amr_destroy(a);
  }
  { // fast
    cup2d_amr *a = nullptr;
    CHECK(cup2d_amr_create(nb, lij.data(), 1, 1, 1.0 / 32, 1e-3, 0, &a));
    CHECK(cup2d_amr_set_fast(a, 1));
    const int rc = tag_adapt_tag(a, "fast");
    cup2d_amr_destroy(a);
    if (rc) return rc;
  }
  { // distributed, one rank
    cup2d_amr *a = nullptr;
    const int64_t rb[2] = {0, nb};
    CHECK(cup2d_amr_create_ranks(nb, lij.data(), 1, 1, 1.0 / 32, 1e-3, 0, 1, rb, 0, &a));
    std::vector<unsigned char> blob(cup2d_peer_blob_size());
    CHECK(cup2d_amr_peer_export(a, blob.data()));
    CHECK(cup2d_amr_peer_attach(a, blob.data()));
    const int rc = tag_adapt_tag(a, "distributed");
    cup2d_amr_destroy(a);
    if (rc) return rc;
  }
  return 0;
}
