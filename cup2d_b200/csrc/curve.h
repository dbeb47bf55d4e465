// The order of a new block list after adapt(): fill_pos sorts the blocks by Encode (main.cpp:1550-1553, 422-445) over the
// space-filling curve of SpaceCurve (main.cpp:342-421, 6342-6376).  One implementation for the host decision
// (cup2d_amr_adapt_mesh, csrc/amr_plan.cpp, compiled by g++) and the device decision (cup2d_amr_adapt, csrc/amr_regrid.cu):
// the functions are __host__ __device__ under nvcc and plain functions elsewhere.  A Curve holds pointers to its zsave / inv
// tables (CurveTables builds them on the host; the device decision uploads a copy per call).
#pragma once
#include <algorithm>
#include <cstdint>
#include <vector>

#if defined(__CUDACC__)
#define CUP2D_HD __host__ __device__
#else
#define CUP2D_HD
#endif

namespace cup2d {

struct Curve { // SpaceCurve::forward / inverse / Encode
  int bpdx, bpdy, lmax, base;
  bool regular;
  const int64_t *zsave; // [j * bpdx + i]
  const int32_t *inv;   // [2 * zsave value]: (i, j)
  static CUP2D_HD int64_t xy2d(int b, int x, int y) {
    const int n = 1 << b;
    int64_t d = 0;
    for (int s = n / 2; s > 0; s /= 2) {
      const int rx = (x & s) > 0, ry = (y & s) > 0;
      d += (int64_t)s * s * ((3 * rx) ^ ry);
      if (ry == 0) {
        if (rx == 1) x = n - 1 - x, y = n - 1 - y;
        const int t = x;
        x = y, y = t;
      }
    }
    return d;
  }
  static CUP2D_HD void d2xy(int b, int64_t t, int &x, int &y) {
    const int n = 1 << b;
    x = y = 0;
    for (int64_t s = 1; s < n; s *= 2) {
      const int64_t rx = 1 & (t / 2), ry = 1 & (t ^ rx);
      if (ry == 0) {
        if (rx == 1) x = (int)s - 1 - x, y = (int)s - 1 - y;
        const int u = x;
        x = y, y = u;
      }
      x += (int)(s * rx), y += (int)(s * ry);
      t /= 4;
    }
  }
  CUP2D_HD int64_t forward(int l, int i, int j) const {
    if (l >= lmax) return 0;
    if (regular) return xy2d(l + base, i, j);
    const int aux = 1 << l, I = i / aux, J = j / aux;
    return xy2d(l, i - I * aux, j - J * aux) + zsave[(size_t)J * bpdx + I] * aux * aux;
  }
  CUP2D_HD void inverse(int64_t Z, int l, int &i, int &j) const {
    if (regular) return d2xy(l + base, Z, i, j);
    const int64_t aux = 1LL << l;
    d2xy(l, Z % (aux * aux), i, j);
    const int32_t *IJ = inv + 2 * (size_t)(Z / (aux * aux));
    i += IJ[0] * (int)aux, j += IJ[1] * (int)aux;
  }
  CUP2D_HD int64_t encode(int level, int i, int j) const {
    int64_t r = 0;
    for (int l = level, ix = i, iy = j; l >= 0; l--, ix /= 2, iy /= 2) r += forward(l, ix, iy);
    int ix = 2 * i, iy = 2 * j;
    for (int l = level + 1; l < lmax; l++) {
      int64_t Zc = forward(l, ix, iy);
      Zc -= Zc % 4;
      r += Zc;
      int ix1, iy1;
      inverse(Zc, l, ix1, iy1);
      ix = 2 * ix1, iy = 2 * iy1;
    }
    return r + level;
  }
};

// the curve's tables of a bpdx x bpdy domain (SpaceCurve's constructor); regular = false for rectangular and
// non-power-of-two domains, whose curve skips the positions outside the domain
struct CurveTables {
  int bpdx, bpdy, base = 0;
  bool regular = true;
  std::vector<int64_t> zsave;
  std::vector<int32_t> inv;
  CurveTables(int bx, int by) : bpdx(bx), bpdy(by), zsave((size_t)bx * by), inv(2 * (size_t)bx * by) {
    while ((1 << base) < std::max(bx, by)) base++;
    for (int j = 0; j < by; j++)
      for (int i = 0; i < bx; i++) {
        int64_t index = Curve::xy2d(base, i, j), sub = 0;
        for (int64_t h = 0; h < index; h++) {
          int x, y;
          Curve::d2xy(base, h, x, y);
          sub += x >= bx || y >= by;
        }
        if (sub) regular = false;
        zsave[(size_t)j * bx + i] = index - sub;
        inv[2 * (index - sub)] = i, inv[2 * (index - sub) + 1] = j;
      }
  }
  // the curve over these tables (host) or over copies of them at zs / iv (device)
  Curve curve(int lmax, const int64_t *zs = nullptr, const int32_t *iv = nullptr) const {
    return Curve{bpdx, bpdy, lmax, base, regular, zs ? zs : zsave.data(), iv ? iv : inv.data()};
  }
};

} // namespace cup2d
