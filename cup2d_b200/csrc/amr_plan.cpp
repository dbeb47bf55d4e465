// Host-side plan builder for multi-level (block-AMR) meshes: ghost-cell stencil tables (SURVEY §8(f) rank 2).
//
// On a multi-level mesh every ghost cell of a block's lab is a fixed linear combination of cells owned by nearby
// blocks — a copy (same-level neighbour), a 2x2 average (finer neighbour), a wall reflection, or the reference's
// coarse->fine interpolation (2-D Taylor from the 3x3 coarse cells for the outer layer and corners, 1-D quadratic
// along the face plus the LI/LE closure across it for the two layers next to the block) — with weights that depend
// on the mesh only.  This file evaluates the reference's ghost assembly (BlockLab::load / post_load,
// main.cpp:2247-2933; FillCoarseVersion / UseCoarseStencil0, main.cpp:2935-2993; LI/LE/TestInterp, main.cpp:2203-2230;
// wall ghosts main.cpp:3131-3255) ONCE PER REGRID on symbolic values (sparse linear combinations of source cells
// instead of numbers) and emits the result as CSR tables.  The device applies a table with a gather (the tile loaders'
// irregular-ghost pass); nothing here touches the GPU.  Same operation order as the reference inside every ghost, so
// the table reproduces its values up to the rounding of a flat sum (pinned at 1e-13 against labs dumped from the
// unmodified reference, tests/test_amr_plan.py).  Three properties of the reference that shape its ghosts are kept:
// the row mix-up in the fine->coarse average across x faces (main.cpp:2529-2530) and the Taylor ghosts of a vector lab
// taking component 0 for every component (main.cpp:2751-2765); see DESIGN.md 7.1.
#include "../../include/cup2d_b200.h"
#include <algorithm>
#include <array>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <thread>
#include <vector>

namespace cup2d {
void set_error(const std::string &msg);
}

namespace {
constexpr int BS = CUP2D_BS, H = BS / 2;

// sparse linear combination of source values; key = ((block * 64 + cell) * dim + comp)
struct LC {
  std::vector<std::pair<int64_t, double>> t; // sorted by key
  bool set = false;
  static LC src(int64_t key) {
    LC r;
    r.t.push_back({key, 1.0});
    r.set = true;
    return r;
  }
  static LC axpy(const LC &a, double s, const LC &b) { // a + s*b
    LC r;
    r.set = a.set && b.set; // a ghost built from a cell nobody wrote is itself unwritten
    r.t.reserve(a.t.size() + b.t.size());
    size_t i = 0, j = 0;
    while (i < a.t.size() || j < b.t.size()) {
      if (j == b.t.size() || (i < a.t.size() && a.t[i].first < b.t[j].first)) r.t.push_back(a.t[i++]);
      else if (i == a.t.size() || b.t[j].first < a.t[i].first) { r.t.push_back({b.t[j].first, s * b.t[j].second}); j++; }
      else { r.t.push_back({a.t[i].first, a.t[i].second + s * b.t[j].second}); i++; j++; }
    }
    return r;
  }
};
LC operator+(const LC &a, const LC &b) { return LC::axpy(a, 1.0, b); }
LC operator-(const LC &a, const LC &b) { return LC::axpy(a, -1.0, b); }
LC operator*(double s, const LC &a) {
  LC r = a;
  for (auto &e : r.t) e.second *= s;
  return r;
}
LC operator-(const LC &a) { return -1.0 * a; }

int cdiv(int a, int b) { return a / b; } // C truncation, as the reference's index arithmetic

struct Mesh {
  std::vector<int> lij; // [n][3]
  std::map<std::array<int, 3>, int> index;
  int bpdx, bpdy;
  int state(int l, int i, int j) const { // >= 0 block id, -1 refined further, -2 covered by a coarser block
    auto it = index.find({l, i, j});
    if (it != index.end()) return it->second;
    while (l > 0) {
      l--, i >>= 1, j >>= 1;
      if (index.count({l, i, j})) return -2;
    }
    return -1;
  }
  int find(int l, int i, int j) const {
    auto it = index.find({l, i, j});
    return it == index.end() ? -1 : it->second;
  }
};

LC LI(const LC &a, const LC &b, const LC &c) {
  LC kappa = ((4.0 / 15.0) * a + (6.0 / 15.0) * c) + (-10.0 / 15.0) * b;
  LC lambda = (b - c) - kappa;
  return (4.0 * kappa + 2.0 * lambda) + c;
}
LC LE(const LC &a, const LC &b, const LC &c) {
  LC kappa = ((4.0 / 15.0) * a + (6.0 / 15.0) * c) + (-10.0 / 15.0) * b;
  LC lambda = (b - c) - kappa;
  return (9.0 * kappa + 3.0 * lambda) + c;
}
LC taylor2d(const LC C[3][3], int x, int y) { // C[i][j] at (XX-1+i, YY-1+j)
  const double dx = 0.25 * (2 * x - 1), dy = 0.25 * (2 * y - 1);
  LC dudx = 0.5 * (C[2][1] - C[0][1]);
  LC dudy = 0.5 * (C[1][2] - C[1][0]);
  LC dudxdy = 0.25 * ((C[0][0] + C[2][2]) - (C[2][0] + C[0][2]));
  LC dudx2 = (C[0][1] + C[2][1]) - 2.0 * C[1][1];
  LC dudy2 = (C[1][0] + C[1][2]) - 2.0 * C[1][1];
  return (C[1][1] + (dx * dudx + dy * dudy)) + (((0.5 * dx * dx) * dudx2 + (0.5 * dy * dy) * dudy2) + (dx * dy) * dudxdy);
}

struct LabBuilder {
  const Mesh &mesh;
  int dim, sx, sy, ex, ey;
  bool tens, vector_bc, use_averages;
  int nmx, nmy, ox, oy, ncx, ncy;
  std::vector<LC> m, c;
  int level, I, J, NX, NY;
  std::vector<std::array<int, 2>> coarsened_codes;
  std::map<std::array<int, 2>, int> myblocks;
  bool coarsened;

  LabBuilder(const Mesh &ms, int which) : mesh(ms) {
    if (which == 0) { dim = 2; sx = sy = -3; ex = ey = 4; tens = true; vector_bc = true; }
    else if (which == 1) { dim = 2; sx = sy = -1; ex = ey = 2; tens = false; vector_bc = true; }
    else if (which == 2) { dim = 1; sx = sy = -1; ex = ey = 2; tens = false; vector_bc = false; }
    // 4, 5: the labs adapt() refines a block from (main.cpp:4908-4967): +-1 with corners, vector / scalar wall rules
    else if (which == 4) { dim = 2; sx = sy = -1; ex = ey = 2; tens = true; vector_bc = true; }
    else if (which == 5) { dim = 1; sx = sy = -1; ex = ey = 2; tens = true; vector_bc = false; }
    // 6: KernelComputeForces's velocity lab (main.cpp:5576, 7188): +-4 with corners, vector wall rule
    else if (which == 6) { dim = 2; sx = sy = -4; ex = ey = 5; tens = true; vector_bc = true; }
    else { dim = 1; sx = sy = -4; ex = ey = 5; tens = true; vector_bc = false; } // GradChiOnTmp's chi lab (main.cpp:4633)
    nmx = BS + ex - sx - 1, nmy = BS + ey - sy - 1;
    ox = cdiv(sx - 1, 2) - 1, oy = cdiv(sy - 1, 2) - 1;
    ncx = H + cdiv(ex, 2) + 1 - ox, ncy = H + cdiv(ey, 2) + 1 - oy;
    use_averages = tens || sx < -2 || sy < -2 || ex > 3 || ey > 3;
  }
  LC &M(int ix, int iy, int d) { return m[((size_t)(iy - sy) * nmx + (ix - sx)) * dim + d]; }
  LC &C(int XX, int YY, int d) { return c[((size_t)(YY - oy) * ncx + (XX - ox)) * dim + d]; }
  LC S(int blk, int x, int y, int d) const { return LC::src(((int64_t)blk * 64 + y * BS + x) * dim + d); }
  void region(const int code[2], int s[2], int e[2]) const {
    const int st[2] = {sx, sy}, en[2] = {ex, ey};
    for (int d = 0; d < 2; d++) {
      s[d] = code[d] < 1 ? (code[d] < 0 ? st[d] : 0) : BS;
      e[d] = code[d] < 1 ? (code[d] < 0 ? 0 : BS) : BS + en[d] - 1;
    }
  }
  void cregion(const int code[2], int s[2], int e[2]) const {
    const int of[2] = {ox, oy}, en[2] = {ex, ey};
    for (int d = 0; d < 2; d++) {
      s[d] = code[d] < 1 ? (code[d] < 0 ? of[d] : 0) : H;
      e[d] = code[d] < 1 ? (code[d] < 0 ? 0 : H) : H + cdiv(en[d], 2) + 2 - 1;
    }
  }

  void load(int k) {
    level = mesh.lij[3 * k], I = mesh.lij[3 * k + 1], J = mesh.lij[3 * k + 2];
    NX = mesh.bpdx << level, NY = mesh.bpdy << level;
    m.assign((size_t)nmx * nmy * dim, LC());
    c.assign((size_t)ncx * ncy * dim, LC());
    for (int y = 0; y < BS; y++)
      for (int x = 0; x < BS; x++)
        for (int d = 0; d < dim; d++) M(x, y, d) = S(k, x, y, d);
    const bool xskin = I == 0 || I == NX - 1, yskin = J == 0 || J == NY - 1;
    const int xskip = I == 0 ? -1 : 1, yskip = J == 0 ? -1 : 1;
    std::vector<std::array<int, 2>> same;
    coarsened_codes.clear();
    myblocks.clear();
    for (int icode = 0; icode < 9; icode++) {
      const int code[2] = {icode % 3 - 1, icode / 3 - 1};
      if (code[0] == 0 && code[1] == 0) continue;
      if ((code[0] == xskip && xskin) || (code[1] == yskip && yskin)) continue;
      const int st = mesh.state(level, I + code[0], J + code[1]);
      if (st >= 0) same.push_back({code[0], code[1]});
      else if (st == -2) {
        coarsened_codes.push_back({code[0], code[1]});
        fill_from_coarse(code);
      }
      if (!tens && !use_averages && abs(code[0]) + abs(code[1]) > 1) continue;
      int s[2], e[2];
      region(code, s, e);
      if (st >= 0) {
        if (e[0] - s[0] == 0) continue;
        myblocks[{code[0], code[1]}] = st;
        for (int iy = s[1]; iy < e[1]; iy++)
          for (int ix = s[0]; ix < e[0]; ix++)
            for (int d = 0; d < dim; d++) M(ix, iy, d) = S(st, ix - code[0] * BS, iy - code[1] * BS, d);
      } else if (st == -1)
        fill_from_fine(code, s, e);
    }
    coarsened = false;
    if (!coarsened_codes.empty())
      for (auto &cd : same)
        if (use_coarse_stencil0(cd.data())) {
          fill_coarse_version(cd.data());
          coarsened = true;
        }
    post_load();
  }

  void fill_from_coarse(const int code[2]) { // coarse neighbour -> coarse lab, plain copies
    const int bi = (I + code[0]) >> 1, bj = (J + code[1]) >> 1; // arithmetic shift: floor also for -1
    const int kb = mesh.find(level - 1, bi, bj);
    if (kb < 0) return;
    int s[2], e[2];
    cregion(code, s, e);
    if (e[0] - s[0] == 0) return;
    for (int YY = s[1]; YY < e[1]; YY++)
      for (int XX = s[0]; XX < e[0]; XX++) {
        const int gx = H * I + XX - BS * bi, gy = H * J + YY - BS * bj;
        if (gx < 0 || gx >= BS || gy < 0 || gy >= BS) continue; // outside that block: the reference reads stale memory
        for (int d = 0; d < dim; d++) C(XX, YY, d) = S(kb, gx, gy, d);
      }
  }

  void fill_from_fine(const int code[2], const int s[2], const int e[2]) { // finer neighbours -> 2x2 averages
    const int ac0 = abs(code[0]), ac1 = abs(code[1]);
    const int nbytes = ac0 * (e[0] - s[0]) + (1 - ac0) * ((e[0] - s[0]) / 2);
    if (nbytes == 0) return;
    const int ys = code[1] == 0 ? 2 : 1;
    const int mod = ((e[1] - s[1]) / ys) % 4;
    const int Bstep = ac0 + ac1 == 2 ? 3 : 1;
    for (int B = 0; B <= 3; B += Bstep) {
      const int aux = ac0 == 1 ? (B % 2) : (B / 2);
      const int kb = mesh.find(level + 1, 2 * I + std::max(code[0], 0) + code[0] + (B % 2) * std::max(0, 1 - ac0),
                               2 * J + std::max(code[1], 0) + code[1] + aux * std::max(0, 1 - ac1));
      if (kb < 0) continue;
      const int i = ac0 * (s[0] - sx) + (1 - ac0) * (s[0] - sx + (B % 2) * (e[0] - s[0]) / 2);
      const int x = s[0] - code[0] * BS + std::min(0, code[0]) * (e[0] - s[0]);
      auto krow = [&](int iy) { return ac1 * (iy - sy) + (1 - ac1) * (iy / 2 - sy + aux * (e[1] - s[1]) / 2); };
      auto yrow = [&](int iy) { return ac1 == 1 ? 2 * (iy - code[1] * BS) + std::min(0, code[1]) * BS : iy; };
      auto put = [&](int row, int r0, int r1) {
        for (int ee = 0; ee < nbytes; ee++)
          for (int d = 0; d < dim; d++) {
            LC q00 = S(kb, x + 2 * ee, r0, d), q10 = S(kb, x + 2 * ee, r1, d);
            LC q01 = S(kb, x + 2 * ee + 1, r0, d), q11 = S(kb, x + 2 * ee + 1, r1, d);
            m[((size_t)row * nmx + (i + ee)) * dim + d] = 0.25 * (((q00 + q10) + q01) + q11);
          }
      };
      for (int iy = s[1]; iy < e[1] - mod; iy += 4 * ys)
        for (int r = 0; r < 4; r++) {
          const int y0 = yrow(iy + r * ys);
          // the first row of every group of four pairs fine row y0 with the first fine row of the NEXT coarse row
          const int y1 = r == 0 ? yrow(iy + ys) : y0 + 1;
          put(krow(iy + r * ys), y0, y1);
        }
      for (int iy = e[1] - mod; iy < e[1]; iy += ys) put(krow(iy), yrow(iy), yrow(iy) + 1);
    }
  }

  bool use_coarse_stencil0(const int code[2]) const {
    if (level == 0 || !use_averages) return false;
    const int idx[2] = {I, J}, nei[2] = {I + code[0], J + code[1]}, last[2] = {NX - 1, NY - 1};
    int lo[2], hi[2];
    for (int d = 0; d < 2; d++) {
      lo[d] = idx[d] < nei[d] ? 0 : -1;
      hi[d] = idx[d] > nei[d] ? 0 : 1;
      if (idx[d] == 0 && nei[d] == 0) lo[d] = 0;
      if (idx[d] == last[d] && nei[d] == last[d]) hi[d] = 0;
    }
    for (auto &cc : coarsened_codes)
      if (cc[0] >= lo[0] && cc[0] <= hi[0] && cc[1] >= lo[1] && cc[1] <= hi[1]) return true;
    return false;
  }

  void fill_coarse_version(const int code[2]) { // 2x2 averages of a same-level neighbour -> coarse lab
    auto it = myblocks.find({code[0], code[1]});
    if (it == myblocks.end()) return;
    const int kb = it->second;
    int s[2], e[2];
    cregion(code, s, e);
    if (e[0] - s[0] == 0) return;
    int st[2];
    for (int d = 0; d < 2; d++) st[d] = s[d] + std::max(code[d], 0) * H - code[d] * BS + std::min(0, code[d]) * (e[d] - s[d]);
    for (int iy = s[1]; iy < e[1]; iy++) {
      const int y0 = 2 * (iy - s[1]) + st[1];
      for (int ee = 0; ee < e[0] - s[0]; ee++)
        for (int d = 0; d < dim; d++) {
          LC q00 = S(kb, st[0] + 2 * ee, y0, d), q01 = S(kb, st[0] + 2 * ee + 1, y0, d);
          LC q10 = S(kb, st[0] + 2 * ee, y0 + 1, d), q11 = S(kb, st[0] + 2 * ee + 1, y0 + 1, d);
          C(s[0] + ee, iy, d) = 0.25 * (((q00 + q10) + q01) + q11);
        }
    }
  }

  void apply_bc(bool coarse) { // free-slip (vector) / Neumann (scalar) wall ghosts on the fine or the coarse lab
    const int beg[2] = {coarse ? cdiv(sx - 1, 2) - 1 : sx, coarse ? cdiv(sy - 1, 2) - 1 : sy};
    const int end[2] = {coarse ? cdiv(ex, 2) + 2 : ex, coarse ? cdiv(ey, 2) + 2 : ey};
    const int bsz = coarse ? H : BS;
    const bool on[4] = {I == 0, I == NX - 1, J == 0, J == NY - 1};
    for (int f = 0; f < 4; f++) {
      if (!on[f]) continue;
      const int dr = f / 2, side = f % 2;
      int s[2] = {beg[0], beg[1]}, e[2] = {bsz + end[0] - 1, bsz + end[1] - 1};
      s[dr] = side == 0 ? beg[dr] : bsz;
      e[dr] = side == 0 ? 0 : bsz + end[dr] - 1;
      for (int iy = s[1]; iy < e[1]; iy++)
        for (int ix = s[0]; ix < e[0]; ix++) {
          const int x = dr == 0 ? (side == 0 ? 0 : bsz - 1) : ix, y = dr == 1 ? (side == 0 ? 0 : bsz - 1) : iy;
          for (int d = 0; d < dim; d++) {
            const LC &srcv = coarse ? C(x, y, d) : M(x, y, d);
            const LC v = (vector_bc && d == dr) ? -srcv : srcv; // normal component negated
            if (coarse) C(ix, iy, d) = v; else M(ix, iy, d) = v;
          }
        }
    }
  }

  void post_load() {
    if (coarsened)
      for (int j = 0; j < H; j++)
        for (int i = 0; i < H; i++) {
          if (i > 1 && i < H - 2 && j > 2 && j < H - 2) continue;
          for (int d = 0; d < dim; d++)
            C(i, j, d) = 0.25 * (((M(2 * i, 2 * j + 1, d) + M(2 * i, 2 * j, d)) + M(2 * i + 1, 2 * j, d)) + M(2 * i + 1, 2 * j + 1, d));
        }
    apply_bc(true);
    const bool xskin = I == 0 || I == NX - 1, yskin = J == 0 || J == NY - 1;
    const int xskip = I == 0 ? -1 : 1, yskip = J == 0 ? -1 : 1;
    const int st2[2] = {sx, sy};
    for (auto &cd : coarsened_codes) {
      const int code[2] = {cd[0], cd[1]};
      if ((code[0] == xskip && xskin) || (code[1] == yskip && yskin)) continue;
      if (!tens && !use_averages && abs(code[0]) + abs(code[1]) > 1) continue;
      int s[2], e[2];
      region(code, s, e);
      if (e[0] - s[0] == 0) continue;
      int sC[2];
      for (int d = 0; d < 2; d++) sC[d] = code[d] < 1 ? (code[d] < 0 ? cdiv(st2[d] - 1, 2) : 0) : H;
      auto half = [&](int v, int d, int &par) { // fine index -> coarse index relative to sC, parity inside the coarse cell
        const int t = v - s[d] - std::min(0, code[d]) * ((e[d] - s[d]) % 2);
        par = abs(t) % 2;
        return cdiv(t, 2);
      };
      if (use_averages)
        for (int iy = s[1]; iy < e[1]; iy++)
          for (int ix = s[0]; ix < e[0]; ix++) {
            int x, y;
            const int XX = half(ix, 0, x) + sC[0], YY = half(iy, 1, y) + sC[1];
            LC Cm[3][3];
            for (int i = 0; i < 3; i++)
              for (int j = 0; j < 3; j++) Cm[i][j] = C(XX - 1 + i, YY - 1 + j, 0); // component 0 for every d
            const LC val = taylor2d(Cm, x, y);
            for (int d = 0; d < dim; d++) M(ix, iy, d) = val;
          }
      if (abs(code[0]) + abs(code[1]) != 1) continue;
      for (int iy = s[1]; iy < e[1]; iy += 2)
        for (int ix = s[0]; ix < e[0]; ix += 2) {
          int x, y;
          const int XX = half(ix, 0, x) + sC[0], YY = half(iy, 1, y) + sC[1];
          const int iyp = abs(iy) % 2 == 1 ? -1 : 1, ixp = abs(ix) % 2 == 1 ? -1 : 1;
          const double dx = 0.25 * (2 * x - 1), dy = 0.25 * (2 * y - 1);
          if (ix < -2 || iy < -2 || ix > BS + 1 || iy > BS + 1) continue;
          const bool inx = ix + ixp >= s[0] && ix + ixp < e[0], iny = iy + iyp >= s[1] && iy + iyp < e[1];
          for (int d = 0; d < dim; d++) {
            // 1-D quadratic along the face (tangential direction t), one-sided at the ends of the coarse block
            const bool alongy = code[0] != 0;
            const int T = alongy ? YY : XX;
            auto cc = [&](int k) { return alongy ? C(XX, YY + k, d) : C(XX + k, YY, d); };
            LC du, du2;
            if (T == 0) {
              du = (-0.5 * cc(2) - 1.5 * cc(0)) + 2.0 * cc(1);
              du2 = (cc(2) + cc(0)) - 2.0 * cc(1);
            } else if (T == H - 1) {
              du = (0.5 * cc(-2) + 1.5 * cc(0)) - 2.0 * cc(-1);
              du2 = (cc(-2) + cc(0)) - 2.0 * cc(-1);
            } else {
              du = 0.5 * (cc(1) - cc(-1));
              du2 = (cc(1) + cc(-1)) - 2.0 * cc(0);
            }
            const double dt = alongy ? dy : dx;
            LC plus = (cc(0) + dt * du) + (0.5 * dt * dt) * du2, minus = (cc(0) - dt * du) + (0.5 * dt * dt) * du2;
            M(ix, iy, d) = plus;
            if (alongy) {
              if (iny) M(ix, iy + iyp, d) = minus;
              if (inx) M(ix + ixp, iy, d) = plus;
              if (inx && iny) M(ix + ixp, iy + iyp, d) = minus;
            } else {
              if (iny) M(ix, iy + iyp, d) = plus;
              if (inx) M(ix + ixp, iy, d) = minus;
              if (inx && iny) M(ix + ixp, iy + iyp, d) = minus;
            }
          }
        }
      for (int iy = s[1]; iy < e[1]; iy++)
        for (int ix = s[0]; ix < e[0]; ix++) {
          if (ix < -2 || iy < -2 || ix > BS + 1 || iy > BS + 1) continue;
          int x, y;
          half(ix, 0, x);
          half(iy, 1, y);
          for (int d = 0; d < dim; d++) {
            LC a = M(ix, iy, d);
            if (code[0] == 0 && code[1] == 1) M(ix, iy, d) = y == 0 ? LI(a, M(ix, iy - 1, d), M(ix, iy - 2, d)) : LE(a, M(ix, iy - 2, d), M(ix, iy - 3, d));
            else if (code[0] == 0 && code[1] == -1) M(ix, iy, d) = y == 1 ? LI(a, M(ix, iy + 1, d), M(ix, iy + 2, d)) : LE(a, M(ix, iy + 2, d), M(ix, iy + 3, d));
            else if (code[0] == 1) M(ix, iy, d) = x == 0 ? LI(a, M(ix - 1, iy, d), M(ix - 2, iy, d)) : LE(a, M(ix - 2, iy, d), M(ix - 3, iy, d));
            else M(ix, iy, d) = x == 1 ? LI(a, M(ix + 1, iy, d), M(ix + 2, iy, d)) : LE(a, M(ix + 2, iy, d), M(ix + 3, iy, d));
          }
        }
    }
    apply_bc(false);
  }
};
} // namespace

struct GhostTable { // compact form: ghost rows of irregular blocks only
  std::vector<int64_t> rowptr;
  std::vector<int32_t> dst, src_block, src_cc; // dst = (position in the irregular list * ncell + lab cell) * dim + comp
  std::vector<double> w;
  int npatterns = 0, fallbacks = 0;
  bool built = false;
};

struct cup2d_amr_plan {
  Mesh mesh;
  std::vector<int32_t> irregular; // blocks with a coarser or finer block among their 8 neighbours
  GhostTable ghosts[7];                          // kinds 0-3 and 6
  // CSR per stencil kind: rows = (block, iy, ix, comp)
  std::vector<int64_t> rowptr[7];
  std::vector<int32_t> src_block[7], src_cc[7]; // source block, source cell*dim + comp
  std::vector<double> w[7];
  // coarse-fine faces: (fine block, fine face, coarse block, coarse face, half)
  std::vector<int32_t> faces;
  bool built[7] = {false, false, false, false, false, false, false};
};

// full lab rows of the blocks `ks` (in that order) for stencil kind `which`, appended to the CSR (rp, sb, sc, w)
static void lab_rows(const Mesh &mesh, int which, const int32_t *ks, int64_t n, std::vector<int64_t> &rp, std::vector<int32_t> &sb,
                     std::vector<int32_t> &sc, std::vector<double> &w) {
  LabBuilder lb(mesh, which);
  rp.assign(1, 0);
  for (int64_t q = 0; q < n; q++) {
    lb.load(ks[q]);
    for (auto &row : lb.m) {
      if (row.set)
        for (auto &t : row.t) {
          if (t.second == 0.0) continue;
          sb.push_back((int32_t)(t.first / (64 * lb.dim)));
          sc.push_back((int32_t)(t.first % (64 * lb.dim)));
          w.push_back(t.second);
        }
      rp.push_back((int64_t)w.size());
    }
  }
}

static void build(cup2d_amr_plan *p, int which) {
  const int n = (int)p->mesh.lij.size() / 3;
  std::vector<int32_t> all(n);
  for (int k = 0; k < n; k++) all[k] = k;
  lab_rows(p->mesh, which, all.data(), n, p->rowptr[which], p->src_block[which], p->src_cc[which], p->w[which]);
  p->built[which] = true;
}

const std::vector<int> &amr_plan_level_ij(const cup2d_amr_plan *p, int *bpdx, int *bpdy) {
  *bpdx = p->mesh.bpdx, *bpdy = p->mesh.bpdy;
  return p->mesh.lij;
}

// the full lab rows of a subset of blocks (csrc/amr_regrid.cu: the parents a regrid refines), without building or caching the
// table of the whole mesh
int amr_plan_subset_rows(cup2d_amr_plan *p, int which, int64_t nsub, const int32_t *blocks, std::vector<int64_t> &rowptr,
                         std::vector<int32_t> &src_block, std::vector<int32_t> &src_cellcomp, std::vector<double> &weight) {
  if (!p || which < 0 || which > 6 || nsub < 0) return CUP2D_EINVAL;
  const int64_t n = (int64_t)p->mesh.lij.size() / 3;
  for (int64_t q = 0; q < nsub; q++)
    if (blocks[q] < 0 || blocks[q] >= n) return CUP2D_EINVAL;
  src_block.clear(), src_cellcomp.clear(), weight.clear();
  lab_rows(p->mesh, which, blocks, nsub, rowptr, src_block, src_cellcomp, weight);
  return CUP2D_OK;
}

// ---- compact ghost tables -----------------------------------------------------------------------------------------
// The ghost stencil of a block depends on its surroundings only through a small local configuration: the state of its
// 8 neighbour positions (same level / wall / coarser / finer, and which of the blocks involved exist), the parity of
// its index (which quadrant of its parent it is) and which domain walls it touches.  Blocks with the same configuration
// share one PATTERN — the ghost rows with sources named relative to the block (level offset, block offset) — which is
// evaluated symbolically once (about 2 ms) and then instantiated per block by looking the relative blocks up (microseconds).
struct Pattern {
  std::vector<int64_t> len;
  std::vector<int32_t> cell, ref, sc; // cell = lab cell * dim + comp; ref indexes `refs`
  std::vector<double> w;
  std::vector<std::array<int, 3>> refs; // (level offset, di, dj) relative to (I,J), (I>>1,J>>1) or (2I,2J)
};

static std::vector<int> config_key(const Mesh &m, int k) {
  const int l = m.lij[3 * k], I = m.lij[3 * k + 1], J = m.lij[3 * k + 2];
  const int NX = m.bpdx << l, NY = m.bpdy << l;
  std::vector<int> key = {I & 1, J & 1, I == 0, I == NX - 1, J == 0, J == NY - 1, l == 0};
  for (int c = 0; c < 9; c++) {
    if (c == 4) continue;
    const int cx = c % 3 - 1, cy = c / 3 - 1, ni = I + cx, nj = J + cy;
    if (ni < 0 || nj < 0 || ni >= NX || nj >= NY) { key.push_back(9); continue; }
    const int st = m.state(l, ni, nj);
    if (st >= 0) key.push_back(0);
    else if (st == -2) key.push_back(m.find(l - 1, ni >> 1, nj >> 1) >= 0 ? 1 : 2);
    else { // finer: which of the (up to two) children that touch this block exist one level down
      int mask = 0;
      const int ac0 = abs(cx), ac1 = abs(cy);
      for (int B = 0; B < 2; B++) {
        const int aux = ac0 == 1 ? (B % 2) : (B / 2);
        if (m.find(l + 1, 2 * I + std::max(cx, 0) + cx + (B % 2) * std::max(0, 1 - ac0),
                   2 * J + std::max(cy, 0) + cy + aux * std::max(0, 1 - ac1)) >= 0)
          mask |= 1 << B;
      }
      // faces look at B = 0..3 but only two distinct children exist in 2-D; corners at one child
      for (int B = 2; B < 4; B++) {
        const int aux = ac0 == 1 ? (B % 2) : (B / 2);
        if (m.find(l + 1, 2 * I + std::max(cx, 0) + cx + (B % 2) * std::max(0, 1 - ac0),
                   2 * J + std::max(cy, 0) + cy + aux * std::max(0, 1 - ac1)) >= 0)
          mask |= 1 << B;
      }
      key.push_back(16 + mask);
    }
  }
  return key;
}

static Pattern make_pattern(LabBuilder &lb, const Mesh &m, int k) {
  Pattern pt;
  const int l = m.lij[3 * k], I = m.lij[3 * k + 1], J = m.lij[3 * k + 2];
  std::map<int, int> refidx;
  lb.load(k);
  for (int iy = lb.sy; iy < BS + lb.ey - 1; iy++)
    for (int ix = lb.sx; ix < BS + lb.ex - 1; ix++) {
      if (ix >= 0 && ix < BS && iy >= 0 && iy < BS) continue;
      for (int d = 0; d < lb.dim; d++) {
        const LC &row = lb.M(ix, iy, d);
        if (!row.set) continue;
        int64_t cnt = 0;
        for (auto &t : row.t) {
          if (t.second == 0.0) continue;
          const int blk = (int)(t.first / (64 * lb.dim));
          auto it = refidx.find(blk);
          if (it == refidx.end()) {
            const int bl = m.lij[3 * blk], bi = m.lij[3 * blk + 1], bj = m.lij[3 * blk + 2];
            const int dl = bl - l;
            const int base_i = dl == 0 ? I : (dl < 0 ? I >> 1 : 2 * I), base_j = dl == 0 ? J : (dl < 0 ? J >> 1 : 2 * J);
            it = refidx.emplace(blk, (int)pt.refs.size()).first;
            pt.refs.push_back({dl, bi - base_i, bj - base_j});
          }
          pt.ref.push_back(it->second);
          pt.sc.push_back((int32_t)(t.first % (64 * lb.dim)));
          pt.w.push_back(t.second);
          cnt++;
        }
        pt.len.push_back(cnt);
        pt.cell.push_back((int32_t)((((iy - lb.sy)) * lb.nmx + (ix - lb.sx)) * lb.dim + d));
      }
    }
  return pt;
}

static void build_ghosts(cup2d_amr_plan *p, int which) {
  GhostTable &g = p->ghosts[which];
  const Mesh &m = p->mesh;
  const int n = (int)p->irregular.size();
  LabBuilder lb0(m, which);
  const int ncell = lb0.nmx * lb0.nmy * lb0.dim;
  // 1. dictionary of local configurations (serial: a few dozen patterns even on large meshes)
  std::map<std::vector<int>, int> dict;
  std::vector<Pattern> patterns;
  std::vector<int> pat_of(n);
  for (int q = 0; q < n; q++) {
    auto key = config_key(m, p->irregular[q]);
    auto it = dict.find(key);
    if (it == dict.end()) {
      it = dict.emplace(key, (int)patterns.size()).first;
      patterns.push_back(make_pattern(lb0, m, p->irregular[q]));
    }
    pat_of[q] = it->second;
  }
  g.npatterns = (int)patterns.size();
  // 2. instantiate per block (independent: interleaved static partition over plain threads)
  std::vector<std::vector<int32_t>> ids(n);
  std::vector<char> okv(n, 1);
  auto resolve = [&](int t, int nt) {
    for (int q = t; q < n; q += nt) {
      const int k = p->irregular[q];
      const int l = m.lij[3 * k], I = m.lij[3 * k + 1], J = m.lij[3 * k + 2];
      const Pattern &pt = patterns[pat_of[q]];
      ids[q].resize(pt.refs.size());
      for (size_t r = 0; r < pt.refs.size(); r++) {
        const int dl = pt.refs[r][0];
        const int bi = (dl == 0 ? I : (dl < 0 ? I >> 1 : 2 * I)) + pt.refs[r][1], bj = (dl == 0 ? J : (dl < 0 ? J >> 1 : 2 * J)) + pt.refs[r][2];
        const int id = m.find(l + dl, bi, bj);
        if (id < 0) okv[q] = 0;
        ids[q][r] = id;
      }
    }
  };
  int nt = (int)std::thread::hardware_concurrency();
  nt = std::max(1, std::min({nt, 32, n / 256 + 1}));
  {
    std::vector<std::thread> pool;
    for (int t = 1; t < nt; t++) pool.emplace_back(resolve, t, nt);
    resolve(0, nt);
    for (auto &th : pool) th.join();
  }
  // 3. assemble.  A block whose relative blocks could not all be found is evaluated directly (never seen; kept as a net).
  std::map<int, Pattern> own;
  g.fallbacks = 0;
  for (int q = 0; q < n; q++)
    if (!okv[q]) {
      Pattern &o = own[q] = make_pattern(lb0, m, p->irregular[q]);
      const int k = p->irregular[q];
      const int l = m.lij[3 * k], I = m.lij[3 * k + 1], J = m.lij[3 * k + 2];
      ids[q].resize(o.refs.size());
      for (size_t r = 0; r < o.refs.size(); r++) {
        const int dl = o.refs[r][0];
        ids[q][r] = m.find(l + dl, (dl == 0 ? I : (dl < 0 ? I >> 1 : 2 * I)) + o.refs[r][1], (dl == 0 ? J : (dl < 0 ? J >> 1 : 2 * J)) + o.refs[r][2]);
      }
      g.fallbacks++;
    }
  auto pat = [&](int q) -> const Pattern & { return okv[q] ? patterns[pat_of[q]] : own.at(q); };
  std::vector<int64_t> row0(n + 1, 0), nnz0(n + 1, 0);
  for (int q = 0; q < n; q++) {
    row0[q + 1] = row0[q] + (int64_t)pat(q).len.size();
    nnz0[q + 1] = nnz0[q] + (int64_t)pat(q).w.size();
  }
  g.rowptr.resize(row0[n] + 1);
  g.dst.resize(row0[n]);
  g.src_block.resize(nnz0[n]);
  g.src_cc.resize(nnz0[n]);
  g.w.resize(nnz0[n]);
  g.rowptr[0] = 0;
  auto fill = [&](int t, int nthr) {
    for (int q = t; q < n; q += nthr) {
      const Pattern &pt = pat(q);
      int64_t at = nnz0[q];
      for (size_t r = 0; r < pt.len.size(); r++) {
        at += pt.len[r];
        g.rowptr[row0[q] + r + 1] = at;
        g.dst[row0[q] + r] = (int32_t)((int64_t)q * ncell + pt.cell[r]);
      }
      for (size_t e = 0; e < pt.w.size(); e++) g.src_block[nnz0[q] + e] = ids[q][pt.ref[e]];
      memcpy(g.src_cc.data() + nnz0[q], pt.sc.data(), pt.sc.size() * sizeof(int32_t));
      memcpy(g.w.data() + nnz0[q], pt.w.data(), pt.w.size() * sizeof(double));
    }
  };
  {
    std::vector<std::thread> pool;
    for (int t = 1; t < nt; t++) pool.emplace_back(fill, t, nt);
    fill(0, nt);
    for (auto &th : pool) th.join();
  }
  g.built = true;
}

extern "C" {

int cup2d_amr_plan_create(int64_t nblocks, const int32_t *level_ij, int32_t bpdx, int32_t bpdy, cup2d_amr_plan **out) {
  if (!level_ij || !out || nblocks <= 0 || bpdx <= 0 || bpdy <= 0) {
    cup2d::set_error("cup2d_amr_plan_create: bad arguments");
    return CUP2D_EINVAL;
  }
  auto *p = new cup2d_amr_plan;
  p->mesh.bpdx = bpdx, p->mesh.bpdy = bpdy;
  p->mesh.lij.assign(level_ij, level_ij + 3 * nblocks);
  for (int64_t k = 0; k < nblocks; k++) {
    const int l = level_ij[3 * k], i = level_ij[3 * k + 1], j = level_ij[3 * k + 2];
    if (l < 0 || l > 20 || i < 0 || j < 0 || i >= (bpdx << l) || j >= (bpdy << l) || p->mesh.index.count({l, i, j})) {
      delete p;
      cup2d::set_error("cup2d_amr_plan_create: block " + std::to_string(k) + " is outside the domain or duplicated");
      return CUP2D_EINVAL;
    }
    p->mesh.index[{l, i, j}] = (int)k;
  }
  // coarse-fine faces (what prepare0 registers, main.cpp:1683-1735): faces 0 = x-, 1 = x+, 2 = y-, 3 = y+
  static const int fc[4][2] = {{-1, 0}, {1, 0}, {0, -1}, {0, 1}};
  for (int64_t k = 0; k < nblocks; k++) {
    const int l = level_ij[3 * k], i = level_ij[3 * k + 1], j = level_ij[3 * k + 2];
    for (int f = 0; f < 4; f++) {
      const int ni = i + fc[f][0], nj = j + fc[f][1];
      if (ni < 0 || nj < 0 || ni >= (bpdx << l) || nj >= (bpdy << l)) continue;
      if (p->mesh.state(l, ni, nj) != -2) continue;
      const int kc = p->mesh.find(l - 1, ni >> 1, nj >> 1);
      if (kc < 0) { // 2:1 balance violated
        delete p;
        cup2d::set_error("cup2d_amr_plan_create: neighbouring blocks differ by more than one level");
        return CUP2D_EINVAL;
      }
      const int32_t rec[5] = {(int32_t)k, f, kc, f ^ 1, fc[f][0] != 0 ? j % 2 : i % 2};
      p->faces.insert(p->faces.end(), rec, rec + 5);
    }
  }
  for (int64_t k = 0; k < nblocks; k++) {
    const int l = level_ij[3 * k], i = level_ij[3 * k + 1], j = level_ij[3 * k + 2];
    bool irr = false;
    for (int c = 0; c < 9 && !irr; c++) {
      const int ni = i + c % 3 - 1, nj = j + c / 3 - 1;
      if (c == 4 || ni < 0 || nj < 0 || ni >= (bpdx << l) || nj >= (bpdy << l)) continue;
      irr = p->mesh.state(l, ni, nj) < 0;
    }
    if (irr) p->irregular.push_back((int32_t)k);
  }
  *out = p;
  return CUP2D_OK;
}

void cup2d_amr_plan_destroy(cup2d_amr_plan *p) { delete p; }

int64_t cup2d_amr_plan_irregular(cup2d_amr_plan *p, int32_t *out) {
  if (!p) return CUP2D_EINVAL;
  if (out) memcpy(out, p->irregular.data(), p->irregular.size() * sizeof(int32_t));
  return (int64_t)p->irregular.size();
}

int64_t cup2d_amr_plan_ghosts(cup2d_amr_plan *p, int which, int64_t *nrows, int64_t *rowptr, int32_t *dst, int32_t *src_block,
                              int32_t *src_cellcomp, double *weight) {
  if (!p || which < 0 || (which > 3 && which != 6)) return CUP2D_EINVAL;
  GhostTable &g = p->ghosts[which];
  if (!g.built) build_ghosts(p, which);
  const int64_t nnz = (int64_t)g.w.size();
  if (nrows) *nrows = (int64_t)g.dst.size();
  if (rowptr) memcpy(rowptr, g.rowptr.data(), g.rowptr.size() * sizeof(int64_t));
  if (dst) memcpy(dst, g.dst.data(), g.dst.size() * sizeof(int32_t));
  if (src_block) memcpy(src_block, g.src_block.data(), nnz * sizeof(int32_t));
  if (src_cellcomp) memcpy(src_cellcomp, g.src_cc.data(), nnz * sizeof(int32_t));
  if (weight) memcpy(weight, g.w.data(), nnz * sizeof(double));
  return nnz;
}

int64_t cup2d_amr_plan_stencil(cup2d_amr_plan *p, int which, int64_t *rowptr, int32_t *src_block, int32_t *src_cellcomp,
                               double *weight) {
  if (!p || which < 0 || which > 6) return CUP2D_EINVAL;
  if (!p->built[which]) build(p, which);
  const int64_t nnz = (int64_t)p->w[which].size();
  if (rowptr) memcpy(rowptr, p->rowptr[which].data(), p->rowptr[which].size() * sizeof(int64_t));
  if (src_block) memcpy(src_block, p->src_block[which].data(), nnz * sizeof(int32_t));
  if (src_cellcomp) memcpy(src_cellcomp, p->src_cc[which].data(), nnz * sizeof(int32_t));
  if (weight) memcpy(weight, p->w[which].data(), nnz * sizeof(double));
  return nnz;
}

/* ---- Poisson matrix of a multi-level mesh -----------------------------------------------------------------------------
 * The rows the reference's assembly loop pushes (main.cpp:7051-7113) for the cells whose 5-point stencil crosses a
 * coarse-fine face (makeFlux / interpolate / D1 / D2, main.cpp:5915-5997: weights 2/3, -1/5, 8/15 and the Taylor
 * corrections +-1/8, +-1/2, +-3/8 / 1/32, -1/16), complete, in CSR — every other row is the same-level stencil and is
 * described by the face-neighbour table.  Exactly what cup2d_poisson_create_general consumes.  Entries are accumulated
 * in the reference's order (it sums into a std::map per row), so the values are bitwise the reference's.
 * nbr_out[4k..] = W,E,S,N same-level neighbour of block k or -1 (wall, coarser, finer).  Returns the number of general
 * rows; irr_rows may be NULL to size (then *nnz_out is set and nothing else is written). */
int64_t cup2d_amr_plan_poisson(cup2d_amr_plan *p, int32_t *nbr_out, int64_t *nnz_out, int32_t *irr_rows,
                               int32_t *irr_rowptr, int32_t *irr_col, double *irr_val) {
  if (!p) return CUP2D_EINVAL;
  const Mesh &m = p->mesh;
  const int64_t n = (int64_t)m.lij.size() / 3;
  static const int fc[4][2] = {{-1, 0}, {1, 0}, {0, -1}, {0, 1}};
  int64_t nrows = 0, nnz = 0;
  if (irr_rowptr) irr_rowptr[0] = 0;
  for (int64_t k = 0; k < n; k++) {
    const int l = m.lij[3 * k], I = m.lij[3 * k + 1], J = m.lij[3 * k + 2];
    const int NX = m.bpdx << l, NY = m.bpdy << l;
    int st[4];
    for (int j = 0; j < 4; j++) {
      const int ni = I + fc[j][0], nj = J + fc[j][1];
      st[j] = (ni < 0 || nj < 0 || ni >= NX || nj >= NY) ? -9 : m.state(l, ni, nj); // -9: domain wall
      if (nbr_out) nbr_out[4 * k + j] = st[j] >= 0 ? st[j] : -1;
    }
    auto idx = [](int64_t blk, int x, int y) { return blk * 64 + y * BS + x; };
    for (int iy = 0; iy < BS; iy++)
      for (int ix = 0; ix < BS; ix++) {
        const bool valid[4] = {ix > 0, ix < BS - 1, iy > 0, iy < BS - 1};
        bool general = false;
        for (int j = 0; j < 4; j++) general = general || (!valid[j] && (st[j] == -1 || st[j] == -2));
        if (!general) continue;
        std::map<int64_t, double> row;
        const int64_t self = idx(k, ix, iy);
        const int inb[4][2] = {{ix - 1, iy}, {ix + 1, iy}, {ix, iy - 1}, {ix, iy + 1}};
        for (int j = 0; j < 4; j++) {
          if (valid[j]) {
            row[idx(k, inb[j][0], inb[j][1])] += 1;
            row[self] += -1;
            continue;
          }
          if (st[j] == -9) continue; // Neumann wall: the neighbour is simply absent
          const bool xface = j < 2;
          // tangential coordinate helpers of the face (main.cpp:5793-5812 / 5852-5866)
          auto isBD = [&](int t) { return t == BS - 1 || t == H - 1; };
          auto isFD = [&](int t) { return t == 0 || t == H; };
          auto interpolate = [&](int64_t cblk, int cx, int cy, int64_t close, int64_t far, double signInt, double signTaylor) {
            row[close] += signInt * 2. / 3.;
            row[far] += -signInt * 1. / 5.;
            const double tf = signInt * 8. / 15.;
            row[idx(cblk, cx, cy)] += tf;
            const int t = xface ? cy : cx;
            auto nei = [&](int d) { return xface ? idx(cblk, cx, cy + d) : idx(cblk, cx + d, cy); };
            struct E { int64_t c; double w; };
            E d1[3], d2[3];
            if (isBD(t)) {
              d1[0] = {nei(-2), 1. / 8.}, d1[1] = {nei(-1), -1. / 2.}, d1[2] = {nei(0), 3. / 8.};
              d2[0] = {nei(-2), 1. / 32.}, d2[1] = {nei(-1), -1. / 16.}, d2[2] = {nei(0), 1. / 32.};
            } else if (isFD(t)) {
              d1[0] = {nei(2), -1. / 8.}, d1[1] = {nei(1), 1. / 2.}, d1[2] = {nei(0), -3. / 8.};
              d2[0] = {nei(2), 1. / 32.}, d2[1] = {nei(1), -1. / 16.}, d2[2] = {nei(0), 1. / 32.};
            } else {
              d1[0] = {nei(-1), -1. / 8.}, d1[1] = {nei(1), 1. / 8.}, d1[2] = {nei(0), 0.};
              d2[0] = {nei(-1), 1. / 32.}, d2[1] = {nei(1), 1. / 32.}, d2[2] = {nei(0), -1. / 16.};
            }
            for (auto &e : d1) row[e.c] += signTaylor * tf * e.w;
            for (auto &e : d2) row[e.c] += tf * e.w;
          };
          if (st[j] >= 0) { // same level: the facing cell of the neighbour block
            const int fx = xface ? (j == 0 ? BS - 1 : 0) : ix, fy = xface ? iy : (j == 2 ? BS - 1 : 0);
            row[idx(st[j], fx, fy)] += 1.;
            row[self] += -1.;
          } else if (st[j] == -2) { // coarser: this (fine) cell against the coarse cell behind the face
            const int ni = I + fc[j][0], nj = J + fc[j][1];
            const int64_t cb = m.find(l - 1, ni >> 1, nj >> 1);
            if (cb < 0) {
              cup2d::set_error("cup2d_amr_plan_poisson: neighbouring blocks differ by more than one level");
              return CUP2D_EINVAL;
            }
            const int bx = I % 2 == 0 ? ix / 2 : ix / 2 + H, by = J % 2 == 0 ? iy / 2 : iy / 2 + H;
            const int cx = xface ? (j == 0 ? BS - 1 : 0) : bx, cy = xface ? by : (j == 2 ? BS - 1 : 0);
            const int64_t inward = xface ? idx(k, j == 0 ? ix + 1 : ix - 1, iy) : idx(k, ix, j == 2 ? iy + 1 : iy - 1);
            const double signTaylor = ((xface ? iy : ix) % 2 == 0) ? -1. : 1.;
            interpolate(cb, cx, cy, self, inward, 1., signTaylor);
            row[self] += -1.;
          } else { // finer: this (coarse) cell against the two fine cells behind the face
            const int t = xface ? iy : ix;
            const int hi = t >= H ? 1 : 0;
            const int ci = xface ? 2 * (I + fc[j][0]) + (j == 0 ? 1 : 0) : 2 * I + hi;
            const int cj = xface ? 2 * J + hi : 2 * (J + fc[j][1]) + (j == 2 ? 1 : 0);
            const int64_t fb = m.find(l + 1, ci, cj);
            if (fb < 0) {
              cup2d::set_error("cup2d_amr_plan_poisson: neighbouring blocks differ by more than one level");
              return CUP2D_EINVAL;
            }
            const int tf0 = (t % H) * 2; // first of the two fine cells along the face
            for (int q = 0; q < 2; q++) {
              auto fine = [&](int off) { // off = 0: the fine cell at the face, 1: the one behind it
                const int a = (j == 0 || j == 2) ? BS - 1 - off : off;
                return xface ? idx(fb, a, tf0 + q) : idx(fb, tf0 + q, a);
              };
              row[fine(0)] += 1.;
              interpolate(k, ix, iy, fine(0), fine(1), -1., q == 0 ? -1. : 1.);
            }
          }
        }
        if (irr_rows) {
          irr_rows[nrows] = (int32_t)self;
          for (auto &e : row) {
            irr_col[nnz] = (int32_t)e.first;
            irr_val[nnz] = e.second;
            nnz++;
          }
          irr_rowptr[nrows + 1] = (int32_t)nnz;
        } else
          nnz += (int64_t)row.size();
        nrows++;
      }
  }
  if (nnz_out) *nnz_out = nnz;
  return nrows;
}

/* bookkeeping of the last cup2d_amr_plan_ghosts(which): distinct local configurations, directly evaluated blocks */
int cup2d_amr_plan_stats(cup2d_amr_plan *p, int which, int32_t *npatterns, int32_t *fallbacks) {
  if (!p || which < 0 || (which > 3 && which != 6) || !p->ghosts[which].built) return CUP2D_EINVAL;
  if (npatterns) *npatterns = p->ghosts[which].npatterns;
  if (fallbacks) *fallbacks = p->ghosts[which].fallbacks;
  return CUP2D_OK;
}

/* the 8 neighbour positions of every block, order (-1,-1),(0,-1),(1,-1),(-1,0),(1,0),(-1,1),(0,1),(1,1):
 * >= 0 same-level block, -1 domain wall, -2 covered by a coarser block, -3 refined further */
int cup2d_amr_plan_neighbours(cup2d_amr_plan *p, int32_t *out) {
  if (!p || !out) return CUP2D_EINVAL;
  const Mesh &m = p->mesh;
  const int64_t n = (int64_t)m.lij.size() / 3;
  for (int64_t k = 0; k < n; k++) {
    const int l = m.lij[3 * k], I = m.lij[3 * k + 1], J = m.lij[3 * k + 2];
    int q = 0;
    for (int c = 0; c < 9; c++) {
      if (c == 4) continue;
      const int ni = I + c % 3 - 1, nj = J + c / 3 - 1;
      int v = -1;
      if (ni >= 0 && nj >= 0 && ni < (m.bpdx << l) && nj < (m.bpdy << l)) {
        const int st = m.state(l, ni, nj);
        v = st >= 0 ? st : (st == -2 ? -2 : -3);
      }
      out[8 * k + q++] = v;
    }
  }
  return CUP2D_OK;
}

/* ---- adapt()'s refine / compress decision (main.cpp:4676-4860) and the order of the new block list (fill_pos, Encode:
 * main.cpp:1550-1553, 422-445, SpaceCurve 342-421 and 6342-6376).  Host only: a pure function of the block list and the
 * per-block L-inf of the tagging field (cup2d_amr_adapt_tags).  The states are updated in place in the reference's loop
 * order (blocks in list order, levels from levelMax-1 down), so the result is the reference's, order effects included.
 * Neighbour positions outside the domain are skipped; the reference wraps their index, which differs only on a level with a
 * single block row or column. */
namespace {
struct Curve { // SpaceCurve::forward / inverse / Encode
  int bpdx, bpdy, lmax, base = 0;
  bool regular = true;
  std::vector<int64_t> zsave;            // [j * bpdx + i]
  std::vector<std::array<int, 2>> inv;   // zsave value -> (i, j)
  static int64_t xy2d(int b, int x, int y) {
    const int n = 1 << b;
    int64_t d = 0;
    for (int s = n / 2; s > 0; s /= 2) {
      const int rx = (x & s) > 0, ry = (y & s) > 0;
      d += (int64_t)s * s * ((3 * rx) ^ ry);
      if (ry == 0) {
        if (rx == 1) x = n - 1 - x, y = n - 1 - y;
        std::swap(x, y);
      }
    }
    return d;
  }
  static void d2xy(int b, int64_t t, int &x, int &y) {
    const int n = 1 << b;
    x = y = 0;
    for (int64_t s = 1; s < n; s *= 2) {
      const int64_t rx = 1 & (t / 2), ry = 1 & (t ^ rx);
      if (ry == 0) {
        if (rx == 1) x = (int)s - 1 - x, y = (int)s - 1 - y;
        std::swap(x, y);
      }
      x += (int)(s * rx), y += (int)(s * ry);
      t /= 4;
    }
  }
  Curve(int bx, int by, int lm) : bpdx(bx), bpdy(by), lmax(lm), zsave((size_t)bx * by), inv((size_t)bx * by) {
    while ((1 << base) < std::max(bx, by)) base++;
    for (int j = 0; j < by; j++)
      for (int i = 0; i < bx; i++) {
        int64_t index = xy2d(base, i, j), sub = 0;
        for (int64_t h = 0; h < index; h++) {
          int x, y;
          d2xy(base, h, x, y);
          sub += x >= bx || y >= by;
        }
        if (sub) regular = false;
        zsave[(size_t)j * bx + i] = index - sub;
        inv[index - sub] = {i, j};
      }
  }
  int64_t forward(int l, int i, int j) const {
    if (l >= lmax) return 0;
    if (regular) return xy2d(l + base, i, j);
    const int aux = 1 << l, I = i / aux, J = j / aux;
    return xy2d(l, i - I * aux, j - J * aux) + zsave[(size_t)J * bpdx + I] * aux * aux;
  }
  void inverse(int64_t Z, int l, int &i, int &j) const {
    if (regular) return d2xy(l + base, Z, i, j);
    const int64_t aux = 1LL << l;
    d2xy(l, Z % (aux * aux), i, j);
    const auto &IJ = inv[(size_t)(Z / (aux * aux))];
    i += IJ[0] * (int)aux, j += IJ[1] * (int)aux;
  }
  int64_t encode(int level, int i, int j) const {
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
enum { LEAVE = 0, REFINE = 1, COMPRESS = 2 };
} // namespace

int64_t cup2d_amr_adapt_mesh(int64_t nblocks, const int32_t *level_ij, int32_t bpdx, int32_t bpdy, int32_t level_max,
                             const double *block_linf, double rtol, double ctol, int32_t *new_level_ij) {
  if (!level_ij || !block_linf || nblocks <= 0 || bpdx <= 0 || bpdy <= 0 || level_max < 1 || level_max > 20) {
    cup2d::set_error("cup2d_amr_adapt_mesh: bad arguments");
    return CUP2D_EINVAL;
  }
  Mesh m;
  m.bpdx = bpdx, m.bpdy = bpdy;
  m.lij.assign(level_ij, level_ij + 3 * nblocks);
  for (int64_t k = 0; k < nblocks; k++) {
    const int l = level_ij[3 * k], i = level_ij[3 * k + 1], j = level_ij[3 * k + 2];
    if (l < 0 || l >= level_max || i < 0 || j < 0 || i >= (bpdx << l) || j >= (bpdy << l) || m.index.count({l, i, j})) {
      cup2d::set_error("cup2d_amr_adapt_mesh: block " + std::to_string(k) + " is outside the domain, above levelMax-1 or duplicated");
      return CUP2D_EINVAL;
    }
    m.index[{l, i, j}] = (int)k;
  }
  std::vector<int> st(nblocks);
  auto state_at = [&](int l, int i, int j) { // state of an existing block, LEAVE for a position without one
    const int k = m.find(l, i, j);
    return k < 0 ? (int)LEAVE : st[k];
  };
  for (int64_t k = 0; k < nblocks; k++) { // main.cpp:4682-4688
    const int l = level_ij[3 * k];
    int s = block_linf[k] > rtol ? REFINE : block_linf[k] < ctol ? COMPRESS : LEAVE;
    if ((s == REFINE && l == level_max - 1) || (s == COMPRESS && l == 0)) s = LEAVE;
    st[k] = s;
  }
  auto neighbours = [&](int l, int I, int J, auto &&visit) { // in the reference's (x outer, y inner) order; false stops
    const int NX = bpdx << l, NY = bpdy << l;
    const bool xskin = I == 0 || I == NX - 1, yskin = J == 0 || J == NY - 1;
    const int xskip = I == 0 ? -1 : 1, yskip = J == 0 ? -1 : 1;
    for (int x = -1; x < 2; x++)
      for (int y = -1; y < 2; y++) {
        if ((x == 0 && y == 0) || (x == xskip && xskin) || (y == yskip && yskin)) continue;
        if (I + x < 0 || I + x >= NX || J + y < 0 || J + y >= NY) continue;
        if (!visit(x, y)) return;
      }
  };
  for (int lv = level_max - 1; lv >= 0; lv--) {
    for (int64_t k = 0; k < nblocks; k++) { // main.cpp:4735-4785: finer neighbours
      const int l = level_ij[3 * k], I = level_ij[3 * k + 1], J = level_ij[3 * k + 2];
      if (l != lv || st[k] == REFINE || l == level_max - 1) continue;
      neighbours(l, I, J, [&](int x, int y) {
        if (m.state(l, I + x, J + y) != -1) return true;
        if (st[k] == COMPRESS) st[k] = LEAVE;
        const int Bstep = abs(x) + abs(y) == 2 ? 3 : 1;
        for (int B = 0; B <= 1; B += Bstep) {
          const int aux = abs(x) == 1 ? B % 2 : B / 2;
          const int iN = 2 * I + std::max(x, 0) + x + (B % 2) * std::max(0, 1 - abs(x));
          const int jN = 2 * J + std::max(y, 0) + y + aux * std::max(0, 1 - abs(y));
          if (state_at(lv + 1, iN, jN) == REFINE) {
            st[k] = REFINE;
            return false;
          }
        }
        return true;
      });
    }
    if (lv == 0) break;
    for (int64_t k = 0; k < nblocks; k++) { // main.cpp:4791-4823: a same-level neighbour refines
      const int l = level_ij[3 * k], I = level_ij[3 * k + 1], J = level_ij[3 * k + 2];
      if (l != lv || st[k] != COMPRESS) continue;
      neighbours(l, I, J, [&](int x, int y) {
        if (state_at(l, I + x, J + y) != REFINE) return true;
        st[k] = LEAVE;
        return false;
      });
    }
  }
  for (int64_t k = 0; k < nblocks; k++) { // main.cpp:4825-4860: all four siblings compress, or none does
    const int l = level_ij[3 * k], I = level_ij[3 * k + 1], J = level_ij[3 * k + 2];
    const int i0 = 2 * (I / 2), j0 = 2 * (J / 2);
    bool all = true;
    for (int a = 0; a < 2; a++)
      for (int b = 0; b < 2; b++) {
        const int s = m.find(l, i0 + a, j0 + b);
        all = all && s >= 0 && st[s] == COMPRESS;
      }
    if (all) continue;
    for (int a = 0; a < 2; a++)
      for (int b = 0; b < 2; b++) {
        const int s = m.find(l, i0 + a, j0 + b);
        if (s >= 0 && st[s] == COMPRESS) st[s] = LEAVE;
      }
  }
  std::vector<std::array<int, 3>> out; // main.cpp:4926-5195, then fill_pos
  for (int64_t k = 0; k < nblocks; k++) {
    const int l = level_ij[3 * k], i = level_ij[3 * k + 1], j = level_ij[3 * k + 2];
    if (st[k] == REFINE)
      for (int b = 0; b < 2; b++)
        for (int a = 0; a < 2; a++) out.push_back({l + 1, 2 * i + a, 2 * j + b});
    else if (st[k] == COMPRESS) {
      if (i % 2 == 0 && j % 2 == 0) out.push_back({l - 1, i / 2, j / 2});
    } else
      out.push_back({l, i, j});
  }
  if (new_level_ij) {
    const Curve curve(bpdx, bpdy, level_max);
    std::vector<std::pair<int64_t, size_t>> key(out.size());
    for (size_t q = 0; q < out.size(); q++) key[q] = {curve.encode(out[q][0], out[q][1], out[q][2]), q};
    std::sort(key.begin(), key.end());
    for (size_t q = 0; q < out.size(); q++) memcpy(new_level_ij + 3 * q, out[key[q].second].data(), 3 * sizeof(int32_t));
  }
  return (int64_t)out.size();
}

int64_t cup2d_amr_plan_faces(cup2d_amr_plan *p, int32_t *out) {
  if (!p) return CUP2D_EINVAL;
  if (out) memcpy(out, p->faces.data(), p->faces.size() * sizeof(int32_t));
  return (int64_t)p->faces.size() / 5;
}

} // extern "C"
