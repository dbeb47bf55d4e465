"""TEST INFRASTRUCTURE — not part of the product path.

adapt() on a multi-level (block-AMR) mesh, single rank: a numpy restatement of the refine / compress decision
(main.cpp:4676-4860), of the order of the new block list (fill_pos / SpaceCurve::Encode, main.cpp:1550-1553, 342-446,
6342-6376) and of the field transfer (main.cpp:4902-5195: refine from the {-1,-1,2,2,tensorial} lab of the old mesh, compress
by the 4-cell average, copy the rest).  The labs are those of oracle/cup2d_amr_oracle.py.  Pinned bit for bit against the
reference's own adapt() on its run.sh mesh (tests/golden/amrregrid_lmax*.npz, tests/golden/make_regrid_golden.py).
"""
import numpy as np

from cup2d_amr_oracle import BS, H, Lab, Mesh  # noqa: F401  (Mesh: the block lists these functions take)


class SpaceCurve:
    """SpaceCurve::forward / inverse / Encode (main.cpp:342-446; base curve and Zsave: main.cpp:6342-6376)"""

    def __init__(self, bpdx, bpdy, level_max):
        import cup2d_oracle as orc
        self.xy2d, self.d2xy = orc.hilbert_xy2d, orc.hilbert_d2xy
        self.bpdx, self.bpdy, self.level_max = bpdx, bpdy, level_max
        b = 0
        while (1 << b) < max(bpdx, bpdy):
            b += 1
        self.base, self.regular, self.zsave, self.inv = b, True, {}, {}
        for j in range(bpdy):
            for i in range(bpdx):
                index = self.xy2d(b, i, j)
                sub = 0
                for h in range(index):
                    x, y = self.d2xy(b, h)
                    sub += x >= bpdx or y >= bpdy
                if sub:
                    self.regular = False
                self.zsave[(i, j)] = index - sub
                self.inv[index - sub] = (i, j)

    def forward(self, l, i, j):
        if l >= self.level_max:
            return 0
        if self.regular:
            return self.xy2d(l + self.base, i, j)
        aux = 1 << l
        I, J = i // aux, j // aux
        return self.xy2d(l, i - I * aux, j - J * aux) + self.zsave[(I, J)] * aux * aux

    def inverse(self, Z, l):
        if self.regular:
            return self.d2xy(l + self.base, Z)
        aux = 1 << l
        x, y = self.d2xy(l, Z % (aux * aux))
        I, J = self.inv[Z // (aux * aux)]
        return x + I * aux, y + J * aux

    def encode(self, level, i, j):
        """the sort key id2 of fill_pos (main.cpp:1550-1553)"""
        r, ix, iy = 0, i, j
        for l in range(level, -1, -1):
            r += self.forward(l, ix, iy)
            ix, iy = ix // 2, iy // 2
        ix, iy = 2 * i, 2 * j
        for l in range(level + 1, self.level_max):
            Zc = self.forward(l, ix, iy)
            Zc -= Zc % 4
            r += Zc
            ix1, iy1 = self.inverse(Zc, l)
            ix, iy = 2 * ix1, 2 * iy1
        return r + level


REFINE, LEAVE, COMPRESS = 1, 0, -1


def amr_adapt_states(mesh, block_linf, rtol, ctol, level_max):
    """adapt()'s per-block decision (main.cpp:4676-4860) in `infos` order, with the reference's in-place updates: the
    thresholds; Refine at levelMax-1 and Compress at level 0 dropped; from levelMax-1 down to 0, a block with finer
    neighbours cannot compress and refines if one of the finer blocks it touches refines, then (levels > 0) a Compress next
    to a same-level Refine is dropped; finally a Compress stays only if its three siblings exist and compress too.
    Neighbours outside the domain are skipped (the reference wraps their index, which matters only on a level with a single
    block row or column)."""
    blocks = mesh.blocks
    st = {}
    for k, (l, i, j) in enumerate(blocks):
        s = REFINE if block_linf[k] > rtol else (COMPRESS if block_linf[k] < ctol else LEAVE)
        if (s == REFINE and l == level_max - 1) or (s == COMPRESS and l == 0):
            s = LEAVE
        st[(l, i, j)] = s

    def neighbours(l, I, J):
        NX, NY = mesh.bpdx << l, mesh.bpdy << l
        xskin, yskin = I == 0 or I == NX - 1, J == 0 or J == NY - 1
        xskip, yskip = (-1 if I == 0 else 1), (-1 if J == 0 else 1)
        for x in (-1, 0, 1):
            for y in (-1, 0, 1):
                if (x, y) == (0, 0) or (x == xskip and xskin) or (y == yskip and yskin):
                    continue
                if 0 <= I + x < NX and 0 <= J + y < NY:
                    yield x, y

    for m in range(level_max - 1, -1, -1):
        for (l, I, J) in blocks:
            if l != m or st[(l, I, J)] == REFINE or l == level_max - 1:
                continue
            done = False
            for x, y in neighbours(l, I, J):
                if done:
                    break
                if mesh.state(l, I + x, J + y) != -1:
                    continue
                if st[(l, I, J)] == COMPRESS:
                    st[(l, I, J)] = LEAVE
                for B in range(0, 2, 3 if abs(x) + abs(y) == 2 else 1):
                    aux = B % 2 if abs(x) == 1 else B // 2
                    iN = 2 * I + max(x, 0) + x + (B % 2) * max(0, 1 - abs(x))
                    jN = 2 * J + max(y, 0) + y + aux * max(0, 1 - abs(y))
                    if st.get((m + 1, iN, jN), LEAVE) == REFINE:
                        st[(l, I, J)] = REFINE
                        done = True
                        break
        if m == 0:
            break
        for (l, I, J) in blocks:
            if l != m or st[(l, I, J)] != COMPRESS:
                continue
            for x, y in neighbours(l, I, J):
                if st.get((l, I + x, J + y)) == REFINE:
                    st[(l, I, J)] = LEAVE
                    break
    for (l, I, J) in blocks:
        sib = [(l, 2 * (I // 2) + a, 2 * (J // 2) + b) for a in (0, 1) for b in (0, 1)]
        if not all(st.get(s) == COMPRESS for s in sib):
            for s in sib:
                if st.get(s) == COMPRESS:
                    st[s] = LEAVE
    return [st[b] for b in blocks]


def amr_adapt_mesh(mesh, block_linf, rtol, ctol, level_max):
    """the block list after adapt() (main.cpp:4926-5195), in the reference's order: sorted by Encode (fill_pos,
    main.cpp:1550-1553, 422-445)"""
    states = amr_adapt_states(mesh, block_linf, rtol, ctol, level_max)
    new = []
    for (l, i, j), s in zip(mesh.blocks, states):
        if s == REFINE:
            new += [(l + 1, 2 * i + a, 2 * j + b) for b in (0, 1) for a in (0, 1)]
        elif s == COMPRESS:
            if i % 2 == 0 and j % 2 == 0:
                new.append((l - 1, i // 2, j // 2))
        else:
            new.append((l, i, j))
    sc = SpaceCurve(mesh.bpdx, mesh.bpdy, level_max)
    new.sort(key=lambda b: sc.encode(*b))
    return np.array(new, dtype=np.int32).reshape(-1, 3)


def refine_block(m, dim):
    """the four children of a parent from its {-1,-1,2,2,tensorial} lab m[10, 10, dim] (main.cpp:4982-5031), in the reference's
    expression order; returns children[J*2 + I] as (8, 8, dim) arrays"""
    out = np.zeros((4, BS, BS, dim))
    for J in range(2):
        for I in range(2):
            b = out[2 * J + I]
            for j in range(0, BS, 2):
                for i in range(0, BS, 2):
                    i0, j0 = i // 2 + I * H + 1, j // 2 + J * H + 1
                    for d in range(dim):
                        l00, l0p, lm0 = m[j0, i0, d], m[j0 + 1, i0, d], m[j0, i0 - 1, d]
                        lmm, lmp, lp0 = m[j0 - 1, i0 - 1, d], m[j0 + 1, i0 - 1, d], m[j0, i0 + 1, d]
                        lpm, lpp, l0m = m[j0 - 1, i0 + 1, d], m[j0 + 1, i0 + 1, d], m[j0 - 1, i0, d]
                        x = 0.5 * (lp0 - lm0)
                        y = 0.5 * (l0p - l0m)
                        x2 = (lp0 + lm0) - 2.0 * l00
                        y2 = (l0p + l0m) - 2.0 * l00
                        xy = 0.25 * ((lpp + lmm) - (lpm + lmp))
                        c = 0.03125 * x2 + 0.03125 * y2
                        b[j, i, d] = (l00 + (-0.25 * x - 0.25 * y)) + (c + 0.0625 * xy)
                        b[j, i + 1, d] = (l00 + (+0.25 * x - 0.25 * y)) + (c - 0.0625 * xy)
                        b[j + 1, i, d] = (l00 + (-0.25 * x + 0.25 * y)) + (c - 0.0625 * xy)
                        b[j + 1, i + 1, d] = (l00 + (+0.25 * x + 0.25 * y)) + (c + 0.0625 * xy)
    return out


def compress_blocks(children):
    """the parent of four children[J*2 + I] (main.cpp:5147-5166): (b[i00] + b[i01] + b[i10] + b[i11]) / 4, i01 = the row
    above, i10 = the next column"""
    out = np.empty_like(children[0])
    for J in range(2):
        for I in range(2):
            b = children[2 * J + I]
            out[J * H:(J + 1) * H, I * H:(I + 1) * H] = (((b[0::2, 0::2] + b[1::2, 0::2]) + b[0::2, 1::2]) + b[1::2, 1::2]) / 4
    return out


def amr_regrid(mesh, new_blocks, fields):
    """adapt()'s field transfer (main.cpp:4902-5195) onto `new_blocks` (any order): fields = {name: (array[nb, 8, 8, dim],
    'vector' | 'scalar')}.  A refined parent's children come from its {-1,-1,2,2,tensorial} lab on the OLD mesh with wall
    ghosts; a compressed group becomes its parent; every other block is copied.  Returns {name: array[len(new_blocks), ...]}."""
    out = {}
    for name, (f, kind) in fields.items():
        dim = f.shape[-1]
        lab = Lab(mesh, f, (-1, -1, 2, 2, True), kind)
        res = np.empty((len(new_blocks), BS, BS, dim))
        kids = {}
        for n, (l, i, j) in enumerate(map(tuple, new_blocks)):
            k = mesh.index.get((l, i, j))
            if k is not None:
                res[n] = f[k]
            elif (l - 1, i // 2, j // 2) in mesh.index:
                kp = mesh.index[(l - 1, i // 2, j // 2)]
                if kp not in kids:
                    kids[kp] = refine_block(lab.load(kp), dim)
                res[n] = kids[kp][2 * (j % 2) + (i % 2)]
            else:
                res[n] = compress_blocks([f[mesh.index[(l + 1, 2 * i + a, 2 * j + b)]] for b in (0, 1) for a in (0, 1)])
        out[name] = res
    return out
