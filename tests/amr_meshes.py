"""Generated 2:1-balanced multi-level meshes and block orders, shared by the CPU tests of the plan (tests/test_amr_meshes.py)
and the device tests on them (tests/test_gpu_amr_meshes.py), so that both always exercise the same cases.

A mesh is a list of (level, i, j) leaves covering a domain of bpdx x bpdy level-0 blocks.  Neighbouring leaves, across a face
or a corner, differ by at most one level: the rule cup2d_amr_plan_create enforces."""
import numpy as np

import cup2d_b200


def _cover(blocks, l, i, j):
    """the leaf covering the level-l block position (i, j), or None when finer leaves cover it"""
    while l >= 0:
        if (l, i, j) in blocks:
            return (l, i, j)
        l, i, j = l - 1, i >> 1, j >> 1
    return None


def _refine(blocks, b):
    l, i, j = b
    blocks.discard(b)
    blocks.update((l + 1, 2 * i + a, 2 * j + c) for a in (0, 1) for c in (0, 1))


def _balance(blocks, bpdx, bpdy):
    """refine coarse leaves until every face and corner neighbour of every leaf is at most one level coarser"""
    changed = True
    while changed:
        changed = False
        for (l, i, j) in sorted(blocks, reverse=True):
            if (l, i, j) not in blocks:
                continue
            for di in (-1, 0, 1):
                for dj in (-1, 0, 1):
                    a, c = i + di, j + dj
                    if (di, dj) == (0, 0) or not (0 <= a < bpdx << l and 0 <= c < bpdy << l):
                        continue
                    cov = _cover(blocks, l, a, c)
                    if cov is not None and cov[0] < l - 1:
                        _refine(blocks, cov)
                        changed = True


def balanced_mesh(bpdx, bpdy, base, top, seeds=(), radius=1.0, sprinkle=0.0, seed=0):
    """level `base` everywhere, then level by level up to `top`: a level-L leaf is refined if its centre lies within
    radius / 2^(L - base) (level-0 block units) of a seed point, or with probability `sprinkle`; 2:1 balance across faces
    and corners is restored after every level.  Returns the leaves sorted by (level, i, j) as an int32 array [nb, 3]."""
    rng = np.random.default_rng(seed)
    blocks = {(base, i, j) for i in range(bpdx << base) for j in range(bpdy << base)}
    pts = np.asarray(seeds, dtype=np.float64).reshape(-1, 2)
    for L in range(base, top):
        r = radius / (1 << (L - base))
        for b in sorted(blocks):
            l, i, j = b
            if l != L:
                continue
            c = np.array([(i + 0.5) / (1 << l), (j + 0.5) / (1 << l)])
            near = len(pts) > 0 and np.hypot(*(pts - c).T).min() < r
            if near or rng.uniform() < sprinkle:
                _refine(blocks, b)
        _balance(blocks, bpdx, bpdy)
    return np.array(sorted(blocks), dtype=np.int32).reshape(-1, 3)


def uniform_mesh(bpdx, bpdy, level=0):
    return np.array([(level, i, j) for i in range(bpdx << level) for j in range(bpdy << level)], dtype=np.int32)


ORDERS = ["sorted", "hilbert", "reversed", "random"]


def order(blocks, bpdx, bpdy, kind, seed=0):
    """the block list in one of ORDERS: sorted by (level, i, j); level by level, each level in the order of
    cup2d_block_order; the sorted list reversed; a seeded random permutation"""
    b = np.asarray(blocks, dtype=np.int32)
    s = b[np.lexsort((b[:, 2], b[:, 1], b[:, 0]))]
    if kind == "sorted":
        return np.ascontiguousarray(s)
    if kind == "reversed":
        return np.ascontiguousarray(s[::-1])
    if kind == "random":
        return np.ascontiguousarray(s[np.random.default_rng(len(b) + seed).permutation(len(b))])
    if kind == "hilbert":
        out = []
        for L in np.unique(s[:, 0]):
            rank = {tuple(ij): q for q, ij in enumerate(cup2d_b200.block_order(bpdx, bpdy, int(L)).tolist())}
            lv = s[s[:, 0] == L]
            out.append(lv[np.argsort([rank[(i, j)] for _, i, j in lv.tolist()], kind="stable")])
        return np.ascontiguousarray(np.concatenate(out))
    raise ValueError(kind)


def reference_order(blocks, bpdx, bpdy, level_max):
    """the reference's list order (fill_pos: sorted by SpaceCurve::Encode, tests/amr_adapt_oracle.py)"""
    import amr_adapt_oracle as ado
    sc = ado.SpaceCurve(bpdx, bpdy, level_max)
    b = [tuple(x) for x in np.asarray(blocks).tolist()]
    b.sort(key=lambda x: sc.encode(*x))
    return np.array(b, dtype=np.int32).reshape(-1, 3)


# ---- the fixed case list ---------------------------------------------------------------------------------------------
# name: (bpdx, bpdy, blocks, level_max).  level_max is the reference's levelMax of a run on the mesh: one above its top level.
def _generated():
    out = {}

    def add(name, bx, by, base, top, seeds, radius, sprinkle=0.0, seed=0):
        out[name] = (bx, by, balanced_mesh(bx, by, base, top, seeds, radius, sprinkle, seed), top + 1)

    # refined toward the four corners (points just inside them, so that the corner blocks themselves sit at a level jump)
    add("1x1_corners", 1, 1, 1, 6, [(0.1, 0.1), (0.9, 0.1), (0.1, 0.9), (0.9, 0.9)], 0.3)
    # toward a point on each wall
    add("2x1_walls", 2, 1, 1, 5, [(0.7, 0), (2, 0.4), (1.3, 1), (0, 0.6)], 0.8)
    # corners, walls and a few random blocks
    add("1x3_mixed", 1, 3, 1, 5, [(0, 0), (1, 3), (1, 1.5), (0.5, 0)], 0.8, sprinkle=0.04, seed=3)
    # the middle, one corner, one wall
    add("3x2_middle", 3, 2, 1, 5, [(1.5, 1.0), (3, 0), (0, 1.3)], 0.8)
    return out


def _tiny():
    return {"tiny1": (1, 1, uniform_mesh(1, 1), 1), "tiny2": (2, 1, uniform_mesh(2, 1), 1), "tiny3": (3, 1, uniform_mesh(3, 1), 1),
            "tiny5": (1, 2, np.array([(0, 0, 1), (1, 0, 0), (1, 1, 0), (1, 0, 1), (1, 1, 1)], dtype=np.int32), 2)}


# one-level meshes whose block counts sit at the pass boundaries of the device reductions (1024 threads, 4096 blocks a pass)
COUNT_SHAPES = {1023: (1023, 1), 1024: (32, 32), 1025: (25, 41), 4095: (63, 65), 4097: (17, 241)}


def _counts():
    return {"n%d" % n: (bx, by, uniform_mesh(bx, by), 1) for n, (bx, by) in COUNT_SHAPES.items()}


def _large():
    """above two reduction passes of 4096 blocks, with a partial third"""
    return {"large": (2, 1, balanced_mesh(2, 1, 6, 8, [(0.5, 0.5), (2, 1)], 0.12), 9)}


GENERATED = _generated()
TINY = _tiny()
COUNTS = _counts()
LARGE = _large()
ALL = {**GENERATED, **TINY, **COUNTS, **LARGE}


def neighbourhood_classes(blocks, bpdx, bpdy):
    """which of the hard cases a mesh contains: level jumps along each wall, a corner block next to a block of another level,
    diagonal-only coarse-fine contact, a coarse block with finer neighbours on two or more faces"""
    from cup2d_amr_oracle import Mesh
    m = Mesh(blocks, bpdx, bpdy)
    out = set()
    for (l, i, j) in m.blocks:
        NX, NY = bpdx << l, bpdy << l
        st = {}
        for di in (-1, 0, 1):
            for dj in (-1, 0, 1):
                if (di, dj) != (0, 0) and 0 <= i + di < NX and 0 <= j + dj < NY:
                    s = m.state(l, i + di, j + dj)
                    st[(di, dj)] = "same" if s >= 0 else ("coarse" if s == -2 else "fine")
        jump = {c for c, s in st.items() if s != "same"}
        # a coarse-fine face ending on a wall: the neighbour along the wall is at another level
        if i == 0 and {(0, -1), (0, 1)} & jump:
            out.add("jump_on_wall_x-")
        if i == NX - 1 and {(0, -1), (0, 1)} & jump:
            out.add("jump_on_wall_x+")
        if j == 0 and {(-1, 0), (1, 0)} & jump:
            out.add("jump_on_wall_y-")
        if j == NY - 1 and {(-1, 0), (1, 0)} & jump:
            out.add("jump_on_wall_y+")
        # the neighbours of a corner leaf above the base level are its siblings, so the jump there is toward finer blocks
        if (i in (0, NX - 1)) and (j in (0, NY - 1)) and jump:
            out.add("corner_jump_%s%s" % ("x-" if i == 0 else "x+", "y-" if j == 0 else "y+"))
        if jump and all(abs(a) + abs(b) == 2 for a, b in jump):
            out.add("diagonal_only")
        if sum(st.get(c) == "fine" for c in ((-1, 0), (1, 0), (0, -1), (0, 1))) >= 2:
            out.add("fine_on_two_faces")
    out.add("nb_mod4_%d" % (len(blocks) % 4))
    return out
