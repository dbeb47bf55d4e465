"""CPU tests of the host tables of the uniform-grid context (cup2d_plan_create / cup2d_plan_table) on domains of any
bpdx x bpdy and with any block order, on one and several ranks, against a numpy restatement: the halo plan (table 0),
the W, E, S, N neighbour slots (table 3) and the 4x4-block tiles of the advect stage and the three-kernel Krylov
iteration (tables 4 and 5)."""
import ctypes as C

import numpy as np
import pytest

import cup2d_b200
from block_orders import ORDERS, SHAPES, make_order
from cup2d_b200 import lib as L

DIRS = [(-1, 0), (1, 0), (0, -1), (0, 1)]   # W, E, S, N


def plan_tables(nbx, nby, order, rank, nranks):
    lib = cup2d_b200.load_library()
    nglob = len(order)
    base, rem = divmod(nglob, nranks)
    rb = np.concatenate([[0], np.cumsum([base + (1 if r < rem else 0) for r in range(nranks)])]).astype(np.int64)
    cfg = L.Config(nbx, nby, nglob, order.ctypes.data_as(C.POINTER(C.c_int32)), rank, nranks,
                   rb.ctypes.data_as(C.POINTER(C.c_int64)), 1.0 / (8 * max(nbx, nby)), 1e-3, 0.5, -1, 0)
    h = C.c_void_p()
    L.check(lib.cup2d_plan_create(C.byref(cfg), C.byref(h)))

    def table(which):
        n = lib.cup2d_plan_table(h, which, None)
        out = np.empty(n, dtype=np.int32)
        if n:
            lib.cup2d_plan_table(h, which, out.ctypes.data_as(C.POINTER(C.c_int32)))
        return out

    try:
        nloc = int(lib.cup2d_nblocks_local(h))
        return rb, nloc, table(0), table(3).reshape(-1, 4), table(4).reshape(-1, 32), table(5).reshape(-1, 2)
    finally:
        lib.cup2d_destroy(h)


def check_tables(bpdx, bpdy, level, kind, rank, nranks):
    nbx, nby = bpdx << level, bpdy << level
    order = make_order(bpdx, bpdy, level, kind)
    rb, nloc, halo, nbr, tiles, torg = plan_tables(nbx, nby, order, rank, nranks)
    gb, ge = int(rb[rank]), int(rb[rank + 1])
    assert nloc == ge - gb
    gid = np.full((nby, nbx), -1)
    gid[order[:, 1], order[:, 0]] = np.arange(len(order))

    def gid_at(i, j):
        return gid[j, i] if 0 <= i < nbx and 0 <= j < nby else -1

    # halo: the non-local face neighbours of the local blocks, ascending global id
    want_halo = sorted({g for i, j in order[gb:ge] for di, dj in DIRS
                        if (g := gid_at(i + di, j + dj)) >= 0 and not gb <= g < ge})
    assert halo.tolist() == want_halo
    assert (nranks == 1) == (len(halo) == 0)

    def slot_of(g):
        if g < 0:
            return -1
        if gb <= g < ge:
            return g - gb
        return nloc + want_halo.index(g) if g in want_halo else -1

    # nbr equals the face-neighbour table: -1 exactly at the domain walls
    for k, (i, j) in enumerate(order[gb:ge]):
        for d, (di, dj) in enumerate(DIRS):
            inside = 0 <= i + di < nbx and 0 <= j + dj < nby
            assert nbr[k, d] == slot_of(gid_at(i + di, j + dj)) and (nbr[k, d] >= 0) == inside, (k, d)
    # tiles: aligned 4x4 groups holding a local block, in the order the local blocks first meet them
    want_org = []
    for i, j in order[gb:ge]:
        if (4 * (i // 4), 4 * (j // 4)) not in want_org:
            want_org.append((4 * (i // 4), 4 * (j // 4)))
    assert [tuple(t) for t in torg] == want_org
    assert (torg % 4 == 0).all()
    seen = np.zeros(nloc, dtype=int)
    for ts, (i0, j0) in zip(tiles, torg):
        for by in range(4):
            for bx in range(4):
                s = ts[4 * by + bx]
                assert s == slot_of(gid_at(i0 + bx, j0 + by))
                if 0 <= s < nloc:
                    seen[s] += 1
        ring = [(i0 - 1, j0 + k) for k in range(4)] + [(i0 + 4, j0 + k) for k in range(4)] + \
               [(i0 + k, j0 - 1) for k in range(4)] + [(i0 + k, j0 + 4) for k in range(4)]
        for r, (i, j) in enumerate(ring):
            assert ts[16 + r] == slot_of(gid_at(i, j)), (i0, j0, r)
            if nranks == 1:   # every block is local: -1 exactly outside the domain
                assert (ts[16 + r] < 0) == (not (0 <= i < nbx and 0 <= j < nby))
    assert (seen == 1).all()   # every local block is the interior of exactly one tile
    return len(tiles), len(halo)


@pytest.mark.parametrize("kind", ORDERS)
@pytest.mark.parametrize("shape", SHAPES + [(1, 1, 3)], ids=lambda s: f"{s[0]}x{s[1]}L{s[2]}")
def test_tables_single_rank(shape, kind):
    ntiles, _ = check_tables(*shape, kind, 0, 1)
    bpdx, bpdy, level = shape
    assert ntiles == -(-(bpdx << level) // 4) * -(-(bpdy << level) // 4)


@pytest.mark.parametrize("kind", ["hilbert", "row", "random"])
@pytest.mark.parametrize("nranks", [2, 3, 5])
@pytest.mark.parametrize("shape", [(3, 2, 1), (5, 3, 1)], ids=lambda s: f"{s[0]}x{s[1]}L{s[2]}")
def test_tables_several_ranks(shape, kind, nranks):
    """contiguous ranges of the caller's order per rank (uneven for 3 and 5 ranks)"""
    for rank in range(nranks):
        _, nhalo = check_tables(*shape, kind, rank, nranks)
        assert nhalo > 0
