"""CPU tests of the host-side multi-level plan (cup2d_b200/csrc/amr_plan.cpp) on generated meshes (tests/amr_meshes.py): level
jumps at every wall and corner, rectangular domains, every block order.  The Poisson rows and the ghost tables are compared
with the oracle (oracle/cup2d_amr_oracle.py), whose Poisson assembly is first pinned value for value against the COO the
reference itself assembled on its run.sh mesh."""
import os

import numpy as np
import pytest

import amr_meshes as M
import cup2d_amr_oracle as ao
from cup2d_b200.amr import AmrPlan, LAB_SHAPES
from test_amr_plan import apply

CASES = {**M.GENERATED, **M.TINY}
MESH_ORDERS = [(n, o) for n in CASES for o in M.ORDERS]


def _canon(r, c, v):
    """(row, col, val) sorted by (row, col), zeros dropped"""
    r, c, v = np.asarray(r, dtype=np.int64), np.asarray(c, dtype=np.int64), np.asarray(v)
    nz = v != 0
    o = np.lexsort((c[nz], r[nz]))
    return r[nz][o], c[nz][o], v[nz][o]


def plan_matrix(plan):
    """AmrPlan.poisson() as one matrix: the same-level 5-point stencil through the face-neighbour table (Neumann walls: the
    absent neighbour is left out), the general rows where a coarse-fine face is crossed"""
    nbr, rows, rowptr, col, val = plan.poisson()
    nb = len(plan.blocks)
    k, iy, ix = (a.reshape(-1) for a in np.meshgrid(np.arange(nb), np.arange(8), np.arange(8), indexing="ij"))
    r = 64 * k + 8 * iy + ix
    R, C, V = [], [], []
    diag = np.zeros(len(r))
    for face, (dx, dy) in enumerate(ao.FACE_CODES):
        x, y = ix + dx, iy + dy
        inside = (x >= 0) & (x < 8) & (y >= 0) & (y < 8)
        nk = np.where(inside, k, nbr[k, face])
        ok = inside | (nk >= 0)
        R.append(r[ok])
        C.append(64 * nk[ok] + 8 * (y[ok] % 8) + (x[ok] % 8))
        V.append(np.ones(ok.sum()))
        diag -= ok
    R.append(r)
    C.append(r)
    V.append(diag)
    R, C, V = np.concatenate(R), np.concatenate(C), np.concatenate(V)
    keep = ~np.isin(R, rows)
    R, C, V = [R[keep]], [C[keep]], [V[keep]]
    R.append(np.repeat(rows.astype(np.int64), np.diff(rowptr)))
    C.append(col.astype(np.int64))
    V.append(val)
    return _canon(np.concatenate(R), np.concatenate(C), np.concatenate(V))


def test_case_list_covers_the_hard_neighbourhoods():
    """the generated list keeps every class of neighbourhood these tests are there for; a corner leaf above the base level
    only neighbours its siblings, so its level jump is toward finer blocks"""
    seen = set()
    for name, (bx, by, blocks, _) in {**M.GENERATED, **M.TINY}.items():
        seen |= M.neighbourhood_classes(blocks, bx, by)
    for name, (bx, by, blocks, _) in {**M.COUNTS, **M.LARGE}.items():
        seen.add("nb_mod4_%d" % (len(blocks) % 4))
    want = {"jump_on_wall_x-", "jump_on_wall_x+", "jump_on_wall_y-", "jump_on_wall_y+", "corner_jump_x-y-", "corner_jump_x+y-",
            "corner_jump_x-y+", "corner_jump_x+y+", "diagonal_only", "fine_on_two_faces", "nb_mod4_1", "nb_mod4_2", "nb_mod4_3"}
    assert want <= seen, want - seen
    for name, (bx, by, blocks, lmax) in M.GENERATED.items():
        levels = set(blocks[:, 0].tolist())
        assert 4 <= len(levels) <= 5 and 100 <= len(blocks) <= 600, name
        assert max(levels) == lmax - 1
    assert sorted(len(b[2]) for b in M.TINY.values()) == [1, 2, 3, 5]
    assert any(len(set(b[2][:, 0].tolist())) == 2 for b in M.TINY.values())
    assert sorted(len(b[2]) for b in M.COUNTS.values()) == [1023, 1024, 1025, 4095, 4097]
    (bx, by, large, _), = M.LARGE.values()
    assert len(large) > 8192 and len(large) % 4096 != 0 and len(set(large[:, 0].tolist())) > 1
    # the orders are permutations of one another and differ from each other
    for name, (bx, by, blocks, _) in M.GENERATED.items():
        lists = [M.order(blocks, bx, by, o) for o in M.ORDERS]
        assert all(sorted(map(tuple, x.tolist())) == sorted(map(tuple, blocks.tolist())) for x in lists)
        assert len({x.tobytes() for x in lists}) == len(lists)


def test_meshes_are_two_to_one_balanced_across_faces_and_corners():
    for name, (bx, by, blocks, _) in {**M.GENERATED, **M.TINY, **M.LARGE}.items():
        m = ao.Mesh(blocks, bx, by)
        for (l, i, j) in m.blocks:
            for di in (-1, 0, 1):
                for dj in (-1, 0, 1):
                    if 0 <= i + di < bx << l and 0 <= j + dj < by << l:
                        # touching is symmetric: no leaf with a neighbour two levels coarser means none two levels finer
                        if m.state(l, i + di, j + dj) == -2:
                            assert m.state(l - 1, (i + di) // 2, (j + dj) // 2) >= 0, (name, l, i, j, di, dj)


def test_oracle_poisson_assembly_equals_the_reference_coo(golden_dir):
    """the restated assembly loop on the reference's run.sh mesh: the COO its own loop pushed, value for value"""
    d = np.load(os.path.join(golden_dir, "amrlab_lmax8.npz"))
    mesh = ao.Mesh(d["blocks"], int(d["bpdx"]), int(d["bpdy"]))
    r, c, v = ao.amr_poisson_matrix(mesh)
    assert len(set(zip(r.tolist(), c.tolist()))) == len(r)
    got, want = _canon(r, c, v), _canon(d["coo_row"], d["coo_col"], d["coo_val"])
    for a, b in zip(got, want):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("name,order", MESH_ORDERS)
def test_plan_poisson_rows_equal_the_oracle_assembly(name, order):
    bx, by, blocks, _ = CASES[name]
    b = M.order(blocks, bx, by, order)
    plan = AmrPlan(b, bx, by)
    got = plan_matrix(plan)
    plan.close()
    want = _canon(*ao.amr_poisson_matrix(ao.Mesh(b, bx, by)))
    for a, w in zip(got, want):
        assert np.array_equal(a, w)


def test_plan_poisson_rows_on_the_large_mesh():
    (bx, by, blocks, _), = M.LARGE.values()
    b = M.order(blocks, bx, by, "random")
    plan = AmrPlan(b, bx, by)
    got = plan_matrix(plan)
    plan.close()
    want = _canon(*ao.amr_poisson_matrix(ao.Mesh(b, bx, by)))
    for a, w in zip(got, want):
        assert np.array_equal(a, w)


# kind: (stencil, lab kind, field dim) of the oracle's Lab for the plan's table `kind`
LABS = {0: ((-3, -3, 4, 4, True), "vector", 2), 1: ((-1, -1, 2, 2, False), "vector", 2), 2: ((-1, -1, 2, 2, False), "scalar", 1),
        3: ((-4, -4, 5, 5, True), "scalar", 1)}


@pytest.fixture(scope="module")
def oracle_labs():
    """per generated mesh (sorted order) and table kind: a seeded field and the oracle's labs of every block"""
    out = {}
    for name, (bx, by, blocks, _) in CASES.items():
        b = M.order(blocks, bx, by, "sorted")
        mesh = ao.Mesh(b, bx, by)
        rng = np.random.default_rng(len(b))
        for kind, (stencil, lk, dim) in LABS.items():
            f = rng.uniform(-1, 1, (len(b), 8, 8, dim))
            lab = ao.Lab(mesh, f, stencil, lk)
            out[(name, kind)] = (f, np.stack([lab.load(k).copy() for k in range(len(b))]))
    return out


@pytest.mark.parametrize("kind", sorted(LABS))
@pytest.mark.parametrize("name,order", [(n, o) for n in CASES for o in ("sorted", "random")])
def test_plan_ghost_tables_equal_the_oracle_labs(oracle_labs, name, order, kind):
    """the tables applied to a seeded field equal the oracle's labs of the same blocks wherever the oracle writes a cell
    (it leaves NaN where the reference leaves its buffers stale); the plan writes every one of those cells"""
    bx, by, blocks, _ = CASES[name]
    s = M.order(blocks, bx, by, "sorted")
    b = M.order(blocks, bx, by, order)
    perm = np.array([{tuple(x): q for q, x in enumerate(s.tolist())}[tuple(x)] for x in b.tolist()])
    f, want = oracle_labs[(name, kind)]
    plan = AmrPlan(b, bx, by)
    got = apply(plan, kind, f[perm])
    plan.close()
    want = want[perm]
    assert got.shape[1:] == LAB_SHAPES[kind]
    ref = ~np.isnan(want)
    assert not np.isnan(got[ref]).any()
    assert np.abs(got[ref] - want[ref]).max() <= 1e-13 * np.abs(want[ref]).max()
