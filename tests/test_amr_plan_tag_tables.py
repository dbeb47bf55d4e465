"""The tables the fused tagging kernel (amr_tags_fast_kernel, csrc/amr_fast.cu) reads give the labs of the full per-cell
tables that the baseline tagging gathers, term for term, so that both paths compute the same bits:
  - the compact ghost rows of kinds 1 (+-1 velocity lab) and 3 (16 x 16 chi lab) hold the terms of the full rows of the same
    lab cells.  The full rows list them in ascending (block, cell) order; the compact rows in the order of the block their
    pattern was made from, which differs on meshes in the reference's order.  With each row's terms put in ascending
    (block, cell) order, as the tagging kernel's tables hold them (amr_ghost_rows with source_order), they are the full
    rows: the same counts, sources and weights in the same order;
  - every other lab cell the kernel reads is, in the full table, a single term of weight 1 at the cell the kernel reads
    directly (own cells; same-level neighbours of the 8-neighbour table; the scalar wall clamp), and the ghost cells of an
    irregular block that the compact table leaves out have empty full rows (0, which never fires the chi rule).
On the run.sh tagging mesh, a synthetic mesh of a few thousand blocks and the generated meshes of tests/amr_meshes.py."""
import os

import numpy as np
import pytest

import amr_meshes as M
from cup2d_b200.amr import LAB_SHAPES, AmrPlan
from test_amr_plan import balanced_disc_mesh


def _meshes():
    out = {"disc_4_8": (1, 1, balanced_disc_mesh(4, 8))}
    d = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "amrtags_lmax8.npz"))
    out["runsh_tags"] = (int(d["bpdx"]), int(d["bpdy"]), d["blocks"])
    for name, (bx, by, blocks, lmax) in M.GENERATED.items():
        out[name] = (bx, by, M.reference_order(blocks, bx, by, lmax))
    return out


MESHES = _meshes()


def _full_rows_of_compact(plan, which, irr):
    ny, nx, dim = LAB_SHAPES[which]
    ncell = ny * nx * dim
    rp, dst, sb, sc, w = plan.ghosts(which)
    frp, fsb, fsc, fw = plan.stencil(which)
    q, rem = np.divmod(dst.astype(np.int64), ncell)
    rows = irr[q].astype(np.int64) * ncell + rem
    return (rp, sb, sc, w), (frp, fsb, fsc, fw), rows


def _clamp_source(n8, k, gx, gy):
    """(block, cell) the kernel reads for lab cell (gx, gy) of regular block k: fo_labs' scalar wall clamp"""
    ox = -1 if gx < 0 else int(gx > 7)
    oy = -1 if gy < 0 else int(gy > 7)
    wx = ox != 0 and n8[k, 3 if ox < 0 else 4] == -1
    wy = oy != 0 and n8[k, 1 if oy < 0 else 6] == -1
    cx = (0 if ox < 0 else 7) if wx else gx
    cy = (0 if oy < 0 else 7) if wy else gy
    qx = -1 if cx < 0 else int(cx > 7)
    qy = -1 if cy < 0 else int(cy > 7)
    if qx == 0 and qy == 0:
        return k, cy * 8 + cx
    c = (qy + 1) * 3 + (qx + 1)
    return int(n8[k, c - (c > 4)]), (cy & 7) * 8 + (cx & 7)


@pytest.mark.parametrize("which", [1, 3])
@pytest.mark.parametrize("name", list(MESHES))
def test_compact_rows_are_the_full_rows_term_for_term(name, which):
    bx, by, blocks = MESHES[name]
    plan = AmrPlan(blocks, bx, by)
    irr = plan.irregular()
    (rp, sb, sc, w), (frp, fsb, fsc, fw), rows = _full_rows_of_compact(plan, which, irr)
    plan.close()
    assert len(rows) > 0 and len(np.unique(rows)) == len(rows)
    assert np.array_equal(np.diff(rp), frp[rows + 1] - frp[rows])
    dim = LAB_SHAPES[which][2]
    row_of = lambda ptr: np.repeat(np.arange(len(ptr) - 1), np.diff(ptr))
    fkey = fsb.astype(np.int64) * 64 * dim + fsc
    frow = row_of(frp)
    assert np.all((np.diff(fkey) > 0) | (np.diff(frow) != 0))          # full rows: ascending sources
    o = np.lexsort((sb.astype(np.int64) * 64 * dim + sc, row_of(rp)))  # compact rows, each in ascending source order
    take = np.concatenate([np.arange(frp[r], frp[r + 1]) for r in rows])
    assert len(take) == len(w)
    assert np.array_equal(sb[o], fsb[take]) and np.array_equal(sc[o], fsc[take]) and np.array_equal(w[o], fw[take])


@pytest.mark.parametrize("name", list(MESHES))
def test_direct_reads_are_single_unit_terms(name):
    bx, by, blocks = MESHES[name]
    plan = AmrPlan(blocks, bx, by)
    irr = plan.irregular()
    n8 = plan.neighbours()
    nb = len(blocks)
    is_irr = np.zeros(nb, dtype=bool)
    is_irr[irr] = True
    checked = 0
    for which in (1, 3):
        ny, nx, dim = LAB_SHAPES[which]
        g = (ny - 8) // 2 if which == 1 else 4
        _, (frp, fsb, fsc, fw), rows = _full_rows_of_compact(plan, which, irr)
        in_compact = np.zeros(len(frp) - 1, dtype=bool)
        in_compact[rows] = True
        cnt = np.diff(frp)

        def row(k, gx, gy, d):
            return ((k * ny + gy + g) * nx + gx + g) * dim + d

        def single(r, blk, cc):
            e = frp[r]
            return cnt[r] == 1 and fsb[e] == blk and fsc[e] == cc and fw[e] == 1.0

        # own cells of every block
        for k in range(nb):
            for c in range(64):
                for d in range(dim):
                    assert single(row(k, c & 7, c >> 3, d), k, c * dim + d), (which, k, c, d)
        if which == 1:
            # the cells the vorticity reads: u on the y faces, v on the x faces; direct loads where the compact rows are absent
            faces = [(t, -1, 0, 1) for t in range(8)] + [(t, 8, 0, 6) for t in range(8)]
            faces += [(-1, t, 1, 3) for t in range(8)] + [(8, t, 1, 4) for t in range(8)]
            for k in range(nb):
                for gx, gy, d, slot in faces:
                    r = row(k, gx, gy, d)
                    if in_compact[r]:
                        continue
                    nbf = n8[k, slot]
                    assert nbf >= -1, (k, gx, gy)       # a level jump is always in the compact rows
                    blk = k if nbf == -1 else int(nbf)
                    sx, sy = (gx & 7, gy) if slot in (3, 4) else (gx, gy & 7)
                    if nbf == -1:
                        sx, sy = min(max(gx, 0), 7), min(max(gy, 0), 7)
                    assert single(r, blk, (sy * 8 + sx) * 2 + d), (k, gx, gy, d)
                    checked += 1
        else:
            for k in range(nb):
                for gy in range(-4, 12):
                    for gx in range(-4, 12):
                        if 0 <= gx < 8 and 0 <= gy < 8:
                            continue
                        r = row(k, gx, gy, 0)
                        if is_irr[k]:
                            assert in_compact[r] or cnt[r] == 0, (k, gx, gy)
                        else:
                            assert not in_compact[r]
                            blk, cc = _clamp_source(n8, k, gx, gy)
                            assert blk >= 0 and single(r, blk, cc), (k, gx, gy)
                            checked += 1
    plan.close()
    assert checked > 0
