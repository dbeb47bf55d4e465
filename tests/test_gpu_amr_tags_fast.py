"""GPU tests of adapt()'s tagging on the fused kernel (amr_tags_fast_kernel, csrc/amr_fast.cu), which fast and distributed
contexts run instead of gathering both labs through the full per-cell tables: the same fields in a baseline context and a
fast one must give bitwise the same per-block L-inf and tagging field (tmp).  Meshes: the reference's run.sh mesh, the
generated meshes of tests/amr_meshes.py in every block order, the tiny and block-count meshes, synthetic three-level meshes
(also against the oracle), chi placed so that the rule fires only through ghost cells, chi = 0, finest and non-finest
levels.  Also cup2d_amr_adapt, tag -> adapt -> tag, tagging between enqueued steps and a one-rank distributed context.
They also pass on the CPU against the emulated build of the same sources (tests/test_amr_tags_fast_emulation.py)."""
import os
import sys

import numpy as np
import pytest

import amr_meshes as M

pytestmark = [pytest.mark.gpu]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H0, NU = 1 / 8, 4e-5


def _sim(blocks, bx, by, h0=H0, fast=False):
    from cup2d_b200.amr import AmrSimulation
    sim = AmrSimulation(blocks, bx, by, h0, NU)
    sim.set_fast(fast)
    return sim


def _tags(blocks, bx, by, vel, chi, rtol, lmax, fast, h0=H0):
    sim = _sim(blocks, bx, by, h0, fast)
    sim.upload("vel", vel)
    sim.upload("chi", chi)
    linf = sim.adapt_tags(rtol, lmax)
    tmp = sim.download("tmp")
    sim.close()
    return linf, tmp


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _same(blocks, bx, by, vel, chi, rtol, lmax, h0=H0):
    """baseline and fast tagging: bitwise equal; returns the L-inf"""
    lb, tb = _tags(blocks, bx, by, vel, chi, rtol, lmax, False, h0)
    lf, tf = _tags(blocks, bx, by, vel, chi, rtol, lmax, True, h0)
    assert np.array_equal(_bits(lb), _bits(lf)), np.flatnonzero(lb != lf)[:10]
    assert np.array_equal(_bits(tb), _bits(tf))
    return lb


def _fields(nb, seed, chi_density=0.02):
    """velocity of order 1, chi positive in a few scattered cells"""
    rng = np.random.default_rng(seed)
    vel = rng.uniform(-1, 1, (nb, 8, 8, 2))
    chi = np.where(rng.uniform(0, 1, (nb, 8, 8, 1)) < chi_density, rng.uniform(0.01, 1, (nb, 8, 8, 1)), 0.0)
    return vel, chi


def _rtol(vel, blocks, h0=H0):
    """a threshold inside the vorticity range, so that some blocks refine on vorticity alone and others do not"""
    h = h0 / (1 << blocks[:, 0].astype(np.int64))
    return 0.5 / h.min() * 0.6


def test_runsh_golden(golden_dir):
    """the reference's run.sh mesh with its two fish: fast bitwise the baseline, the chi rule on the reference's 80 blocks,
    the same refine / compress sets"""
    d = np.load(os.path.join(golden_dir, "amrtags_lmax8.npz"))
    blocks, nb, rtol, ctol = d["blocks"], len(d["blocks"]), float(d["rtol"]), float(d["ctol"])
    lmax, bx, by, h0 = int(d["level_max"]), int(d["bpdx"]), int(d["bpdy"]), float(d["h0"])
    lb, tb = _tags(blocks, bx, by, d["vel"], d["chi"], rtol, lmax, False, h0)
    sim = _sim(blocks, bx, by, h0, True)
    sim.upload("vel", d["vel"])
    sim.upload("chi", d["chi"])
    for _ in range(2):   # the second call reuses the tables of the first
        lf = sim.adapt_tags(rtol, lmax)
        tf = sim.download("tmp")
        assert np.array_equal(_bits(lb), _bits(lf)) and np.array_equal(_bits(tb), _bits(tf))
    sim.close()
    want = d["tagfield"]
    field = tf.reshape(nb, 8, 8)
    fired = (d["vort"] != want).reshape(nb, -1).any(axis=1)
    assert fired.sum() == 80
    assert np.array_equal(field.reshape(nb, 64)[fired][:, [27, 28, 35, 36]], np.full((fired.sum(), 4), 2 * rtol))
    wl = np.abs(want).reshape(nb, -1).max(axis=1)
    assert np.array_equal(lf > rtol, wl > rtol) and np.array_equal(lf < ctol, wl < ctol)


@pytest.mark.parametrize("order", M.ORDERS)
@pytest.mark.parametrize("name", list(M.GENERATED))
def test_generated_meshes_every_order(name, order):
    bx, by, blocks, lmax = M.GENERATED[name]
    b = M.order(blocks, bx, by, order)
    vel, chi = _fields(len(b), len(b))
    rtol = _rtol(vel, b)
    for lm in (lmax, lmax + 1):   # the top level finest (offset 4 there), then no block finest (offset 2 everywhere)
        linf = _same(b, bx, by, vel, chi, rtol, lm)
        assert (linf == 2 * rtol).any() or lm > lmax
    _same(b, bx, by, vel, 0 * chi, rtol, lmax)


@pytest.mark.parametrize("name", list(M.TINY) + list(M.COUNTS))
def test_tiny_and_count_meshes(name):
    bx, by, blocks, lmax = {**M.TINY, **M.COUNTS}[name]
    vel, chi = _fields(len(blocks), 7 + len(blocks), 0.01)
    _same(blocks, bx, by, vel, chi, 1.0, lmax)
    _same(blocks, bx, by, vel, 0 * chi, 1.0, lmax)


@pytest.mark.parametrize("base", [3, 4, 5])
def test_three_level_meshes_and_the_oracle(base):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import bench_amr
    import cup2d_amr_oracle as ao
    blocks = bench_amr.three_level_mesh(base, r1=0.3, r2=0.15, centre=(0.45, 0.55))
    vel, chi = _fields(len(blocks), base, 0.005)
    rtol, lmax = _rtol(vel, blocks), base + 3
    linf = _same(blocks, 1, 1, vel, chi, rtol, lmax)
    want, wl = ao.amr_adapt_tags(ao.Mesh(blocks, 1, 1), H0, vel, chi, rtol, lmax)
    _, tf = _tags(blocks, 1, 1, vel, chi, rtol, lmax, True)
    assert np.abs(tf.reshape(want.shape) - want).max() <= 1e-12 * np.abs(want).max()
    assert np.abs(linf - wl).max() <= 1e-12 * wl.max()
    assert np.array_equal(linf > rtol, wl > rtol)


def _ghost_cases():
    """(name, blocks, bx, by, target block, source block, source cell, level_max): chi = 1 in that one cell, which lies in the
    target's {-4,-4,5,5} chi lab at distance 1 from the block (inside the window at every level) but not in the block"""
    from cup2d_b200.amr import AmrPlan
    out = []
    meshes = [("1x1_corners",) + M.GENERATED["1x1_corners"], ("2x1_walls",) + M.GENERATED["2x1_walls"]]
    for mname, bx, by, blocks, lmax in meshes:
        b = M.reference_order(blocks, bx, by, lmax)
        plan = AmrPlan(b, bx, by)
        n8 = plan.neighbours()
        frp, fsb, fsc, fw = plan.stencil(3)
        plan.close()
        found = {}
        for k in range(len(b)):
            walls = n8[k, [3, 4, 1, 6]] == -1
            for gy in range(-1, 9):
                for gx in range(-1, 9):
                    if 0 <= gx < 8 and 0 <= gy < 8:
                        continue
                    r = (k * 16 + gy + 4) * 16 + gx + 4
                    terms = [(int(fsb[e]), int(fsc[e])) for e in range(frp[r], frp[r + 1]) if fw[e] > 0 and fsb[e] != k]
                    if not terms:
                        continue
                    src = terms[0]
                    diag = gx in (-1, 8) and gy in (-1, 8)
                    kinds = []
                    if b[src[0], 0] != b[k, 0]:
                        kinds.append("level_jump")
                    if walls.any() and ((gx < 0 and walls[0]) or (gx > 7 and walls[1]) or (gy < 0 and walls[2]) or (gy > 7 and walls[3])):
                        kinds.append("wall")
                    if walls[:2].any() and walls[2:].any():
                        kinds.append("corner")
                    if diag and src[0] == n8[k, (0 if gx < 0 else 2) + (0 if gy < 0 else 5)] and src[0] not in n8[k, [1, 3, 4, 6]]:
                        kinds.append("diagonal_only")
                    for kind in kinds:
                        found.setdefault(kind, (k, src[0], src[1]))
        for kind, (k, sb, sc) in sorted(found.items()):
            out.append(pytest.param(b, bx, by, k, sb, sc, lmax, id=f"{mname}-{kind}"))
    return out


@pytest.mark.parametrize("blocks,bx,by,k,sb,sc,lmax", _ghost_cases())
def test_the_rule_fires_through_ghost_cells_only(blocks, bx, by, k, sb, sc, lmax):
    nb = len(blocks)
    rng = np.random.default_rng(k)
    vel = 1e-3 * rng.uniform(-1, 1, (nb, 8, 8, 2))   # vorticity far below rtol: only the chi rule reaches it
    chi = np.zeros((nb, 8, 8, 1))
    chi[sb, sc // 8, sc % 8, 0] = 1.0
    rtol = 10.0
    for lm in (lmax, lmax + 1):
        linf = _same(blocks, bx, by, vel, chi, rtol, lm)
        assert linf[k] == 2 * rtol and linf[sb] == 2 * rtol


def test_adapt_on_a_fast_context_equals_the_baseline():
    """cup2d_amr_adapt with its own tags; then tag -> adapt -> tag, the second tagging on the tables of the new mesh"""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import bench_amr
    blocks = M.reference_order(bench_amr.three_level_mesh(3, r1=0.3, r2=0.15, centre=(0.45, 0.55)), 1, 1, 6)
    nb = len(blocks)
    rng = np.random.default_rng(11)
    f = {"vel": rng.uniform(-1, 1, (nb, 8, 8, 2)), "vold": rng.uniform(-1, 1, (nb, 8, 8, 2)), "pres": rng.uniform(-1, 1, (nb, 8, 8, 1)),
         "pold": rng.uniform(-1, 1, (nb, 8, 8, 1)), "chi": np.where(rng.uniform(0, 1, (nb, 8, 8, 1)) < 0.01, 1.0, 0.0)}
    rtol, ctol, lmax = _rtol(f["vel"], blocks), 1.0, 6
    sims = [_sim(blocks, 1, 1, fast=fast) for fast in (False, True)]
    for s in sims:
        for n, a in f.items():
            s.upload(n, a)
    for it in range(2):
        ch = [s.adapt(rtol, ctol, lmax) for s in sims]
        assert ch[0] == ch[1] and (ch[0] or it > 0)
        assert np.array_equal(sims[0].blocks, sims[1].blocks)
        for n in ("tmp", "chi", "vel", "vold", "pres", "pold"):
            assert np.array_equal(_bits(sims[0].download(n)), _bits(sims[1].download(n))), n
        la, lb = (s.adapt_tags(rtol, lmax) for s in sims)
        assert np.array_equal(_bits(la), _bits(lb))
        assert np.array_equal(_bits(sims[0].download("tmp")), _bits(sims[1].download("tmp")))
    # the fast context's tables are the new mesh's: a fresh baseline context on it tags the same
    cur = sims[1].blocks.copy()
    vel, chi = sims[1].download("vel"), sims[1].download("chi")
    lf = sims[1].adapt_tags(rtol, lmax)
    lb, _ = _tags(cur, 1, 1, vel, chi, rtol, lmax, False)
    assert np.array_equal(_bits(lf), _bits(lb))
    for s in sims:
        s.close()


def test_tagging_between_enqueued_steps():
    bx, by, blocks, lmax = M.GENERATED["2x1_walls"]
    b = M.reference_order(blocks, bx, by, lmax)
    vel, chi = _fields(len(b), 5)
    rtol = _rtol(vel, b)
    sim = _sim(b, bx, by, fast=True)
    sim.upload("vel", vel)
    sim.upload("chi", chi)
    for _ in range(3):
        v, c = sim.download("vel"), sim.download("chi")
        lf, tf = sim.adapt_tags(rtol, lmax), sim.download("tmp")
        lb, tb = _tags(b, bx, by, v, c, rtol, lmax, False)
        assert np.array_equal(_bits(lf), _bits(lb)) and np.array_equal(_bits(tf), _bits(tb))
        sim.step_enqueue(cfl=0.5, max_iter=3)
        sim.step_result()
    sim.close()


def test_one_rank_distributed_context_equals_the_plain_one(golden_dir):
    from cup2d_b200.amr import AmrSimulation
    d = np.load(os.path.join(golden_dir, "amrtags_lmax8.npz"))
    blocks, rtol, lmax = d["blocks"], float(d["rtol"]), int(d["level_max"])
    bx, by, h0 = int(d["bpdx"]), int(d["bpdy"]), float(d["h0"])
    lb, tb = _tags(blocks, bx, by, d["vel"], d["chi"], rtol, lmax, False, h0)
    sim = AmrSimulation.distributed(blocks, bx, by, h0, NU, 0, np.array([0, len(blocks)], dtype=np.int64), None)
    sim.upload("vel", d["vel"])
    sim.upload("chi", d["chi"])
    lf = sim.adapt_tags(rtol, lmax)
    assert np.array_equal(_bits(lf), _bits(lb)) and np.array_equal(_bits(sim.download("tmp")), _bits(tb))
    sim.close()
