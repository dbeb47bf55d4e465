"""GPU tests of adapt() in one call (cup2d_amr_adapt, csrc/amr_regrid.cu): the refine / compress decision and the order of the
new block list on the device must equal the host decision (cup2d_amr_adapt_mesh) array for array, and the regridded context
must hold bitwise the fields of the composed path (cup2d_amr_adapt_tags -> cup2d_amr_adapt_mesh -> cup2d_amr_regrid) on an
identical context.  Meshes: the reference's run.sh mesh (tests/golden/amrregrid_lmax8.npz), the generated meshes of
tests/amr_meshes.py in every block order, synthetic three-level meshes with per-group tags, and small meshes whose tags hit
each rule of the decision.  They also pass on the CPU against the emulated build of the same sources
(tests/test_amr_adapt_emulation.py)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import amr_meshes as M

pytestmark = [pytest.mark.gpu]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = ("vel", "vold", "pres", "pold", "chi", "tmp", "tmpV")


@pytest.fixture(scope="module")
def g(golden_dir):
    sys.path.insert(0, golden_dir)
    import make_regrid_golden
    return make_regrid_golden.load(os.path.join(golden_dir, "amrregrid_lmax8.npz"))


def _sim(blocks, bpdx, bpdy, h0=1 / 8, fields=None):
    from cup2d_b200.amr import AmrSimulation
    sim = AmrSimulation(blocks, bpdx, bpdy, h0, 4e-5)
    for n, a in (fields or {}).items():
        sim.upload(n, a)
    return sim


def _fields(nb, seed):
    rng = np.random.default_rng(seed)
    v = lambda: rng.uniform(-1, 1, (nb, 8, 8, 2))
    s = lambda: rng.uniform(-1, 1, (nb, 8, 8, 1))
    return {"vel": v(), "vold": v(), "tmpV": v(), "pres": s(), "pold": s(), "chi": rng.uniform(0, 1, (nb, 8, 8, 1)), "tmp": s()}


def _device_list(blocks, bx, by, lmax, linf, rtol, ctol):
    """the new list of cup2d_amr_adapt with the caller's tags, and whether it reported a change"""
    sim = _sim(blocks, bx, by)
    changed = sim.adapt(rtol, ctol, lmax, block_linf=linf)
    n = sim.lib.cup2d_amr_blocks(sim._h, None)
    got = sim.blocks.copy()
    sim.close()
    assert n == len(got)
    return got, changed


def _check_decision(blocks, bx, by, lmax, linf, rtol, ctol):
    from cup2d_b200.amr import adapt_mesh
    want = adapt_mesh(blocks, bx, by, lmax, linf, rtol, ctol)
    got, changed = _device_list(blocks, bx, by, lmax, linf, rtol, ctol)
    assert np.array_equal(got, want)
    assert changed == (not np.array_equal(want, blocks))
    return want


def _kinds(old, new):
    """(refined parents, compressed groups) of the step old -> new"""
    o = {tuple(b) for b in np.asarray(old).tolist()}
    nl = np.asarray(new).tolist()
    return (sum((l - 1, i // 2, j // 2) in o for l, i, j in nl) // 4,
            sum((l + 1, 2 * i, 2 * j) in o for l, i, j in nl))


# ---- the decision against the host ----------------------------------------------------------------------------------------

def test_decision_on_the_reference_mesh_with_recorded_and_device_tags(g):
    bx, by, lmax = int(g["bpdx"]), int(g["bpdy"]), int(g["level_max"])
    rtol, ctol = float(g["rtol"]), float(g["ctol"])
    want = _check_decision(g["blocks"], bx, by, lmax, g["block_linf"], rtol, ctol)
    assert np.array_equal(want, g["new_blocks"])
    # the device's own tags: the same list as the host decision on the downloaded tags of an identical context
    from cup2d_b200.amr import adapt_mesh
    f = {n: g[n] for n in ("vel", "vold", "pres", "pold", "chi")}
    a, b = _sim(g["blocks"], bx, by, float(g["h0"]), f), _sim(g["blocks"], bx, by, float(g["h0"]), f)
    host = adapt_mesh(g["blocks"], bx, by, lmax, a.adapt_tags(rtol, lmax), rtol, ctol)
    assert b.adapt(rtol, ctol, lmax)
    assert np.array_equal(b.blocks, host) and np.array_equal(b.blocks, g["new_blocks"])
    a.close()
    b.close()


@pytest.mark.parametrize("order", M.ORDERS)
@pytest.mark.parametrize("name", list(M.GENERATED) + list(M.TINY))
def test_decision_on_generated_meshes(name, order):
    """every generated mesh (1x1, 2x1, 1x3, 3x2 domains; 1, 2, 3 and 5 blocks) in every order, a few seeded tag vectors with
    one level of headroom above the mesh's top"""
    bx, by, blocks, lmax = {**M.GENERATED, **M.TINY}[name]
    b = M.order(blocks, bx, by, order)
    lmax = max(lmax, int(b[:, 0].max()) + 1) + 1
    rng = np.random.default_rng(len(b))
    changed = 0
    for t in range(3):
        linf = rng.uniform(0, 1, len(b))
        rtol, ctol = (0.8, 0.3) if t < 2 else (2.0, 0.6)
        want = _check_decision(b, bx, by, lmax, linf, rtol, ctol)
        changed += not np.array_equal(want, b)
    assert changed > 0


@pytest.mark.parametrize("base,centre", [(3, (0.45, 0.55)), (4, (0.7, 0.3)), (3, (0.1, 0.9))])
def test_decision_on_three_level_meshes_with_group_tags(base, centre):
    """one tag per sibling group, so that whole groups compress; the library's order and a shuffled one"""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import bench_amr
    blocks = bench_amr.three_level_mesh(base, r1=0.3, r2=0.15, centre=centre)
    lmax = base + 3
    rng = np.random.default_rng(base)
    ncomp = nref = 0
    for b in (blocks, blocks[rng.permutation(len(blocks))]):
        for _ in range(3):
            groups = {}
            for l, i, j in b.tolist():
                groups.setdefault((l, i // 2, j // 2), rng.uniform(0, 1))
            linf = np.array([groups[(l, i // 2, j // 2)] for l, i, j in b.tolist()])
            want = _check_decision(b, 1, 1, lmax, linf, 0.7, 0.35)
            r, c = _kinds(b, want)
            nref, ncomp = nref + r, ncomp + c
    assert nref > 0 and ncomp > 0


def _two_level():
    """level 1 on the unit square with (1, 0, 0) refined: three coarse blocks and four fine ones"""
    return np.array([(2, 0, 0), (2, 1, 0), (2, 0, 1), (2, 1, 1), (1, 1, 0), (1, 0, 1), (1, 1, 1)], dtype=np.int32)


def test_decision_rules_one_by_one():
    """tags that hit each rule of the decision; every case also against the host decision"""
    u2 = M.reference_order(M.uniform_mesh(1, 1, 2), 1, 1, 4)   # 16 blocks of level 2 in the reference's order
    at = {tuple(b): k for k, b in enumerate(u2.tolist())}
    # Refine at level_max - 1 is dropped: nothing changes
    got, changed = _device_list(u2, 1, 1, 3, np.ones(16), 0.5, 0.1)
    assert not changed and np.array_equal(got, u2)
    assert np.array_equal(_check_decision(u2, 1, 1, 3, np.ones(16), 0.5, 0.1), u2)
    # Compress at level 0 is dropped: nothing changes
    u0 = M.reference_order(M.uniform_mesh(2, 1, 0), 2, 1, 3)
    assert np.array_equal(_check_decision(u0, 2, 1, 3, np.zeros(2), 0.5, 0.1), u0)
    # a finer neighbour that refines turns a coarse Compress into Refine
    b = _two_level()
    linf = np.array([0.3, 1.0, 0.3, 0.3, 0.0, 0.0, 0.0])
    newset = {tuple(x) for x in _check_decision(b, 1, 1, 4, linf, 0.5, 0.1).tolist()}
    assert (3, 2, 0) in newset and (2, 2, 0) in newset and (1, 0, 1) in newset
    # a same-level Refine vetoes a Compress, and with it the whole group's
    linf = np.full(16, 0.3)
    for i in (2, 3):
        for j in (2, 3):
            linf[at[(2, i, j)]] = 0.0
    linf[at[(2, 1, 2)]] = 1.0
    assert _kinds(u2, _check_decision(u2, 1, 1, 4, linf, 0.5, 0.1)) == (1, 0)
    linf[at[(2, 1, 2)]] = 0.3   # without the Refine the group compresses
    assert _kinds(u2, _check_decision(u2, 1, 1, 4, linf, 0.5, 0.1)) == (0, 1)
    # three of four siblings compressing: none does
    linf[at[(2, 3, 3)]] = 0.3
    assert np.array_equal(_check_decision(u2, 1, 1, 4, linf, 0.5, 0.1), u2)
    # nothing changes: a no-op; in another order the new list is the old one in the reference's order
    got, changed = _device_list(u2, 1, 1, 4, np.full(16, 0.3), 0.5, 0.1)
    assert not changed and np.array_equal(got, u2)
    assert np.array_equal(_check_decision(u2[::-1].copy(), 1, 1, 4, np.full(16, 0.3), 0.5, 0.1), u2)


def test_rectangular_and_non_power_of_two_domains():
    """domains whose curve skips positions outside them (regular = false) and square ones (regular = true)"""
    for bx, by in ((3, 1), (1, 3), (5, 3), (3, 2), (4, 4), (2, 2), (6, 1)):
        for L in (0, 1):
            b = M.uniform_mesh(bx, by, L)
            rng = np.random.default_rng(bx * 10 + by + L)
            for _ in range(2):
                groups = {}
                for l, i, j in b.tolist():
                    groups.setdefault((l, i // 2, j // 2), rng.uniform(0, 1))
                linf = np.array([groups[(l, i // 2, j // 2)] for l, i, j in b.tolist()])
                _check_decision(M.order(b, bx, by, "random"), bx, by, 4, linf, 0.6, 0.4)


# ---- the fields against the composed path ---------------------------------------------------------------------------------

def _same_as_composed(blocks, bx, by, h0, lmax, rtol, ctol, linf, seed, fast_steps=True):
    from cup2d_b200.amr import adapt_mesh
    f = _fields(len(blocks), seed)
    a, b = _sim(blocks, bx, by, h0, f), _sim(blocks, bx, by, h0, f)
    tags = a.adapt_tags(rtol, lmax) if linf is None else linf
    new = adapt_mesh(blocks, bx, by, lmax, tags, rtol, ctol)
    a.regrid(new)
    assert b.adapt(rtol, ctol, lmax, block_linf=linf)
    assert np.array_equal(b.blocks, new) and np.array_equal(a.blocks, new)
    for n in FIELDS:
        assert np.array_equal(a.download(n), b.download(n)), n
    if fast_steps:
        for fast in (False, True):
            a.set_fast(fast)
            b.set_fast(fast)
            ra, rb = a.step(cfl=0.5, max_iter=3), b.step(cfl=0.5, max_iter=3)
            assert ra == rb
            for n in ("vel", "pres", "tmp"):
                assert np.array_equal(a.download(n), b.download(n)), (fast, n)
    a.close()
    b.close()
    return new


def test_fields_equal_the_composed_path_on_the_reference_mesh(g):
    """device tags (tmp holds the tagging field on both sides) and recorded tags"""
    bx, by, h0, lmax = int(g["bpdx"]), int(g["bpdy"]), float(g["h0"]), int(g["level_max"])
    _same_as_composed(g["blocks"], bx, by, h0, lmax, float(g["rtol"]), float(g["ctol"]), None, 1)
    new = _same_as_composed(g["blocks"], bx, by, h0, lmax, float(g["rtol"]), float(g["ctol"]), g["block_linf"], 2, False)
    assert np.array_equal(new, g["new_blocks"])


@pytest.mark.parametrize("base", [3, 4])
def test_fields_equal_the_composed_path_with_compression(base):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import bench_amr
    blocks = bench_amr.three_level_mesh(base, r1=0.3, r2=0.15, centre=(0.45, 0.55))
    rng = np.random.default_rng(base + 10)
    groups = {}
    for l, i, j in blocks.tolist():
        groups.setdefault((l, i // 2, j // 2), rng.uniform(0, 1))
    linf = np.array([groups[(l, i // 2, j // 2)] for l, i, j in blocks.tolist()])
    new = _same_as_composed(blocks, 1, 1, 1 / 8, base + 3, 0.7, 0.35, linf, base)
    r, c = _kinds(blocks, new)
    assert r > 0 and c > 0


# ---- errors ---------------------------------------------------------------------------------------------------------------

def test_errors_leave_the_context_untouched(g):
    from cup2d_b200 import lib as L
    bx, by, lmax = int(g["bpdx"]), int(g["bpdy"]), int(g["level_max"])
    f = _fields(len(g["blocks"]), 5)
    sim = _sim(g["blocks"], bx, by, float(g["h0"]), f)
    lib = sim.lib
    top = int(g["blocks"][:, 0].max())
    for bad in (0, -1, 21, top, top - 1):    # outside 1..20, or a block at or above level_max
        assert lib.cup2d_amr_adapt(sim._h, None, float(g["rtol"]), float(g["ctol"]), bad, None, None) == -1
        assert b"cup2d_amr_adapt" in lib.cup2d_last_error()
    assert lib.cup2d_amr_adapt(None, None, 1.0, 0.1, lmax, None, None) == -1
    for n in FIELDS:
        assert np.array_equal(sim.download(n), f[n]), n
    assert np.array_equal(sim.block_list(), g["blocks"])
    assert sim.adapt(float(g["rtol"]), float(g["ctol"]), lmax, block_linf=g["block_linf"])   # still usable
    rb = np.array([0, len(sim.blocks) // 2, len(sim.blocks)], dtype=np.int64)
    L.check(lib.cup2d_amr_set_ranks(sim._h, 0, 2, rb.ctypes.data_as(C.POINTER(C.c_int64))))
    assert lib.cup2d_amr_adapt(sim._h, None, float(g["rtol"]), float(g["ctol"]), lmax, None, None) == -4
    sim.close()
