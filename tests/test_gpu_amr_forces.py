"""Device tests of cup2d_amr_surface / _surface_get / _forces (csrc/amr_forces.cu): the reference's own surface normals and
force diagnostics (tests/golden/amrforces_lmax8.npz), the chain after cup2d_amr_ongrid, synthetic three-level meshes against
the oracle (tests/amr_forces_oracle.py), repeated calls, state and error paths.  Bitwise where the labs involved are plain
copies; elsewhere the labs come from the plan's ghost rows and the results agree to 1e-12 (relative to the largest |value| for
per-point values, to the sum of |terms| for sums)."""
import os
import sys

import numpy as np
import pytest

import amr_body_oracle as bo
import amr_forces_oracle as fo

pytestmark = [pytest.mark.gpu]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NU = 4e-5


@pytest.fixture(scope="module")
def steps(golden_dir):
    sys.path.insert(0, golden_dir)
    import make_forces_golden
    return make_forces_golden.load(os.path.join(golden_dir, "amrforces_lmax8.npz"))


def _sim(blocks, bpdx, bpdy, h0, nu=NU):
    from cup2d_b200.amr import AmrSimulation
    return AmrSimulation(blocks, bpdx, bpdy, h0, nu)


def _copy_only(blocks, bpdx, bpdy, kind):
    """blocks whose lab of stencil kind `kind` is plain copies (wall negations included): bitwise the reference's"""
    from cup2d_b200.amr import AmrPlan, LAB_SHAPES
    p = AmrPlan(blocks, bpdx, bpdy)
    rowptr, _, _, w = p.stencil(kind)
    p.close()
    n = np.diff(rowptr)
    first = np.abs(w[np.minimum(rowptr[:-1], len(w) - 1)])
    ok = ((n == 1) & (first == 1.0)) | (n == 0)
    return ok.reshape(len(blocks), -1).all(axis=1)


def _close(got, want, exact, scale):
    assert got.shape == want.shape
    assert np.array_equal(got[exact], want[exact])
    assert np.abs(got - want).max(initial=0.0) <= 1e-12 * scale


def _check(sim, blocks, bpdx, bpdy, shapes, pts, res, out):
    """the device's surface points / skins / sums against the oracle's (or the record's) pts and res"""
    en = _copy_only(blocks, bpdx, bpdy, 2)
    ef = en & _copy_only(blocks, bpdx, bpdy, 3) & _copy_only(blocks, bpdx, bpdy, 6)
    for k, (s, P, r) in enumerate(zip(shapes, pts, res)):
        g = sim.surface_get(k)
        ids = np.asarray(s["ids"])
        blk = np.array([ids[q] for q, b in enumerate(P) for _ in b], dtype=np.int32)
        w = np.array([p for b in P for p in b]).reshape(-1, 5)
        assert np.array_equal(g["block"], blk)
        assert np.array_equal(g["ixy"], w[:, :2].astype(np.int32))
        _close(g["normal"], w[:, 2:], en[blk], np.abs(w[:, 2:]).max(initial=0.0))
        for c in range(14):
            _close(g["skin"][:, c], r["skin"][:, c], ef[blk], np.abs(r["skin"][:, c]).max(initial=0.0))
        if ef[ids].all():
            assert np.array_equal(out[k, :19], r["q19"])
        else:
            assert (np.abs(out[k, :19] - r["q19"]) <= 1e-12 * r["abs19"]).all()
        assert np.array_equal(out[k, 19:], fo.derived(out[k, :19], float(s["u"]), float(s["v"])))


def _replay(st):
    """a context holding the record's fields and shapes, surface and forces run"""
    sim = _sim(st["blocks"], st["bpdx"], st["bpdy"], st["h0"], st["nu"])
    sim.upload("chi", st["chi_n"])
    sim.upload("tmp", st["tmp"])
    for k, s in enumerate(st["shapes"]):
        sim.shape_set(k, s["ids"], s["chi"], s["udef"])
    sim.surface(len(st["shapes"]))
    sim.upload("vel", st["vel"])
    sim.upload("pres", st["pres"])
    return sim, sim.forces(st["shapes"])


def test_fixture_replay(steps):
    for st in steps:
        sim, out = _replay(st)
        pts = [[[tuple(p) for p in np.split(s["surf"], np.cumsum(s["npts"])[:-1])[q]] for q in range(len(s["ids"]))]
               for s in st["shapes"]]
        res = [dict(skin=s["skin"], q19=s["q19"], abs19=fo.forces(st["blocks"], st["bpdx"], st["bpdy"], st["h0"], st["nu"],
                                                                   st["vel"], st["pres"], st["chi_n"], [s], [P])[0]["abs19"])
               for s, P in zip(st["shapes"], pts)]
        _check(sim, st["blocks"], st["bpdx"], st["bpdy"], st["shapes"], pts, res, out)
        for k, s in enumerate(st["shapes"]):
            assert np.array_equal(out[k, 19:], s["derived4"]) or not _copy_only(st["blocks"], st["bpdx"], st["bpdy"], 6)[s["ids"]].all()
        sim.close()


def test_surface_after_ongrid(golden_dir):
    """the device chain ongrid -> surface on the ongrid fixture, against the oracle's normals of the chi and tmp ongrid left"""
    sys.path.insert(0, golden_dir)
    import make_ongrid_golden
    c = make_ongrid_golden.load(os.path.join(golden_dir, "amrongrid_lmax8.npz"))[0]
    sim = _sim(c["blocks"], c["bpdx"], c["bpdy"], c["h0"])
    bodies = [{**{n: s[n] for n in bo.MIDLINE}, "center": s["center"], "orientation": s["orientation"],
               "center_of_mass": s["center_of_mass"]} for s in c["shapes"]]
    sim.ongrid(bodies)
    sim.surface(len(bodies))
    chi, tmp = sim.download("chi")[..., 0], sim.download("tmp")[..., 0]
    shapes = [sim.shape_get(k) for k in range(len(bodies))]
    pts = fo.normals(c["blocks"], c["bpdx"], c["bpdy"], c["h0"], chi, tmp, [s["ids"] for s in shapes])
    en = _copy_only(c["blocks"], c["bpdx"], c["bpdy"], 2)
    for k, (s, P) in enumerate(zip(shapes, pts)):
        g = sim.surface_get(k)
        w = np.array([p for b in P for p in b]).reshape(-1, 5)
        blk = np.array([s["ids"][q] for q, b in enumerate(P) for _ in b], dtype=np.int32)
        assert np.array_equal(g["block"], blk) and np.array_equal(g["ixy"], w[:, :2].astype(np.int32))
        _close(g["normal"], w[:, 2:], en[blk], np.abs(w[:, 2:]).max())
        assert not g["skin"].any()  # no forces call yet
    sim.close()


def _three_level(base, centre):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import bench_amr
    return bench_amr.three_level_mesh(base, r1=0.3, r2=0.15, centre=centre)


def _seed(blocks, h0):
    """smooth vel and pres on the cell centres"""
    b = np.asarray(blocks)
    h = (h0 / (1 << b[:, 0]).astype(np.float64))[:, None, None]
    c = np.arange(8) + 0.5
    x = (b[:, 1, None, None] * 8 + c[None, None, :]) * h
    y = (b[:, 2, None, None] * 8 + c[None, :, None]) * h
    vel = np.stack([0.3 * np.sin(2.1 * x + 0.3) * np.cos(1.7 * y) + 0.05, 0.2 * np.cos(1.3 * x) * np.sin(2.3 * y + 0.1)], -1)
    return vel, 0.5 * np.cos(1.9 * x - 0.2) * np.cos(1.1 * y + 0.4)


SYNTH = {  # (mesh centre, bodies, (u, v) of every shape)
    "level_jumps": ((0.45, 0.55), lambda: [bo.synthetic_body((0.62, 0.55), 0.2, 161, -0.2)], (0.2, -0.1)),
    "wall_and_corner": ((0.1, 0.15), lambda: [bo.synthetic_body((0.012, 0.5), 0.15, 121, 1.5708, bend=0.1),
                                               bo.synthetic_body((0.03, 0.025), 0.05, 41, 0.8, bend=0.2)], (0.1, 0.05)),
    "shared_blocks": ((0.45, 0.55), lambda: [bo.synthetic_body((0.45, 0.55), 0.12, 97, 0.3, com_offset=(0.002, -0.001)),
                                             bo.synthetic_body((0.47, 0.56), 0.10, 81, 2.5, bend=0.5, phase=1.0)], (-0.15, 0.12)),
    "at_rest": ((0.45, 0.55), lambda: [bo.synthetic_body((0.45, 0.5), 0.15, 121, 0.7)], (0.0, 0.0)),
}


@pytest.mark.parametrize("case", sorted(SYNTH))
def test_synthetic_three_level_vs_oracle(case):
    base, h0 = 3, 1 / 8
    centre, make, uv = SYNTH[case]
    blocks = _three_level(base, centre)
    bodies = make()
    sim = _sim(blocks, 1, 1, h0, 1e-3)
    sim.ongrid(bodies)
    n = len(bodies)
    chi, tmp = sim.download("chi")[..., 0], sim.download("tmp")[..., 0]
    shapes = [dict(sim.shape_get(k), u=uv[0], v=uv[1], center_of_mass=np.asarray(bodies[k]["center"], float)) for k in range(n)]
    vel, pres = _seed(blocks, h0)
    sim.upload("vel", vel)
    sim.upload("pres", pres)
    margins = []
    pts = fo.normals(blocks, 1, 1, h0, chi, tmp, [s["ids"] for s in shapes], margins=margins)
    assert min(margins) > 1e-10  # no cell within 1e-10 of a normals threshold: the point lists cannot differ by rounding
    res = fo.forces(blocks, 1, 1, h0, 1e-3, vel, pres, chi, shapes, pts)
    sim.surface(n)
    out = sim.forces(shapes)
    _check(sim, blocks, 1, 1, shapes, pts, res, out)
    irregular = ~_copy_only(blocks, 1, 1, 6)
    npts = [[len(b) for b in P] for P in pts]
    assert any(0 in c for c in npts)  # obstacle blocks without surface points
    if case == "level_jumps":
        assert any(irregular[s["ids"][q]] and npts[k][q] for k, s in enumerate(shapes) for q in range(len(s["ids"])))
    if case == "wall_and_corner":
        xy = [(blocks[s["ids"][q], 1], blocks[s["ids"][q], 2]) for k, s in enumerate(shapes) for q in range(len(s["ids"])) if npts[k][q]]
        assert any(i == 0 for i, _ in xy) and (0, 0) in xy
    if case == "shared_blocks":
        common = set(shapes[0]["ids"].tolist()) & set(shapes[1]["ids"].tolist())
        assert len(common) > 4
        g0, g1 = sim.surface_get(0), sim.surface_get(1)
        for b in common:  # the same points for both shapes: the normals come from the global chi and tmp
            assert np.array_equal(g0["normal"][g0["block"] == b], g1["normal"][g1["block"] == b])
    if case == "at_rest":
        assert out[0, 16] == 0 and out[0, 19] == 0 and out[0, 20] == 0  # vel_unit = 0: no thrust; Pthrust = Pdrag = 0
    sim.close()


def _state(sim, n):
    f = {k: sim.download(k).copy() for k in ("vel", "pres", "chi", "tmp")}
    return f, [sim.shape_get(k, dist=False) for k in range(n)]


def _same_state(a, b):
    for k in a[0]:
        assert np.array_equal(a[0][k], b[0][k]), k
    for s, t in zip(a[1], b[1]):
        for k in ("ids", "chi", "udef"):
            assert np.array_equal(s[k], t[k]), k


def test_repeated_calls_are_identical_and_change_nothing(steps):
    st = steps[0]
    sim, out = _replay(st)
    n = len(st["shapes"])
    before = _state(sim, n)
    g = [sim.surface_get(k) for k in range(n)]
    sim.surface(n)
    out2 = sim.forces(st["shapes"])
    assert np.array_equal(out, out2)
    for k in range(n):
        h = sim.surface_get(k)
        for key in g[k]:
            assert np.array_equal(g[k][key], h[key])
    _same_state(before, _state(sim, n))
    sim.close()


def test_surface_is_dropped_by_shape_set_ongrid_and_regrid(steps, golden_dir):
    from cup2d_b200 import lib as L
    from cup2d_b200.amr import adapt_mesh
    st = steps[0]
    sim, _ = _replay(st)
    n = len(st["shapes"])
    s0 = st["shapes"][0]
    sim.shape_set(0, s0["ids"], s0["chi"], s0["udef"])
    with pytest.raises(L.Cup2dError, match="error -4"):
        sim.forces(st["shapes"])
    with pytest.raises(L.Cup2dError, match="error -4"):
        sim.surface_get(0)
    sim.surface(n)
    sim.forces(st["shapes"])
    sys.path.insert(0, golden_dir)
    import make_ongrid_golden
    c = make_ongrid_golden.load(os.path.join(golden_dir, "amrongrid_lmax8.npz"))[0]
    assert np.array_equal(c["blocks"], st["blocks"])
    bodies = [{**{m: s[m] for m in bo.MIDLINE}, "center": s["center"], "orientation": s["orientation"],
               "center_of_mass": s["center_of_mass"]} for s in c["shapes"]]
    sim.ongrid(bodies)
    with pytest.raises(L.Cup2dError, match="error -4"):
        sim.forces(st["shapes"])
    sim.surface(n)
    sim.forces(st["shapes"])
    # regrid: the shapes are gone (not set: EINVAL); placed again, the points are missing until surface runs
    linf = np.zeros(len(sim.blocks))
    linf[0] = 10.0
    new = adapt_mesh(sim.blocks, st["bpdx"], st["bpdy"], 8, linf, 1.0, 0.1)
    assert not np.array_equal(new, sim.blocks)
    sim.regrid(new)
    with pytest.raises(L.Cup2dError, match="error -1"):
        sim.forces(st["shapes"])
    sim.ongrid(bodies)
    with pytest.raises(L.Cup2dError, match="error -4"):
        sim.forces(st["shapes"])
    sim.surface(n)
    assert np.isfinite(sim.forces(st["shapes"])).all()
    sim.close()


def test_error_paths_leave_the_context_unchanged(steps):
    import ctypes as C
    from cup2d_b200 import lib as L
    st = steps[0]
    sim, out = _replay(st)
    n = len(st["shapes"])
    before = _state(sim, n)
    g = [sim.surface_get(k) for k in range(n)]
    lib, h = sim.lib, sim._h
    buf = np.full((64, 23), 7.0)
    P = buf.ctypes.data_as(C.POINTER(C.c_double))
    R = (L.Rigid * 64)()
    for k, s in enumerate(st["shapes"]):
        R[k].u, R[k].v = s["u"], s["v"]
        R[k].center_of_mass[0], R[k].center_of_mass[1] = s["center_of_mass"]
    assert lib.cup2d_amr_forces(h, 0, R, P) == -1
    assert lib.cup2d_amr_forces(h, 65, R, P) == -1
    assert lib.cup2d_amr_forces(h, n + 1, R, P) == -1          # a shape not set
    assert lib.cup2d_amr_forces(h, n, None, P) == -1
    assert lib.cup2d_amr_forces(h, n, R, None) == -1
    assert lib.cup2d_amr_surface(h, 0) == -1 and lib.cup2d_amr_surface(h, 65) == -1 and lib.cup2d_amr_surface(h, n + 1) == -1
    assert lib.cup2d_amr_surface_get(h, n, None, None, None, None) == -1
    assert lib.cup2d_amr_surface_get(h, -1, None, None, None, None) == -1
    assert (buf == 7.0).all()
    _same_state(before, _state(sim, n))
    for k in range(n):
        hh = sim.surface_get(k)
        for key in g[k]:
            assert np.array_equal(g[k][key], hh[key])
    assert np.array_equal(sim.forces(st["shapes"]), out)
    sim.close()
