"""GPU tests of the collision model on multi-level contexts (cup2d_amr_collide, csrc/amr_collide.cu): against the reference's
own collision model on its run.sh mesh (tests/golden/amrcollide_lmax8.npz) and against the oracle
(tests/amr_collision_oracle.py) on synthetic three-level meshes, bit for bit.  They also pass on the CPU against the emulated
build of the same sources (tests/test_amr_collide.py)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import amr_body_oracle as bo
import amr_collision_oracle as co

pytestmark = [pytest.mark.gpu]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RIGID = ("u", "v", "omega", "center_of_mass", "M", "J", "length")


@pytest.fixture(scope="module")
def calls(golden_dir):
    sys.path.insert(0, golden_dir)
    import make_collide_golden
    return make_collide_golden.load(os.path.join(golden_dir, "amrcollide_lmax8.npz"))


def _sim(blocks, bpdx, bpdy, h0):
    from cup2d_b200.amr import AmrSimulation
    return AmrSimulation(blocks, bpdx, bpdy, h0, 4e-5)


def _upload(sim, shapes):
    for k, s in enumerate(shapes):
        sim.shape_set(k, s["ids"], s["chi"], s["udef"])
        sim.shape_set_dist(k, s["dist"])


def _motions(shapes):
    return [{n: s[n] for n in RIGID} for s in shapes]


def _state(sim, n):
    return [sim.download("vel"), sim.download("chi")] + [sim.shape_get(k) for k in range(n)]


def _same_state(a, b):
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    for x, y in zip(a[2:], b[2:]):
        for n in x:
            assert np.array_equal(x[n], y[n]), n


def test_recorded_shapes_reproduce_the_reference(calls):
    for c in calls:
        sim = _sim(c["blocks"], c["bpdx"], c["bpdy"], c["h0"])
        _upload(sim, c["shapes"])
        uvw, sums = sim.collide(_motions(c["shapes"]))
        assert np.array_equal(sums, c["sums20"]), c["config"]
        assert np.array_equal(uvw, c["uvw_after"]), c["config"]
        sim.close()


def test_two_calls_are_bitwise_identical_and_change_nothing(calls):
    c = calls[0]
    nb = len(c["blocks"])
    sim = _sim(c["blocks"], c["bpdx"], c["bpdy"], c["h0"])
    rng = np.random.default_rng(1)
    sim.upload("vel", rng.uniform(-1, 1, (nb, 8, 8, 2)))
    sim.upload("chi", rng.uniform(0, 1, (nb, 8, 8, 1)))
    _upload(sim, c["shapes"])
    before = _state(sim, 2)
    r1 = sim.collide(_motions(c["shapes"]))
    r2 = sim.collide(_motions(c["shapes"]))
    assert np.array_equal(r1[0], r2[0]) and np.array_equal(r1[1], r2[1])
    _same_state(before, _state(sim, 2))
    sim.close()


def test_shape_set_dist_roundtrip_and_shape_set_clears_it(calls):
    from cup2d_b200 import lib as L
    c = calls[0]
    s = c["shapes"][0]
    sim = _sim(c["blocks"], c["bpdx"], c["bpdy"], c["h0"])
    sim.shape_set(0, s["ids"], s["chi"], s["udef"])
    with pytest.raises(L.Cup2dError):
        sim.shape_get(0)
    sim.shape_set_dist(0, s["dist"])
    g = sim.shape_get(0)
    for n in ("ids", "chi", "dist", "udef"):
        assert np.array_equal(g[n], s[n]), n
    sim.shape_set(0, s["ids"], s["chi"], s["udef"])
    with pytest.raises(L.Cup2dError):
        sim.shape_get(0)
    with pytest.raises(L.Cup2dError):
        sim.shape_set_dist(3, s["dist"])      # no such shape
    sim.close()


def _raw_collide(sim, motions, n=None):
    """cup2d_amr_collide on a ctypes array: (return code, the array afterwards as a list of tuples)"""
    from cup2d_b200 import lib as L
    st = (L.Rigid * max(len(motions), 1))()
    for k, m in enumerate(motions):
        st[k].u, st[k].v, st[k].omega = m["u"], m["v"], m["omega"]
        st[k].center_of_mass[0], st[k].center_of_mass[1] = m["center_of_mass"]
        st[k].M, st[k].J, st[k].length = m["M"], m["J"], m["length"]
    sums = np.full(20 * 80, 7.0)
    rc = sim.lib.cup2d_amr_collide(sim._h, len(motions) if n is None else n, st, sums.ctypes.data_as(C.POINTER(C.c_double)))
    return rc, [(r.u, r.v, r.omega, r.center_of_mass[0], r.center_of_mass[1], r.M, r.J, r.length) for r in st], sums


def test_error_paths_leave_shapes_and_the_context_unchanged(calls):
    EINVAL, ESTATE = -1, -4
    c = calls[0]
    shapes = c["shapes"]
    sim = _sim(c["blocks"], c["bpdx"], c["bpdy"], c["h0"])
    _upload(sim, shapes)
    mo = _motions(shapes)
    before = _state(sim, 2)
    _, pristine2, _ = _raw_collide(sim, mo, n=0)
    for n in (0, -1, 65):                                          # nshapes outside 1..64
        rc, st, sums = _raw_collide(sim, mo, n=n)
        assert rc == EINVAL and st == pristine2 and (sums == 7.0).all()
    rc, st, sums = _raw_collide(sim, mo + mo[:1])                  # shape 2 was never set
    assert rc == EINVAL and st == _raw_collide(sim, mo + mo[:1], n=0)[1] and (sums == 7.0).all()
    _same_state(before, _state(sim, 2))
    ids = shapes[1]["ids"]
    desc = np.ascontiguousarray(ids[::-1])                         # ids not strictly ascending
    sim.shape_set(1, desc, shapes[1]["chi"][::-1], shapes[1]["udef"][::-1])
    sim.shape_set_dist(1, shapes[1]["dist"][::-1])
    rc, st, sums = _raw_collide(sim, mo)
    assert "ascending" in sim.lib.cup2d_last_error().decode()
    assert rc == EINVAL and st == _raw_collide(sim, mo, n=0)[1] and (sums == 7.0).all()
    sim.shape_set(1, ids, shapes[1]["chi"], shapes[1]["udef"])    # ascending again, but without dist
    rc, st, sums = _raw_collide(sim, mo)
    assert rc == ESTATE and st == _raw_collide(sim, mo, n=0)[1] and (sums == 7.0).all()
    sim.shape_set_dist(1, shapes[1]["dist"])
    _same_state(before, _state(sim, 2))
    rc, st, _ = _raw_collide(sim, mo)
    assert rc == 0 and st != pristine2                             # the head-to-head record applies an impulse
    from cup2d_b200 import lib as L
    rb = np.array([0, len(c["blocks"]) // 2, len(c["blocks"])], dtype=np.int64)
    L.check(sim.lib.cup2d_amr_set_ranks(sim._h, 0, 2, rb.ctypes.data_as(C.POINTER(C.c_int64))))
    rc, st, sums = _raw_collide(sim, mo)                           # several ranks
    assert rc == ESTATE and st == _raw_collide(sim, mo, n=0)[1] and (sums == 7.0).all()
    sim.close()


# ---- synthetic three-level meshes: ongrid, then collide, against the oracle fed with shape_get's blocks ----
def _three_level(base, centre=(0.45, 0.55)):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import bench_amr
    return bench_amr.three_level_mesh(base, r1=0.3, r2=0.15, centre=centre)


def _fish(center, orientation, L=0.3, **kw):
    return bo.synthetic_body(center, L, 8 * 24 + 1, orientation, **kw)


# case -> (bodies, velocities (u, v, omega) per body, the expected branch of every pair)
SYNTH = {
    # two nearly coincident fish across the finest region's edge: the overlap covers blocks of two levels and block edges
    "level_jump": ([_fish((0.55, 0.62), 0.3), _fish((0.552, 0.623), 0.32, phase=0.5)],
                   [(1.0, 0.5, 0.2), (-1.0, -0.5, -0.1)], None),
    # three overlapping fish, shape 0 with length 0.02: its overlaps with 1 and with 2 have centroids further apart than that,
    # so the pair (0, 2) is rejected by the distance test; (0, 1) recedes and (1, 2) collides
    "three_shapes": ([_fish((0.40, 0.55), 0.0), _fish((0.45, 0.56), 0.1), _fish((0.55, 0.55), 0.0, phase=1.0)],
                     [(1.0, 0.0, 0.0), (-1.0, 0.0, 0.0), (-1.0, 0.0, 0.0)],
                     {(0, 1): "receding", (0, 2): "distance", (1, 2): "impulse"}),
    # a pair that barely touches: the common mass is below 2 cells
    "touching": ([_fish((0.45, 0.55), 0.0), _fish((0.45, 0.5718), 0.0, phase=2.0)],
                 [(0.0, 1.0, 0.0), (0.0, -1.0, 0.0)], {(0, 1): "mass"}),
    # overlapping fish whose mean velocities separate along the contact normal (projVel <= 0)
    "receding": ([_fish((0.45, 0.55), 0.0), _fish((0.452, 0.552), 0.05)],
                 [(0.0, 3.0, 0.0), (0.0, -3.0, 0.0)], {(0, 1): "receding"}),
    # the same fish with the velocities reversed: they approach along the normal and the impulse applies
    "impulse": ([_fish((0.45, 0.55), 0.0), _fish((0.452, 0.552), 0.05)],
                [(0.0, -3.0, 0.0), (0.0, 3.0, 0.0)], {(0, 1): "impulse"}),
    # no common block
    "apart": ([_fish((0.30, 0.45), 0.0), _fish((0.60, 0.65), 0.0)], [(1.0, 0.0, 0.0), (-1.0, 0.0, 0.0)], {(0, 1): "mass"}),
    # one shape
    "single": ([_fish((0.45, 0.55), 0.3)], [(1.0, 2.0, 3.0)], {}),
}


@pytest.mark.parametrize("case", sorted(SYNTH))
def test_synthetic_three_level_collide_vs_oracle(case):
    h0 = 1 / 8
    blocks = _three_level(4)
    bodies, vel, expect = SYNTH[case]
    sim = _sim(blocks, 1, 1, h0)
    out = sim.ongrid(bodies)
    shapes = []
    for k in range(len(bodies)):
        g = sim.shape_get(k)
        u, v, w = vel[k]
        shapes.append({**g, "u": u, "v": v, "omega": w, "center_of_mass": out[k, 3:5], "M": out[k, 5], "J": out[k, 6],
                       "length": 0.02 if (case == "three_shapes" and k == 0) else 0.3})
    before = _state(sim, len(bodies))
    uvw, sums = sim.collide(_motions(shapes))
    want_uvw, want_sums, hits = co.collide(blocks, h0, shapes)
    assert np.array_equal(sums, want_sums)
    assert np.array_equal(uvw, want_uvw)
    _same_state(before, _state(sim, len(bodies)))
    br = co.branches(want_sums, shapes)
    moved = not np.array_equal(uvw, np.array(vel, dtype=np.float64))
    assert moved == bool(hits)
    if expect is not None:
        for pair, b in expect.items():
            assert br[pair] == b, br
    if case == "level_jump":   # contributing cells on blocks of two levels and at block edges, and an applied impulse
        common, ki, kj = np.intersect1d(shapes[0]["ids"], shapes[1]["ids"], return_indices=True)
        on = (shapes[0]["chi"][ki] > 0) & (shapes[1]["chi"][kj] > 0)
        lv = blocks[common, 0]
        assert len(set(lv[on.any(axis=(1, 2))].tolist())) >= 2
        assert on[:, :, [0, 7]].any() and on[:, [0, 7], :].any()
        assert br[0, 1] == "impulse"
    if case == "touching":
        assert 0 < sums[0, 0] < 2
    if case in ("apart", "single"):
        assert (sums == 0).all() and not moved
    sim.close()
