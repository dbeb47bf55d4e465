"""GPU tests of the enqueued multi-level steps (cup2d_amr_step_enqueue / _pressure_enqueue / _step_result / _set_graph,
csrc/amr_ops.cu): against the blocking calls on the reference's run.sh mesh (tests/golden/amrlab_lmax8.npz) and on a
synthetic three-level mesh, both kernel modes; graph replay against direct launches; the WHILE node of a tolerance-driven
solve; regrids between enqueues; the error codes.

The tests that do not need graphs also pass on the CPU against the emulated build of the same sources, where every enqueue
takes the direct path (tests/test_amr_step_enqueue_emulation.py)."""
import os
import sys

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MESHES = ["runsh", "synthetic"]


def rel(a, b):
    return np.abs(a - b).max() / np.abs(b).max()


def _mesh(name, golden_dir):
    """(blocks, bpdx, bpdy, h0, nu, vel, pres)"""
    if name == "runsh":
        d = np.load(os.path.join(golden_dir, "amrlab_lmax8.npz"))
        return d["blocks"], int(d["bpdx"]), int(d["bpdy"]), float(d["h0"]), float(d["nu"]), d["vel"], d["pres"]
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import bench_amr
    blocks = bench_amr.three_level_mesh(3, r1=0.3, r2=0.15, centre=(0.45, 0.55))
    h0 = 1 / 8
    rng = np.random.default_rng(11)
    vel, pres = bench_amr.seeded_fields(blocks, h0)
    return blocks, 1, 1, h0, 1e-3, vel + 0.05 * rng.uniform(-1, 1, vel.shape), pres + 0.05 * rng.uniform(-1, 1, pres.shape)


def _sim(m, fast, graph=True):
    from cup2d_b200.amr import AmrSimulation
    blocks, bx, by, h0, nu, vel, pres = m
    sim = AmrSimulation(blocks, bx, by, h0, nu)
    sim.set_fast(fast)
    sim.set_graph(graph)
    sim.upload("vel", vel)
    sim.upload("pres", pres)
    return sim


def _same(a, b):
    for n in ("vel", "pres"):
        assert np.array_equal(a.download(n), b.download(n)), n


@pytest.mark.parametrize("fast", [False, True])
@pytest.mark.parametrize("mesh", MESHES)
def test_enqueued_steps_match_the_blocking_step(golden_dir, mesh, fast):
    """3 steps with the dt rule on the device and 8 fixed Krylov iterations: dt bitwise the host's rule on the same velocity,
    the same iteration counts, fields equal to rounding (the pressure means are summed in another order)"""
    m = _mesh(mesh, golden_dir)
    a, b = _sim(m, fast), _sim(m, fast)
    for _ in range(3):
        _, dt_host = b.compute_dt(0.5)
        b.step_enqueue(cfl=0.5, dt=0.0, max_iter=8)
        dt_b, it_b, err_b = b.step_result()
        assert dt_b == dt_host
        dt_a, it_a, err_a = a.step(cfl=0.5, max_iter=8)
        assert it_a == it_b == 8
        assert abs(dt_a - dt_b) <= 1e-13 * dt_a
        assert abs(err_a - err_b) <= 1e-9 * err_a
        for n in ("vel", "pres"):
            assert rel(b.download(n), a.download(n)) < 1e-13, n
    a.close()
    b.close()


@pytest.mark.parametrize("fast", [False, True])
@pytest.mark.parametrize("mesh", MESHES)
def test_pressure_enqueue_matches_the_blocking_pressure_section(golden_dir, mesh, fast):
    """u_def from cup2d_amr_udef_assemble and chi as they stand: poisson_rhs + poisson_solve + pressure_correct"""
    m = _mesh(mesh, golden_dir)
    nb = len(m[0])
    rng = np.random.default_rng(5)
    ids = np.arange(0, nb, 3, dtype=np.int32)
    X, U = rng.uniform(0, 1, (len(ids), 8, 8)), rng.uniform(-0.5, 0.5, (len(ids), 8, 8, 2))
    chi = np.zeros((nb, 8, 8, 1))
    chi[ids] = X[..., None]
    dt = 1e-3
    out = []
    for enq in (False, True):
        s = _sim(m, fast)
        s.upload("chi", chi)
        s.shape_set(0, ids, X, U)
        s.udef_assemble()
        if enq:
            s.pressure_enqueue(dt, max_iter=8)
            _, it, err = s.step_result()
        else:
            s.poisson_rhs(dt)
            it, err = s.poisson_solve(max_iter=8)
            s.pressure_correct(dt)
        out.append((it, err, s.download("vel"), s.download("pres")))
        s.close()
    (it_a, err_a, va, pa), (it_b, err_b, vb, pb) = out
    assert it_a == it_b == 8
    assert abs(err_a - err_b) <= 1e-9 * err_a
    assert rel(vb, va) < 1e-13 and rel(pb, pa) < 1e-13


@pytest.mark.parametrize("fast", [False, True])
@pytest.mark.parametrize("mesh", MESHES)
def test_six_enqueues_one_result_equal_six_pairs(golden_dir, mesh, fast):
    m = _mesh(mesh, golden_dir)
    a, b = _sim(m, fast), _sim(m, fast)
    for _ in range(6):
        a.step_enqueue(cfl=0.5, max_iter=8)
        ra = a.step_result()
    for _ in range(6):
        b.step_enqueue(cfl=0.5, max_iter=8)
    assert b.step_result() == ra
    _same(a, b)
    a.close()
    b.close()


@pytest.mark.parametrize("fast", [False, True])
def test_regrid_between_enqueues_steps_like_a_fresh_context(golden_dir, fast):
    """after a regrid the context's enqueued steps (direct, then replayed) are bitwise those of a context created on the new
    mesh with the same fields"""
    sys.path.insert(0, golden_dir)
    import make_regrid_golden
    g = make_regrid_golden.load(os.path.join(golden_dir, "amrregrid_lmax8.npz"))
    bx, by, h0 = int(g["bpdx"]), int(g["bpdy"]), float(g["h0"])
    a = _sim((g["blocks"], bx, by, h0, 4e-5, g["vel"], g["pres"]), fast)
    for _ in range(2):                   # direct, then (on a GPU) a graph of the old mesh
        a.step_enqueue(cfl=0.5, max_iter=5)
    a.step_result()
    for n in ("vel", "pres", "chi"):
        a.upload(n, g[n])
    a.regrid(g["new_blocks"])
    b = _sim((g["new_blocks"], bx, by, h0, 4e-5, a.download("vel"), a.download("pres")), fast)
    b.upload("chi", a.download("chi"))
    for _ in range(3):
        a.step_enqueue(cfl=0.5, max_iter=5)
        b.step_enqueue(cfl=0.5, max_iter=5)
        assert a.step_result() == b.step_result()
        _same(a, b)
    a.close()
    b.close()


def test_error_codes(golden_dir):
    from cup2d_b200 import lib as L
    m = _mesh("synthetic", golden_dir)
    s = _sim(m, True)
    lib, h = s.lib, s._h
    assert lib.cup2d_amr_step_result(h, None, None, None) == -4          # nothing pending
    vel0 = s.download("vel")
    bad = [(0.5, float("nan"), 0.0, 0.0, 0, 8), (0.5, float("inf"), 0.0, 0.0, 0, 8), (0.0, 0.0, 0.0, 0.0, 0, 8),
           (float("nan"), 0.0, 0.0, 0.0, 0, 8), (0.5, 0.0, -1.0, 0.0, 0, 8), (0.5, 0.0, 0.0, -1.0, 0, 8),
           (0.5, 0.0, 0.0, 0.0, -1, 8), (0.5, 0.0, 0.0, 0.0, 0, -1)]
    for args in bad:
        assert lib.cup2d_amr_step_enqueue(h, *args) == -1, args
    for dt in (0.0, -1e-3, float("nan"), float("inf")):
        assert lib.cup2d_amr_pressure_enqueue(h, dt, 0.0, 0.0, 0, 8) == -1, dt
    assert lib.cup2d_amr_pressure_enqueue(h, 1e-3, 0.0, 0.0, 0, -1) == -1
    assert lib.cup2d_amr_step_enqueue(None, 0.5, 0.0, 0.0, 0.0, 0, 8) == -1
    assert lib.cup2d_amr_step_result(h, None, None, None) == -4          # the refused calls left nothing pending
    assert np.array_equal(s.download("vel"), vel0)
    s.step_enqueue(cfl=0.5, max_iter=4)
    assert lib.cup2d_amr_step_result(h, None, None, None) == 0           # any output pointer may be NULL
    assert lib.cup2d_amr_step_result(h, None, None, None) == -4
    s.close()
    r = _sim(m, True)
    r.set_ranks(0, [0, len(m[0])])
    vel0 = r.download("vel")
    assert lib.cup2d_amr_step_enqueue(r._h, 0.5, 0.0, 0.0, 0.0, 0, 8) == -4
    assert lib.cup2d_amr_pressure_enqueue(r._h, 1e-3, 0.0, 0.0, 0, 8) == -4
    assert lib.cup2d_amr_set_graph(r._h, 0) == -4
    assert lib.cup2d_amr_step_result(r._h, None, None, None) == -4
    assert np.array_equal(r.download("vel"), vel0)
    r.close()
    t = _sim(m, True)
    with pytest.raises(L.Cup2dError):
        t.step_result()
    t.close()


# ---- graphs: these need a GPU (the emulated build always launches directly) -----------------------------------------
@pytest.mark.parametrize("fast", [False, True])
@pytest.mark.parametrize("mesh", MESHES)
def test_graph_replay_equals_direct_launch(golden_dir, mesh, fast):
    m = _mesh(mesh, golden_dir)
    g, d = _sim(m, fast, graph=True), _sim(m, fast, graph=False)
    for _ in range(5):
        g.step_enqueue(cfl=0.5, max_iter=10)
        d.step_enqueue(cfl=0.5, max_iter=10)
        assert g.step_result() == d.step_result()
        _same(g, d)
    g.close()
    d.close()


@pytest.mark.parametrize("fast", [False, True])
@pytest.mark.parametrize("mesh", MESHES)
def test_while_node_stops_where_the_host_polled_solve_stops(golden_dir, mesh, fast):
    """tolerance-driven solves: the graph's WHILE node stops at the iteration and residual of the host-polled batches of the
    direct path, step after step; in the first step (same inputs up to the solve) also at those of the blocking step"""
    m = _mesh(mesh, golden_dir)
    kw = dict(tol_abs=1e-7, tol_rel=0.0, max_restarts=100, max_iter=400)
    g, d, b = _sim(m, fast, graph=True), _sim(m, fast, graph=False), _sim(m, fast)
    rb = b.step(cfl=0.5, **kw)
    for k in range(4):
        g.step_enqueue(cfl=0.5, **kw)
        d.step_enqueue(cfl=0.5, **kw)
        rg, rd = g.step_result(), d.step_result()
        assert rg == rd
        assert 0 < rg[1] < 400
        _same(g, d)
        if k == 0:
            assert rg == rb
    g.close()
    d.close()
    b.close()
