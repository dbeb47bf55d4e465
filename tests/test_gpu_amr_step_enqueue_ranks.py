"""GPU tests of the enqueued multi-level steps on distributed contexts (cup2d_amr_create_ranks; one H100, so one rank): the
enqueued body runs in place on the Poisson context's stream and arrays, and dt's maximum and the two pressure means go
through the in-kernel peer all-reduce, a no-op on one rank.  So a one-rank distributed context steps bit for bit like the
plain context's enqueued step, and to rounding like its own blocking step (whose means add the blocks in another order).
Cases as in tests/test_gpu_amr_step_graph.py (tests/amr_step_ranks.py).  Several ranks:
tests/test_amr_step_enqueue_ranks_emulation.py on the CPU, tools/multi_gpu_amr_enqueue_check.py on several GPUs."""
import numpy as np
import pytest

import amr_step_ranks as S

pytestmark = [pytest.mark.gpu]


def _dist(m, graph=True):
    rb = np.array([0, len(m[0])], dtype=np.int64)
    return S.make(m, 0, rb, graph=graph)


def _same(a, b):
    for n in ("vel", "pres"):
        assert np.array_equal(a.download(n), b.download(n)), n


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("mesh", S.MESHES)
def test_enqueued_steps_equal_the_plain_context(mesh, graph):
    """3 steps, dt on the device, 8 fixed Krylov iterations: dt, iterations, residual, vel and pres bit for bit"""
    m = S.mesh(mesh)
    d, p = _dist(m, graph), S.make(m, graph=graph)
    rd, fd = S.run_steps(d, 3, True, dt=0.0, max_iter=8)
    rp, fp = S.run_steps(p, 3, True, dt=0.0, max_iter=8)
    assert rd == rp
    for n in fd:
        assert np.array_equal(fd[n], fp[n]), n
    d.close()
    p.close()


@pytest.mark.parametrize("mesh", S.MESHES)
def test_enqueued_steps_match_the_blocking_distributed_step(mesh):
    """dt bitwise the blocking dt rule on the same velocity, the same iterations, fields to 1e-13"""
    m = S.mesh(mesh)
    e, b = _dist(m), _dist(m)
    for _ in range(3):
        (re_,), fe = S.run_steps(e, 1, True, check_dt=True, max_iter=8)
        (rb_,), fb = S.run_steps(b, 1, False, max_iter=8)
        assert re_[1] == rb_[1] == 8
        assert abs(re_[0] - rb_[0]) <= 1e-13 * rb_[0]
        for n in fe:
            assert S.rel(fe[n], fb[n]) <= S.FIELD_TOL, n
    e.close()
    b.close()


@pytest.mark.parametrize("mesh", S.MESHES)
def test_graph_replay_equals_direct_launch(mesh):
    m = S.mesh(mesh)
    g, d = _dist(m, graph=True), _dist(m, graph=False)
    for _ in range(5):
        g.step_enqueue(cfl=0.5, max_iter=10)
        d.step_enqueue(cfl=0.5, max_iter=10)
        assert g.step_result() == d.step_result()
        _same(g, d)
    g.close()
    d.close()


@pytest.mark.parametrize("mesh", S.MESHES)
def test_while_node_stops_where_the_host_polled_solve_stops(mesh):
    """tolerance-driven solves: the WHILE node of the graph stops at the iteration and residual of the direct path's
    host-polled batches, step after step; in the first step also at those of the blocking distributed step"""
    m = S.mesh(mesh)
    kw = dict(tol_abs=1e-7, tol_rel=0.0, max_restarts=100, max_iter=400)
    g, d, b = _dist(m, graph=True), _dist(m, graph=False), _dist(m)
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
    for s in (g, d, b):
        s.close()


@pytest.mark.parametrize("mesh", S.MESHES)
def test_six_enqueues_one_result_equal_six_pairs(mesh):
    m = S.mesh(mesh)
    a, b = _dist(m), _dist(m)
    for _ in range(6):
        a.step_enqueue(cfl=0.5, max_iter=8)
        ra = a.step_result()
    for _ in range(6):
        b.step_enqueue(cfl=0.5, max_iter=8)
    assert b.step_result() == ra
    _same(a, b)
    a.close()
    b.close()


@pytest.mark.parametrize("mesh", S.MESHES)
def test_pressure_enqueue_matches_the_blocking_pressure_section(mesh):
    m = S.mesh(mesh)
    nb = len(m[0])
    out = []
    for enq in (False, True):
        s = _dist(m)
        out.append(S.pressure_section(s, m, 0, nb, enq, max_iter=8))
        s.close()
    (it_a, err_a, fa), (it_b, err_b, fb) = out
    assert it_a == it_b == 8
    assert abs(err_a - err_b) <= 1e-9 * err_a
    for n in fa:
        assert S.rel(fb[n], fa[n]) <= S.FIELD_TOL, n


def test_adapt_between_enqueues_steps_like_a_fresh_distributed_context():
    """after cup2d_amr_adapt on the distributed context (graphs of the old mesh held), its enqueued steps, direct and then
    replayed, are bitwise those of a distributed context created on the new mesh with the same fields"""
    import amr_adapt_ranks as ar
    c = ar.case("three_level")
    m = (c["blocks"], 1, 1, c["h0"], ar.NU, c["fields"]["vel"], c["fields"]["pres"])
    a = _dist(m)
    for _ in range(2):                   # direct, then a graph of the old mesh
        a.step_enqueue(cfl=0.5, max_iter=5)
    a.step_result()
    for n, f in c["fields"].items():
        a.upload(n, f)
    assert a.adapt(c["rtol"], c["ctol"], c["level_max"], block_linf=c["linf"])
    new = a.block_list()
    assert a.rank_begin().tolist() == [0, len(new)]
    b = _dist((new, 1, 1, c["h0"], ar.NU, a.download("vel"), a.download("pres")))
    b.upload("chi", a.download("chi"))
    for _ in range(3):
        a.step_enqueue(cfl=0.5, max_iter=5)
        b.step_enqueue(cfl=0.5, max_iter=5)
        assert a.step_result() == b.step_result()
        _same(a, b)
    a.close()
    b.close()


def test_error_codes():
    """as tests/test_gpu_amr_step_graph.py::test_error_codes, on a distributed context"""
    from cup2d_b200 import lib as L
    m = S.mesh("synthetic")
    s = _dist(m)
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
    assert lib.cup2d_amr_step_result(h, None, None, None) == -4          # the refused calls left nothing pending
    assert np.array_equal(s.download("vel"), vel0)
    assert lib.cup2d_amr_set_graph(h, 1) == 0
    s.step_enqueue(cfl=0.5, max_iter=4)
    assert lib.cup2d_amr_step_result(h, None, None, None) == 0           # any output pointer may be NULL
    assert lib.cup2d_amr_step_result(h, None, None, None) == -4
    s.close()
    t = _dist(m)
    with pytest.raises(L.Cup2dError):
        t.step_result()
    t.close()
