"""GPU tests (-m gpu) of the branches of the device BiCGSTAB loop (csrc/poisson.cu): the breakdown restart and the restart
cap, the best iterate when it is not the last, the exact stopping iteration under tol_abs and tol_rel, and degenerate
right-hand sides.  The loop's control flow runs on the device (prepare_iteration / end_of_iteration in the last CTA of a
kernel); the right-hand sides that reach each branch with a clear margin come from tests/krylov_cases.py.

  * restart on the three-kernel tile path (k_p_spmv), on the five-kernel path (k_pupdate) of a Poisson-only context with
    the same neighbour table, and inside the captured step graph with its WHILE node: the oracle's count exactly (with
    max_restarts = 1 the breakdown iteration), the iterate to 1e-9 and the two paths to 1e-12 relative;
  * the best iterate 1-3 iterations old: x, err and, through the step, the pressure whose mean comes from st->xsum;
  * tol_abs / tol_rel set between two successive minima: the solve stops at exactly that iteration, host-polled (batches
    of 8) and in the WHILE node;
  * b = 0 (a fluid at rest), b scaled by 1e-150 ... 1e100 (the 1e-21 guards are absolute, so the scale changes the
    iteration): the oracle's count and iterate, no NaN."""
import os
import subprocess
import sys

import numpy as np
import pytest

import cup2d_b200
import cup2d_oracle as orc

import krylov_cases as kc
from block_orders import make_order
from krylov_cases import BREAKDOWNS, STALE, STOP_ITERS, stale_q
from test_gpu_block_orders import five_kernel_solve, neighbour_table

pytestmark = pytest.mark.gpu

NU, CFL, DT = 1e-3, 0.5, 1e-3
GAPS = {}   # largest gap of each kind over the module, printed at its end (pytest -s)


def gap(kind, value):
    GAPS[kind] = max(GAPS.get(kind, 0.0), float(value))
    return value


@pytest.fixture(scope="module", autouse=True)
def report_gaps():
    yield
    for kind, value in sorted(GAPS.items()):
        print(f"\nlargest gap {kind}: {value:.3g}")


def bd_ids(cases=BREAKDOWNS):
    return [pytest.param(c, id=kc.case_id(c)) for c in cases]


def make_sim(shape, kind="hilbert"):
    bpdx, bpdy, level = shape
    return cup2d_b200.Simulation(level, bpdx=bpdx, bpdy=bpdy, order=make_order(bpdx, bpdy, level, kind), nu=NU, cfl=CFL)


def solve_three(sim, b, x0, **kw):
    """poisson_solve of a uniform-grid context (the three-kernel iteration): (iterations, err, x)"""
    sim.upload("tmp", b)
    sim.upload("pres", x0)
    it, err = sim.poisson_solve(**kw)
    return it, err, sim.download("pres")


def solve_five(sim, b, x0, max_iter=1000, **kw):
    """the same solve on a Poisson-only context built from sim's neighbour table (the five-kernel iteration)"""
    it, err, xb = five_kernel_solve(neighbour_table(sim), cup2d_b200.to_blocks(b, sim.local_order, sim.nbx), max_iter,
                                    cup2d_b200.to_blocks(x0, sim.local_order, sim.nbx), **kw)
    return it, err, cup2d_b200.from_blocks(xb, sim.local_order, sim.nbx, sim.nby, 1)


def assert_vs_oracle(got, want):
    """count exactly, iterate to 1e-9, residual to 1e-9 max(1, err) (as tests/test_gpu_parity.py)"""
    it, err, x = got
    xr, itr, errr = want
    assert it == itr, (it, itr)
    assert gap("x vs oracle (abs)", np.abs(x - xr).max()) < 1e-9, np.abs(x - xr).max()
    assert gap("err vs oracle (rel max(1, err))", abs(err - errr) / max(1.0, errr)) < 1e-9, (err, errr)


def assert_paths_agree(a, b, r0):
    assert a[0] == b[0]
    assert gap("x three vs five kernels (rel)", np.abs(a[2] - b[2]).max() / np.abs(b[2]).max()) <= 1e-12
    assert gap("err three vs five kernels (rel |b|)", abs(a[1] - b[1]) / r0) <= 1e-12


def rest_steps(shape, kind, q, graph, n, dt=DT, **kw):
    """n steps of a fluid at rest (vel = 0, chi = 0) from the pressure -q, the fields re-uploaded before every step: the
    step's right-hand side is b = -lap(pold) = A q.  graph: the first step runs directly, the second and third capture
    the two buffer assignments' graphs, the fourth replays the first graph.  -> [(dt, iterations, err, u, v, p)]"""
    sim = make_sim(shape, kind)
    sim.set_graph(graph)
    z = np.zeros_like(q)
    out = []
    for _ in range(n):
        sim.upload("vel", z, z)
        sim.upload("pres", -q)
        sim.step_enqueue(dt=dt, **kw)
        out.append((*sim.step_result(), *sim.download("vel"), sim.download("pres")))
    sim.close()
    return out


def assert_step_vs_oracle(got, q, **kw):
    """the tolerances of tests/test_gpu_block_orders.py::test_step_any_order_vs_oracle"""
    z = np.zeros_like(q)
    ref = orc.step(z, z, -q, NU, CFL, dt=DT, **kw)
    dt, it, err, gu, gv, gp = got
    assert dt == DT and it == ref["iters"], (it, ref["iters"])
    scale = max(np.abs(ref["u"]).max(), np.abs(ref["v"]).max())
    assert gap("step u, v vs oracle (rel)", max(np.abs(gu - ref["u"]).max(), np.abs(gv - ref["v"]).max()) / scale) <= 1e-9
    assert gap("step p vs oracle (rel)", np.abs(gp - ref["p"]).max() / np.abs(ref["p"]).max()) <= 1e-8
    return ref


# ---- 3a / 3b: restart on the three- and five-kernel paths ---------------------------------------------------------------
@pytest.mark.parametrize("kind", ["hilbert", "random"])
@pytest.mark.parametrize("case", bd_ids())
def test_restart_three_and_five_kernels_vs_oracle(case, kind):
    """max_iter = breakdown + 6.  max_restarts = 100 restarts, 1 stops at the breakdown: both to 1e-9 of the oracle and
    1e-12 between the paths.  max_restarts = 0 iterates on through the breakdown, where rho = r-hat.r is a cancellation
    that has lost about 12 digits: from there on the iterates of any two implementations drift apart (the oracle's own
    move by up to 7e-3 for a 1e-14 relative change of b).  That run is held to a tenth of the difference restarting
    makes, which a path that restarted anyway (or never) would exceed tenfold."""
    shape, seed, consistent = case
    bd = kc.uniform_breakdown(*shape, seed, consistent)
    b, k, K = bd["b"], bd["k"], bd["kmax"]
    x0 = np.zeros_like(b)
    ora = np.abs(bd["x100"] - bd["x0"]).max()
    sim = make_sim(shape, kind)
    try:
        for mr in (0, 1, 100):
            want = orc.bicgstab(b, x0, max_restarts=mr, max_iter=K)
            assert want[1] == (k if mr == 1 else K)
            three = solve_three(sim, b, x0, max_restarts=mr, max_iter=K)
            five = solve_five(sim, b, x0, max_restarts=mr, max_iter=K)
            if mr:
                assert_vs_oracle(three, want)
                assert_paths_agree(three, five, np.abs(b).max())
                continue
            for it, err, x in (three, five):
                assert it == K and abs(err - want[2]) <= 2e-2 * want[2]
                assert gap("max_restarts=0 x vs oracle (fraction of the restart's change)",
                           np.abs(x - want[0]).max() / ora) <= 0.1, np.abs(x - want[0]).max() / ora
    finally:
        sim.close()


# ---- 3d: restart inside the captured step graph ---------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["hilbert", "random"])
@pytest.mark.parametrize("case", bd_ids([c for c in BREAKDOWNS if c[2]]))
def test_restart_inside_the_step_graph(case, kind):
    """tol_abs = 1e-300: the graph's solve is a WHILE node that never converges, so it runs max_iter iterations with the
    restart in the middle; max_restarts = 1: the WHILE node ends at the breakdown"""
    shape, seed, _ = case
    bd = kc.uniform_breakdown(*shape, seed, True)
    q, k, K = bd["q"], bd["k"], bd["kmax"]
    for mr, iters in ((100, K), (1, k)):
        kw = dict(tol_abs=1e-300, max_restarts=mr, max_iter=K)
        direct = rest_steps(shape, kind, q, False, 1, **kw)[0]
        graph = rest_steps(shape, kind, q, True, 4, **kw)
        assert direct[1] == iters
        for g in graph:
            assert g[:3] == direct[:3] and all(np.array_equal(a, c) for a, c in zip(g[3:], direct[3:]))
        assert_step_vs_oracle(direct, q, kiter=K, tol=1e-300, max_restarts=mr)


# ---- 3e: the best iterate is not the last -----------------------------------------------------------------------------
@pytest.mark.parametrize("seed,K", STALE)
def test_best_iterate_older_than_the_last(seed, K):
    """6x4 blocks, b = A q: after K iterations the best iterate is 0-3 iterations old (tests/test_krylov_cases.py);
    poisson_solve returns it and its residual, and the step's pressure (whose mean comes from the sum of the best
    iterate) is the oracle's although the last iterate's mean differs by more than the pressure tolerance.  The steps run
    directly, then from the graph: with tol_abs = 0 its K unrolled iterations, with tol_abs = 1e-300 its WHILE node, which
    then ends on iteration K although that iteration (K = 13, 14, 15, 9) does not improve"""
    q = stale_q(seed)
    b = orc.laplacian_neumann(q)
    x0 = np.zeros_like(b)
    sim = make_sim((3, 2, 1), "random")
    try:
        assert_vs_oracle(solve_three(sim, b, x0, max_iter=K), orc.bicgstab(b, x0, max_iter=K))
    finally:
        sim.close()
    for tol in (0.0, 1e-300):
        steps = rest_steps((3, 2, 1), "random", q, True, 2, tol_abs=tol, max_iter=K)
        assert steps[0][:3] == steps[1][:3] and all(np.array_equal(a, c) for a, c in zip(steps[0][3:], steps[1][3:]))
        ref = assert_step_vs_oracle(steps[1], q, kiter=K, tol=tol)
    x_opt, _, _, tr = kc.bicgstab_trace(b, x0, max_iter=K)
    if kc.stale_best(b, K).get(K):
        assert abs(tr["x_last"].mean() - x_opt.mean()) > 1e-8 * np.abs(ref["p"]).max()


# ---- 3f: exact stopping iteration -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["abs", "rel"])
@pytest.mark.parametrize("k", STOP_ITERS)
def test_stops_at_exactly_the_iteration_the_tolerance_picks(k, mode):
    q = stale_q(0)
    b = orc.laplacian_neumann(q)
    x0 = np.zeros_like(b)
    ta, tr_ = kc.stop_tolerance(b, k)
    kw = dict(tol_abs=ta, tol_rel=0.0) if mode == "abs" else dict(tol_abs=0.0, tol_rel=tr_)
    want = orc.bicgstab(b, x0, kw["tol_abs"], kw["tol_rel"], 100, 100)
    assert want[1] == k
    sim = make_sim((3, 2, 1), "hilbert")
    try:
        assert_vs_oracle(solve_three(sim, b, x0, max_restarts=100, max_iter=100, **kw), want)
        assert_vs_oracle(solve_five(sim, b, x0, max_restarts=100, max_iter=100, **kw), want)
    finally:
        sim.close()
    steps = rest_steps((3, 2, 1), "hilbert", q, True, 2, max_restarts=100, max_iter=100, **kw)
    assert [s[1] for s in steps] == [k, k]   # host-polled (first step), then the WHILE node
    for s in steps:
        assert_step_vs_oracle(s, q, kiter=100, tol=kw["tol_abs"], tol_rel=kw["tol_rel"], max_restarts=100)


# ---- 3g: degenerate right-hand sides --------------------------------------------------------------------------------------
@pytest.mark.parametrize("x0val", [0.0, 0.375])
@pytest.mark.parametrize("tol", [(0.0, 0.0), (1e-8, 0.0), (0.0, 1e-6)])
def test_zero_rhs_returns_x0_after_max_iter(x0val, tol):
    """b = 0 and x0 = constant (a dyadic constant: r0 = b - A x0 = 0 exactly): err_init = 0 and no iteration improves
    (0 < 0 is false), so the solve runs max_iter no-op iterations and returns x0, with every 0/0 guarded by the 1e-21"""
    shape = (5, 3, 0)
    sim = make_sim(shape, "random")
    b = np.zeros((sim.NY, sim.NX))
    x0 = np.full_like(b, x0val)
    K = 11
    want = orc.bicgstab(b, x0, tol[0], tol[1], 100, K)
    assert want[1] == K and want[2] == 0.0 and np.array_equal(want[0], x0)
    try:
        for got in (solve_three(sim, b, x0, tol_abs=tol[0], tol_rel=tol[1], max_restarts=100, max_iter=K),
                    solve_five(sim, b, x0, tol_abs=tol[0], tol_rel=tol[1], max_restarts=100, max_iter=K)):
            assert got[0] == K and got[1] == 0.0 and np.array_equal(got[2], x0)
    finally:
        sim.close()


def test_fluid_at_rest_stays_at_rest_in_the_step_graph():
    shape = (5, 3, 0)
    q = np.zeros((24, 40))
    for dt in (DT, 0.0):   # given dt, and dt control on the device (umax = 0)
        for s in rest_steps(shape, "random", q, True, 3, dt=dt, tol_abs=1e-8, tol_rel=1e-6, max_restarts=100, max_iter=9):
            assert s[0] > 0 and s[1] == 9 and s[2] == 0.0
            assert all(np.array_equal(f, q) for f in s[3:])


@pytest.mark.parametrize("scale", [1e-9, 1e-12, 1e-150, 1e100])
def test_scaled_rhs_three_and_five_kernels_vs_oracle(scale):
    """the 1e-21 guards are absolute: at the small scales the iterates are not the scaled iterates of b (the oracle's
    differ by 3 % at 1e-9, tests/test_krylov_cases.py), and the device must follow the oracle, not the scaled solution"""
    shape = (5, 3, 0)
    q = np.random.default_rng(0).uniform(-1, 1, (24, 40))
    b = orc.laplacian_neumann(q) * scale
    x0 = np.zeros_like(b)
    K = 8
    want = orc.bicgstab(b, x0, max_iter=K)
    sim = make_sim(shape, "random")
    try:
        for got in (solve_three(sim, b, x0, max_iter=K), solve_five(sim, b, x0, max_iter=K)):
            assert got[0] == want[1] == K
            assert np.isfinite(got[2]).all()
            assert np.abs(got[2] - want[0]).max() <= 1e-9 * np.abs(want[0]).max()
            assert abs(got[1] - want[2]) <= 1e-9 * want[2]
    finally:
        sim.close()


# ---- several ranks ----------------------------------------------------------------------------------------------------------
RANKS_SCRIPT = r'''
import os, sys
sys.path[:0] = [%r, %r, %r]
import torch, torch.distributed as dist
import krylov_cases as kc
rank, world, lrank = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(lrank)
dist.init_process_group("nccl", device_id=torch.device("cuda", lrank))
mine = kc.restart_on_ranks(rank, world, dist, device=lrank)
parts = [None] * world
dist.all_gather_object(parts, mine)
if rank == 0:
    print("WORST", kc.check_ranks(parts, kc.restart_on_ranks(0, 1, None, device=lrank)))
dist.barrier()
dist.destroy_process_group()
'''


def test_restart_on_two_gpus_matches_one(tmp_path):
    """the breakdown case on two ranks on two GPUs (skipped on a one-GPU box): k_pupdate pushes p = r and z = M p to the
    peer, every rank decides the restart on all-reduced sums.  max_restarts 1 and 100: the one-rank count and residual,
    the iterate to 1e-10 (the three-rank emulation of the same case: tests/test_full_emulation.py)"""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    script = tmp_path / "restart_ranks.py"
    script.write_text(RANKS_SCRIPT % (root, here, os.path.join(root, "oracle")))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29579", str(script)],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0 and "WORST" in r.stdout, r.stdout[-2000:]
