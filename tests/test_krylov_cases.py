"""CPU tests of tests/krylov_cases.py: its restatement of the oracle's BiCGSTAB is the oracle bit for bit, and every case
the device tests (tests/test_gpu_krylov_branches.py) build meets its margins in the oracle."""
import numpy as np
import pytest

import cup2d_oracle as orc

import krylov_cases as kc
from krylov_cases import BREAKDOWNS, STALE, STOP_ITERS, stale_q


def bd_ids(cases=BREAKDOWNS):
    return [pytest.param(c, id=kc.case_id(c)) for c in cases]


def _runs():
    """(b, x0, keyword arguments) of every solve the device tests make, plus the tolerance-driven ones"""
    out = []
    for shape, seed, consistent in BREAKDOWNS:
        bd = kc.uniform_breakdown(*shape, seed, consistent)
        for mr in (0, 1, 2, 100):
            out.append((bd["b"], np.zeros_like(bd["b"]), dict(max_restarts=mr, max_iter=bd["kmax"])))
    b = orc.laplacian_neumann(stale_q(0))
    out.append((b, np.zeros_like(b), dict(max_error=3e-3, max_rel_error=0.0, max_restarts=100, max_iter=40)))
    out.append((b, np.zeros_like(b), dict(max_error=0.0, max_rel_error=1e-4, max_restarts=100, max_iter=40)))
    out.append((np.zeros_like(b), np.full_like(b, 0.375), dict(max_error=1e-8, max_restarts=100, max_iter=5)))
    return out


@pytest.mark.parametrize("i", range(len(_runs())))
def test_restatement_is_the_oracle_bitwise(i):
    b, x0, kw = _runs()[i]
    x, n, e, tr = kc.bicgstab_trace(b, x0, **kw)
    xr, nr, er = orc.bicgstab(b, x0, **kw)
    assert np.array_equal(x, xr) and n == nr and e == er
    assert len(tr["err"]) == len(tr["xsum"]) == n and tr["xsum"][-1] == xr.sum()


@pytest.mark.parametrize("case", bd_ids())
def test_breakdown_cases_meet_their_margins(case):
    shape, seed, consistent = case
    bd = kc.uniform_breakdown(*shape, seed, consistent)
    assert bd is not None
    kc.check_breakdown(bd)
    if consistent:   # the step's right-hand side for a fluid at rest with pressure -q is this b, bit for bit
        z = np.zeros_like(bd["q"])
        assert np.array_equal(orc.pressure_rhs1(orc.pressure_rhs(z, z, z, z, z, 0.1, 1e-3), -bd["q"]), bd["b"])


def test_breakdown_table():
    """the iterations before the breakdown and where the families break down (the oracle's restart of cuda.cu:457-477:
    rho = |r|^2 after it, and max_restarts = 1 ends the solve at the breakdown)"""
    got = {c: kc.uniform_breakdown(*c[0], c[1], c[2]) for c in BREAKDOWNS}
    assert [got[c]["k"] for c in BREAKDOWNS] == [7, 10, 9, 5]
    assert abs(got[BREAKDOWNS[0]]["c"] - 1.72343) < 1e-5 and abs(got[BREAKDOWNS[1]]["c"] + 0.71452) < 1e-5
    bd = got[BREAKDOWNS[0]]
    x, n, _, tr = kc.bicgstab_trace(bd["b"], np.zeros_like(bd["b"]), max_restarts=1, max_iter=bd["kmax"])
    assert n == bd["k"] == tr["restarts"][0] and len(tr["err"]) == n


@pytest.mark.parametrize("seed,K", STALE)
def test_stale_best_iterate_cases(seed, K):
    """the best iterate after K iterations is the oracle's x_opt, 0-3 iterations old, and where it is old the mean of the
    last iterate differs from its mean by more than 30 times the step's pressure tolerance of 1e-8 relative (so a sum
    of x taken from the wrong iterate shows in the pressure)"""
    b = orc.laplacian_neumann(stale_q(seed))
    ages = kc.stale_best(b, 16)
    assert ages == ({13: 1, 14: 2, 15: 3} if seed == 0 else {9: 1})
    x, _, _, tr = kc.bicgstab_trace(b, np.zeros_like(b), max_iter=K)
    if K in ages:
        assert abs(tr["x_last"].mean() - x.mean()) > 3e-7 * np.abs(x).max()


@pytest.mark.parametrize("k", STOP_ITERS)
def test_stop_tolerances_pick_exactly_one_iteration(k):
    b = orc.laplacian_neumann(stale_q(0))
    ta, tr_ = kc.stop_tolerance(b, k)
    for kw in (dict(max_error=ta), dict(max_rel_error=tr_)):
        assert orc.bicgstab(b, np.zeros_like(b), max_restarts=100, max_iter=100, **kw)[1] == k
        for f in (1 - 2e-5, 1 + 2e-5):   # the margins: 2e-5 relative either way does not move the stop
            kw2 = {key: val * f for key, val in kw.items()}
            assert orc.bicgstab(b, np.zeros_like(b), max_restarts=100, max_iter=100, **kw2)[1] == k


def test_the_eps_guards_depend_on_the_scale_of_b():
    """8 iterations on b s, divided by s, against 8 iterations on b: the 1e-21 guards are absolute, so at small scales
    the iteration is not scale invariant (a kernel without them passes no test at the scale of 1)"""
    q = np.random.default_rng(0).uniform(-1, 1, (24, 40))
    b = orc.laplacian_neumann(q)
    x1 = orc.bicgstab(b, np.zeros_like(b), max_iter=8)[0]
    d = {s: np.abs(orc.bicgstab(b * s, np.zeros_like(b), max_iter=8)[0] / s - x1).max() / np.abs(x1).max()
         for s in (1e-9, 1e-12, 1e-150, 1e100)}
    assert d[1e-9] > 1e-3 and d[1e-12] > 1e-1 and d[1e-150] > 1e-1 and d[1e100] < 1e-12, d
