"""A time step starts its Poisson solve inside the kernel that forms the right-hand side.

The step's right-hand-side kernel used to write b to tmp and x0 = 0 to pres, and k_init read both back to form r = b - A*0,
r^ = r and x = x0.  pressure_rhs_start_kernel forms b with the same expression and writes r = r^ = b and x = 0 directly, on
k_init's grid and row partition, so the Krylov state it leaves is bitwise k_init's.  Iteration 0 of the tile path then reads
neither r^ (it equals r) nor x (it is +0).  The stand-alone entry points keep the old composition (cup2d_pressure_rhs writes
tmp and pres, cup2d_poisson_solve starts from them through k_init), so it serves as the yardstick here: after every step,
vel and pres, dt, the iteration count and the residual are bitwise those of

    compute_dt -> advect_diffuse_rk2 -> pressure_rhs -> poisson_solve -> pressure_correct

on a second context with the same blocks, with bodies (keep_udef = 1).  Without bodies the step's right-hand side leaves
out the chi * div(u_def) term, which the stand-alone one always includes: with chi = 0 the term is zero, but the compiler
contracts fac * div(vel) into a different FMA in the two instantiations, so b differs in the last bit and the fields within
1e-11 (p) and 1e-13 (u, v) of their maximum, dt from the second step on within 1e-12, the same iteration count.  That path is checked bit for bit
against the previous build by bench.py --dump-outputs instead.  General-rows contexts cannot step (they are Poisson-only),
so the general-rows path of a solve keeps k_init and is covered by the existing Krylov tests.

GPU tests run with -m gpu; the CPU tests run a subset of them, and the same comparison on two ranks, on the emulated library
(tests/host_emu/build.py)."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
K = 10
NU, CFL = 1e-3, 0.5

# (bpdx, bpdy, level), block order: square and rectangular domains, partial tiles, Hilbert and other orders
CASES = [((1, 1, 3), "hilbert"), ((3, 2, 1), "hilbert"), ((5, 3, 1), "random"), ((3, 5, 1), "col"), ((2, 1, 2), "rhilbert"),
         ((7, 1, 1), "row")]


def _fields(NX, NY, seed):
    rng = np.random.default_rng(seed)
    X, Y = np.meshgrid((np.arange(NX) + 0.5) / NX, (np.arange(NY) + 0.5) / NY)
    u = np.sin(2 * np.pi * X) * np.cos(2 * np.pi * Y) + 0.05 * rng.uniform(-1, 1, (NY, NX))
    v = -np.cos(2 * np.pi * X) * np.sin(2 * np.pi * Y) + 0.05 * rng.uniform(-1, 1, (NY, NX))
    p = np.cos(2 * np.pi * X) * np.cos(2 * np.pi * Y) + 0.05 * rng.uniform(-1, 1, (NY, NX))
    chi = np.exp(-((X - 0.4) ** 2 + (Y - 0.55) ** 2) / 0.02)
    return u, v, p, chi


def _pair(shape, kind, bodies, seed=3, **kw):
    import cup2d_b200
    from block_orders import make_order
    bpdx, bpdy, level = shape
    order = make_order(bpdx, bpdy, level, kind)
    sims = [cup2d_b200.Simulation(level, bpdx=bpdx, bpdy=bpdy, nu=NU, cfl=CFL, order=order, **kw) for _ in range(2)]
    u, v, p, chi = _fields(sims[0].NX, sims[0].NY, seed)
    for s in sims:
        s.upload("vel", u, v)
        s.upload("pres", p)
        if bodies:
            s.upload("chi", chi)
    return sims


def _composed_step(sim, bodies, tol, max_restarts):
    """one step through the stand-alone entry points: right-hand side into tmp / pres, solve from them (k_init)"""
    _, dt = sim.compute_dt()
    sim.rk2(dt)
    sim.pressure_rhs(dt)   # with bodies: tmpV holds what the fused step reads as u_def (the RK scratch), as in the step
    it, err = sim.poisson_solve(tol, tol, max_restarts, K if tol == 0 else 200)
    sim.pressure_correct(dt)
    return dt, it, err


def _check_steps(fused, composed, bodies, tol, max_restarts, nsteps=3):
    for n in range(nsteps):   # step 1 runs kernel by kernel, steps 2 and 3 are captured into (and run as) step graphs
        got = fused.step(dt=0.0, keep_udef=bodies, tol_abs=tol, tol_rel=tol, max_restarts=max_restarts,
                         max_iter=K if tol == 0 else 200)
        want = _composed_step(composed, bodies, tol, max_restarts)
        if bodies:
            assert got == want, (n, got, want)
        else:
            assert got[1] == want[1] and abs(got[0] - want[0]) <= 1e-12 * want[0] and abs(got[2] - want[2]) <= 1e-10 * want[2], \
                (n, got, want)
        for name, bound in (("vel", 1e-13), ("pres", 1e-11)):
            a, b = fused.download_blocks(name), composed.download_blocks(name)
            if bodies:
                assert np.array_equal(a.view(np.uint64), b.view(np.uint64)), (n, name, np.abs(a - b).max())
            else:
                assert np.abs(a - b).max() <= bound * np.abs(b).max(), (n, name, np.abs(a - b).max() / np.abs(b).max())


@pytest.mark.gpu
@pytest.mark.parametrize("bodies", [False, True], ids=["no_bodies", "bodies"])
@pytest.mark.parametrize("shape,kind", CASES, ids=[f"{s[0]}x{s[1]}L{s[2]}_{k}" for s, k in CASES])
def test_steps_bitwise_equal_the_standalone_composition(shape, kind, bodies):
    """fixed work as bench.py runs it (10 iterations, tolerance 0, no restarts), three steps"""
    fused, composed = _pair(shape, kind, bodies)
    _check_steps(fused, composed, bodies, 0.0, 0)
    fused.close()
    composed.close()


@pytest.mark.gpu
@pytest.mark.parametrize("shape,kind", CASES[:3], ids=[f"{s[0]}x{s[1]}L{s[2]}_{k}" for s, k in CASES[:3]])
def test_tolerance_driven_steps_bitwise_equal_the_standalone_composition(shape, kind):
    """tolerance-driven solves with restarts allowed: the same stopping iteration (graph WHILE node from step 2 on)"""
    fused, composed = _pair(shape, kind, True, seed=11)
    _check_steps(fused, composed, True, 1e-7, 100)
    fused.close()
    composed.close()


@pytest.mark.gpu
def test_standalone_solve_after_steps_reads_its_x0():
    """a solve from an arbitrary x0 on a context that has stepped: iteration 0 reads x again (the start iterate is +0 only in
    a step), so the result is bitwise that of a context that never stepped"""
    stepped, fresh = _pair((3, 2, 1), "hilbert", False)
    for _ in range(2):
        stepped.step(dt=0.0, max_iter=K, max_restarts=0)
    rng = np.random.default_rng(5)
    b, x0 = rng.uniform(-1, 1, (2, stepped.NY, stepped.NX))
    b -= b.mean()
    for s in (stepped, fresh):
        s.upload("tmp", b)
        s.upload("pres", x0)
    assert stepped.poisson_solve(0.0, 0.0, 0, 7) == fresh.poisson_solve(0.0, 0.0, 0, 7)
    assert np.array_equal(stepped.download_blocks("pres"), fresh.download_blocks("pres"))
    stepped.close()
    fresh.close()


# ---- the same on the emulated library (CPU) ----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emulated_library():
    sys.path.insert(0, os.path.join(HERE, "host_emu"))
    import build
    return build.build_full()


def test_step_start_subset_on_the_emulated_library(emulated_library):
    env = dict(os.environ, CUP2D_B200_LIB=emulated_library)
    r = subprocess.run([sys.executable, "-m", "pytest", __file__, "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider",
                        "-k", "(test_steps_bitwise and 5x3L1) or reads_its_x0"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env, timeout=900, cwd=ROOT)
    tail = r.stdout[-1500:]
    assert r.returncode == 0, tail
    assert " passed" in tail and "failed" not in tail
    assert int(tail.split(" passed")[0].split()[-1]) == 3, tail


def test_two_rank_steps_bitwise_equal_the_standalone_composition_emulated(emulated_library):
    """two ranks as threads of one process (the five-kernel path, all-reduced sums, halo refreshes of vel, u_def and pold):
    on every rank, two fused steps with bodies are bitwise the stand-alone composition on the same two ranks"""
    code = r'''
import sys, threading
sys.path[:0] = [%r, %r, %r]
import test_step_start_fusion as T
W = 2
bar, slots, errs = threading.Barrier(W), [None] * W, []
class Dist:                       # in-process stand-in for torch.distributed (only carries the opaque blobs)
    def __init__(self, rank): self.rank = rank
    def all_gather_object(self, out, obj):
        slots[self.rank] = obj; bar.wait()
        out[:] = slots; bar.wait()
    def barrier(self): bar.wait()
def run(rank):
    try:
        sims = T._pair((2, 1, 2), "hilbert", True, rank=rank, nranks=W)
        for s in sims:
            s.attach_peers(Dist(rank))
        T._check_steps(sims[0], sims[1], True, 0.0, 0, nsteps=2)
        bar.wait()
        for s in sims:
            s.close()
    except BaseException as e:
        errs.append(repr(e)); bar.abort()
ths = [threading.Thread(target=run, args=(r,)) for r in range(W)]
[t.start() for t in ths]; [t.join() for t in ths]
assert not errs, errs
print("SAME")
''' % (ROOT, HERE, os.path.join(ROOT, "oracle"))
    r = subprocess.run([sys.executable, "-c", code], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900,
                       env=dict(os.environ, CUP2D_B200_LIB=emulated_library))
    assert r.returncode == 0 and "SAME" in r.stdout, r.stdout[-1500:]
