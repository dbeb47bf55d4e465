"""The enqueued multi-level steps on distributed contexts with several ranks (tests/amr_step_ranks.py), on the CPU against a
g++ build of the product sources (tests/host_emu/build.py build_full) with 2 and 3 ranks running as threads of one process:
their device buffers are mapped into each other through the emulated IPC handles, so the halo pulls and the in-kernel
all-reduces of dt's maximum and of the pressure means run as they do across GPUs.  Graphs do not exist there: every
enqueue takes the direct path, a tolerance-driven solve polled by the host every 8 iterations.  Each partition moves its
cuts onto level interfaces (coarse side on one rank, fine side on the next)."""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def emulated_library():
    sys.path.insert(0, os.path.join(HERE, "host_emu"))
    import build
    return build.build_full()


def _run(code, lib):
    r = subprocess.run([sys.executable, "-c", "import sys\nsys.path.insert(0, %r)\n" % HERE + code], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=1800, env=dict(os.environ, CUP2D_B200_LIB=lib), cwd=ROOT)
    assert r.returncode == 0 and "DONE" in r.stdout, r.stdout[-3000:]
    return r.stdout


def test_enqueued_steps_on_two_and_three_ranks_emulated(emulated_library):
    """2 steps, dt on the device, 8 fixed iterations: dt bitwise the blocking distributed dt rule, dt / iterations / residual
    the same bits on every rank, iterations those of the blocking distributed step, fields within 1e-13 of it and of the
    plain context's enqueued steps"""
    code = r'''
import numpy as np
import amr_step_ranks as S
m = S.mesh("synthetic")
p = S.make(m)
plain, fp = S.run_steps(p, 2, True, max_iter=8)
p.close()
def run(rb, enqueued):
    def fn(rank, dist, barrier):
        s = S.make(m, rank, rb, dist)
        r = S.run_steps(s, 2, enqueued, check_dt=enqueued, max_iter=8)
        barrier(); s.close()
        return r
    res = S.on_threads(len(rb) - 1, fn)
    for r, _ in res[1:]:
        assert r == res[0][0], "ranks disagree"
    return res[0][0], {n: np.concatenate([f[n] for _, f in res]) for n in ("vel", "pres")}
for W in (2, 3):
    rb = S.level_cut(m, W)
    enq, fe = run(rb, True)
    blk, fb = run(rb, False)
    assert [r[1] for r in enq] == [r[1] for r in blk] == [8, 8]
    assert enq[0][0] == blk[0][0]                      # the same velocity before the first step
    assert abs(enq[1][0] - blk[1][0]) <= 1e-13 * blk[1][0]
    worst = max(max(S.rel(fe[n], fb[n]), S.rel(fe[n], fp[n])) for n in fe)
    assert worst <= S.FIELD_TOL, worst
    assert all(abs(e[0] - q[0]) <= 1e-13 * q[0] and e[1] == q[1] for e, q in zip(enq, plain))
    print(W, rb.tolist(), enq, "worst", worst, flush=True)
print("DONE")
'''
    print(_run(code, emulated_library)[-800:])


def test_tolerance_driven_solve_and_pressure_enqueue_on_two_ranks_emulated(emulated_library):
    """a tolerance-driven solve stops at the blocking distributed step's iteration; the pressure section after shape_set +
    udef_assemble, enqueued, within 1e-13 of the blocking one"""
    code = r'''
import numpy as np
import amr_step_ranks as S
m = S.mesh("synthetic")
rb = S.level_cut(m, 2)
kw = dict(tol_abs=1e-4, tol_rel=0.0, max_restarts=100, max_iter=400)
def both(fn):
    out = []
    for enqueued in (True, False):
        res = S.on_threads(2, lambda rank, dist, barrier: fn(rank, dist, barrier, enqueued))
        assert all(r[:2] == res[0][:2] for r in res[1:]), "ranks disagree"
        out.append((res[0][:2], {n: np.concatenate([r[2][n] for r in res]) for n in ("vel", "pres")}))
    return out
def step(rank, dist, barrier, enqueued):
    s = S.make(m, rank, rb, dist)
    (r,), f = S.run_steps(s, 1, enqueued, **kw)
    barrier(); s.close()
    return r[0], r[1:], f
(e, fe), (b, fb) = both(step)
assert e == b and 8 < e[1][0] < 400, (e, b)     # same dt, then the same iteration and residual
worst = max(S.rel(fe[n], fb[n]) for n in fe)
assert worst <= S.FIELD_TOL, worst
print("tolerance", e, worst, flush=True)
def pressure(rank, dist, barrier, enqueued):
    s = S.make(m, rank, rb, dist)
    it, err, f = S.pressure_section(s, m, int(rb[rank]), int(rb[rank + 1]), enqueued, max_iter=8)
    barrier(); s.close()
    return it, err, f
(e, fe), (b, fb) = both(pressure)
assert e[0] == b[0] == 8 and abs(e[1] - b[1]) <= 1e-9 * b[1], (e, b)
worst = max(S.rel(fe[n], fb[n]) for n in fe)
assert worst <= S.FIELD_TOL, worst
print("pressure", e, worst, flush=True)
print("DONE")
'''
    print(_run(code, emulated_library)[-800:])


def test_enqueue_before_peer_attach_is_refused_emulated(emulated_library):
    """two ranks created without cup2d_amr_peer_attach: CUP2D_ESTATE from both enqueue calls, nothing pending, fields
    untouched"""
    code = r'''
import ctypes as C
import numpy as np
import amr_step_ranks as S
from cup2d_b200 import lib as L
lib = L.load_library()
blocks, bx, by, h0, nu, vel, pres = S.mesh("synthetic")
allb = np.ascontiguousarray(blocks, dtype=np.int32)
rb = S.level_cut(S.mesh("synthetic"), 2)
for rank in (0, 1):
    h = C.c_void_p()
    L.check(lib.cup2d_amr_create_ranks(len(allb), allb.ctypes.data_as(C.POINTER(C.c_int32)), bx, by, h0, nu, rank, 2,
                                       rb.ctypes.data_as(C.POINTER(C.c_int64)), 0, C.byref(h)))
    b0, b1 = int(rb[rank]), int(rb[rank + 1])
    v0, p0 = np.ascontiguousarray(vel[b0:b1]), np.ascontiguousarray(pres[b0:b1])
    L.check(lib.cup2d_amr_field_upload(h, L.FIELDS["vel"], v0.ctypes.data_as(C.c_void_p)))
    L.check(lib.cup2d_amr_field_upload(h, L.FIELDS["pres"], p0.ctypes.data_as(C.c_void_p)))
    assert lib.cup2d_amr_step_enqueue(h, 0.5, 0.0, 0.0, 0.0, 0, 8) == -4
    assert "peer_attach" in lib.cup2d_last_error().decode()
    assert lib.cup2d_amr_step_enqueue(h, 0.5, 1e-3, 0.0, 0.0, 0, 8) == -4
    assert lib.cup2d_amr_pressure_enqueue(h, 1e-3, 0.0, 0.0, 0, 8) == -4
    assert lib.cup2d_amr_step_result(h, None, None, None) == -4        # nothing pending
    for name, want in (("vel", v0), ("pres", p0)):
        got = np.empty_like(want)
        L.check(lib.cup2d_amr_field_download(h, L.FIELDS[name], got.ctypes.data_as(C.c_void_p)))
        assert np.array_equal(got, want), name
    lib.cup2d_amr_destroy(h)
print("DONE")
'''
    _run(code, emulated_library)
