"""GPU parity tests (-m gpu): the CUDA path, called through the C ABI, against
  (1) golden outputs of the unmodified reference (tests/golden/*.npz), and
  (2) the numpy oracle on seeded inputs at sizes the oracle finishes in seconds,
  (3) size-independent properties at large sizes.
Tolerances: the contract is L-inf(u,p) < 1e-6 (BASELINE.json); operators are held to 1e-12 relative
(FMA contraction and the single-division WENO weights change rounding only), Krylov results at equal
iteration count to 1e-9 (dot-product summation order differs)."""
import os

import numpy as np
import pytest

import cup2d_b200
import cup2d_oracle as orc

pytestmark = pytest.mark.gpu


def rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def make_fields(N, seed, kind="tg"):
    rng = np.random.default_rng(seed)
    x = (np.arange(N) + 0.5) / N
    X, Y = np.meshgrid(x, x)
    if kind == "random":
        u, v, p = (rng.uniform(-1, 1, (N, N)) for _ in range(3))
    else:
        u = np.sin(2 * np.pi * X) * np.cos(2 * np.pi * Y) + 0.05 * rng.uniform(-1, 1, (N, N))
        v = -np.cos(2 * np.pi * X) * np.sin(2 * np.pi * Y) + 0.05 * rng.uniform(-1, 1, (N, N))
        p = np.cos(2 * np.pi * X) * np.cos(2 * np.pi * Y)
    chi = np.exp(-((X - 0.4) ** 2 + (Y - 0.55) ** 2) / 0.02)
    udu, udv = 0.3 * np.sin(3 * X + Y), 0.2 * np.cos(2 * Y - X)
    return u, v, p, chi, udu, udv


@pytest.mark.parametrize("name", ["ops_L2_random", "ops_L3_tg"])
def test_operators_vs_reference_golden(golden_dir, name):
    d = np.load(os.path.join(golden_dir, name + ".npz"))
    L, nu, dt = int(d["L"]), float(d["nu"]), float(d["dt"])
    sim = cup2d_b200.Simulation(L, nu=nu)
    sim.upload("vel", d["u"], d["v"])
    sim.advect_diffuse_rhs(dt)
    au, av = sim.download("tmpV")
    assert rel(au, d["adv_u"]) < 1e-12 and rel(av, d["adv_v"]) < 1e-12
    # pressure_rhs: tmp = rhs(vel, udef, chi) - lap(pold) with pold = previous pres
    sim.upload("tmpV", d["udef_u"], d["udef_v"])
    sim.upload("chi", d["chi"])
    sim.upload("pres", d["p"])
    sim.pressure_rhs(dt)
    assert rel(sim.download("tmp"), d["rhs1"]) < 1e-13
    assert np.array_equal(sim.download("pold"), d["p"])
    assert np.abs(sim.download("pres")).max() == 0.0
    sim.close()


@pytest.mark.parametrize("name", ["steps_L2_tg_k12", "steps_L2_random_k8", "steps_L3_tg_k15"])
def test_time_steps_vs_reference_golden(golden_dir, name):
    d = np.load(os.path.join(golden_dir, name + ".npz"))
    L, nu, cfl, K = int(d["L"]), float(d["nu"]), float(d["cfl"]), int(d["kiter"])
    sim = cup2d_b200.Simulation(L, nu=nu, cfl=cfl)
    sim.upload("vel", d["u0"], d["v0"])
    sim.upload("pres", d["p0"])
    for s in range(len(d["dt"])):
        dt, iters, err = sim.step(max_iter=K)
        assert abs(dt - d["dt"][s]) < 1e-15 and iters == K
        u, v = sim.download("vel")
        p = sim.download("pres")
        assert np.abs(u - d["u"][s]).max() < 1e-9 and np.abs(v - d["v"][s]).max() < 1e-9
        assert np.abs(p - d["p"][s]).max() < 1e-9
    sim.close()


@pytest.mark.parametrize("L,kind,seed", [(0, "random", 1), (1, "random", 2), (2, "tg", 3), (5, "tg", 4), (5, "random", 5), (6, "tg", 6)])
def test_advect_stage_vs_oracle(L, kind, seed):
    """Covers grids smaller than one tile (L=0,1: 8^2, 16^2 cells), one tile, and many tiles."""
    N = 8 << L
    u, v, *_ = make_fields(N, seed, kind)
    nu, dt = 1e-3, 0.3 / N
    sim = cup2d_b200.Simulation(L, nu=nu)
    sim.upload("vel", u, v)
    sim.advect_diffuse_rhs(dt)
    au, av = sim.download("tmpV")
    ru, rv = orc.advect_diffuse(u, v, 1.0 / N, nu, dt)
    assert rel(au, ru) < 1e-12 and rel(av, rv) < 1e-12
    # fused stage: out = old + coef*K(in)/h^2 with old != in
    sim.upload("vold", v, u)
    sim.advect_diffuse_stage("vel", "vold", "tmpV", 0.5, dt)
    su, sv = sim.download("tmpV")
    ih2 = 0.5 * N * N
    assert np.abs(su - (v + ru * ih2)).max() < 1e-12 * max(1.0, np.abs(ru * ih2).max())
    assert np.abs(sv - (u + rv * ih2)).max() < 1e-12 * max(1.0, np.abs(rv * ih2).max())
    sim.close()


@pytest.mark.parametrize("su,sv", [(1, 1), (1, -1), (-1, 1), (-1, -1)])
def test_advect_uniformly_advected_lines_vs_oracle(su, sv):
    """The advect kernel runs lines whose eight cells are all advected one way through a branch-free upwind core — from the
    left as they lie, from the right as the mirrored line (weno.cuh: weno_line_upwind) — and everything else through the
    general core.  Fields of one sign per component put EVERY line on that path, in all four direction combinations; a
    sign-changing stripe in the middle keeps some lines on the general core next to them.  All three stage modes."""
    L = 4
    N = 8 << L
    u, v, *_ = make_fields(N, 91, "random")
    u = su * (1.5 + 0.4 * u)
    v = sv * (1.5 + 0.4 * v)
    u[:, N // 2 - 5:N // 2 + 6] *= np.sign(np.sin(np.arange(11) + 0.3))[None, :]   # stagnation stripe: mixed-sign lines
    v[N // 2 - 5:N // 2 + 6, :] *= np.sign(np.cos(np.arange(11) + 0.1))[:, None]
    nu, dt = 1e-3, 0.2 / N
    sim = cup2d_b200.Simulation(L, nu=nu)
    sim.upload("vel", u, v)
    sim.advect_diffuse_rhs(dt)                                   # raw K(in)
    au, av = sim.download("tmpV")
    ru, rv = orc.advect_diffuse(u, v, 1.0 / N, nu, dt)
    assert rel(au, ru) < 1e-12 and rel(av, rv) < 1e-12
    ih2 = 0.5 * N * N
    sim.advect_diffuse_stage("vel", "vel", "tmpV", 0.5, dt)      # old == in
    au, av = sim.download("tmpV")
    assert np.abs(au - (u + ru * ih2)).max() < 1e-12 * np.abs(ru * ih2).max()
    assert np.abs(av - (v + rv * ih2)).max() < 1e-12 * np.abs(rv * ih2).max()
    sim.upload("vold", v, u)
    sim.advect_diffuse_stage("vel", "vold", "tmpV", 0.5, dt)     # old is another field
    au, av = sim.download("tmpV")
    assert np.abs(au - (v + ru * ih2)).max() < 1e-12 * np.abs(ru * ih2).max()
    assert np.abs(av - (u + rv * ih2)).max() < 1e-12 * np.abs(rv * ih2).max()
    sim.close()


def test_rk2_and_dt_vs_oracle():
    L = 5
    N = 8 << L
    u, v, *_ = make_fields(N, 11)
    sim = cup2d_b200.Simulation(L, nu=1e-3, cfl=0.5)
    sim.upload("vel", u, v)
    umax, dt = sim.compute_dt()
    assert umax == max(np.abs(u).max(), np.abs(v).max())
    assert abs(dt - orc.compute_dt(u, v, 1.0 / N, 1e-3, 0.5)) < 1e-16
    sim.rk2(dt)
    gu, gv = sim.download("vel")
    ru, rv = orc.rk2(u, v, 1.0 / N, 1e-3, dt)
    assert np.abs(gu - ru).max() < 1e-12 and np.abs(gv - rv).max() < 1e-12
    sim.close()


@pytest.mark.parametrize("L,seed", [(0, 21), (1, 22), (4, 23), (6, 24)])
def test_pressure_rhs_and_correction_vs_oracle(L, seed):
    N = 8 << L
    h = 1.0 / N
    u, v, p, chi, udu, udv = make_fields(N, seed, "random" if L < 2 else "tg")
    dt = 0.25 * h
    sim = cup2d_b200.Simulation(L)
    sim.upload("vel", u, v)
    sim.upload("tmpV", udu, udv)
    sim.upload("chi", chi)
    sim.upload("pres", p)
    sim.pressure_rhs(dt)
    ref = orc.pressure_rhs1(orc.pressure_rhs(u, v, udu, udv, chi, h, dt), p)
    assert rel(sim.download("tmp"), ref) < 1e-13
    # correction with the Poisson "solution" x := a given field (0 iterations returns x0 = pres)
    x = np.random.default_rng(seed).uniform(-1, 1, (N, N))
    sim.upload("pres", x)
    it, err = sim.poisson_solve(max_iter=0)
    assert it == 0
    sim.pressure_correct(dt)
    pnew = (x - x.mean()) + p  # pold = p after pressure_rhs
    gu, gv = orc.grad_p(pnew, h, dt)
    assert np.abs(sim.download("pres") - pnew).max() < 1e-13
    cu, cv = sim.download("vel")
    assert np.abs(cu - (u + gu / h / h)).max() < 1e-11 and np.abs(cv - (v + gv / h / h)).max() < 1e-11
    sim.close()


@pytest.mark.parametrize("L,K", [(1, 5), (3, 10), (5, 10)])
def test_poisson_iterations_vs_oracle(L, K):
    """Same b, x0 = 0, exactly K iterations: iterates agree to rounding-amplified tolerance."""
    N = 8 << L
    rng = np.random.default_rng(100 + L)
    x = (np.arange(N) + 0.5) / N
    X, Y = np.meshgrid(x, x)
    xs = np.cos(2 * np.pi * X) * np.cos(2 * np.pi * Y) + 0.1 * rng.uniform(-1, 1, (N, N))
    b = orc.laplacian_neumann(xs)  # consistent right-hand side of the singular Neumann problem
    sim = cup2d_b200.Simulation(L)
    sim.upload("tmp", b)
    sim.upload("pres", np.zeros((N, N)))
    it, err = sim.poisson_solve(max_iter=K)
    xr, itr, errr = orc.bicgstab(b, np.zeros_like(b), max_iter=K)
    assert it == itr == K
    assert abs(err - errr) < 1e-9 * max(1.0, errr)
    assert np.abs(sim.download("pres") - xr).max() < 1e-9
    sim.close()


def test_poisson_preconditioner_matches_dense_p_inv():
    """One iteration from x0=0 exposes z = M r directly: x1 = alpha z1 + omega z2; compare with the
    oracle that applies the reference's dense 64x64 P_inv (main.cpp:6451-6488)."""
    L = 2
    N = 8 << L
    b = np.random.default_rng(5).uniform(-1, 1, (N, N))
    b -= b.mean()
    sim = cup2d_b200.Simulation(L)
    sim.upload("tmp", b)
    sim.upload("pres", np.zeros((N, N)))
    sim.poisson_solve(max_iter=1)
    xr, _, _ = orc.bicgstab(b, np.zeros_like(b), max_iter=1)
    assert np.abs(sim.download("pres") - xr).max() < 1e-12
    sim.close()


def test_poisson_converges_and_stops_like_reference():
    """Tolerance-driven stop: same iteration count as the oracle's restatement of cuda.cu:535-541 and a
    residual that really is below tol (checked with an independent application of A)."""
    L = 4
    N = 8 << L
    x = (np.arange(N) + 0.5) / N
    X, Y = np.meshgrid(x, x)
    b = orc.laplacian_neumann(np.cos(2 * np.pi * X) * np.cos(np.pi * Y))
    sim = cup2d_b200.Simulation(L)
    sim.upload("tmp", b)
    sim.upload("pres", np.zeros((N, N)))
    it, err = sim.poisson_solve(tol_abs=1e-8, tol_rel=0.0, max_restarts=100, max_iter=1000)
    xr, itr, errr = orc.bicgstab(b, np.zeros_like(b), 1e-8, 0.0, 100, 1000)
    assert err <= 1e-8 and abs(it - itr) <= 1
    xg = sim.download("pres")
    assert np.abs(b - orc.laplacian_neumann(xg)).max() <= 1.0001e-8 + 1e-12
    sim.close()


def test_large_grid_properties():
    """2048^2 (65536 blocks): properties that do not need the oracle at this size.
    (a) a field mirrored about the vertical mid-line gives a mirrored update (u odd, v even);
    (b) the Poisson residual reported by the solver equals an independent residual of the returned x;
    (c) pressure_rhs is linear in vel."""
    L = 8
    N = 8 << L
    x = (np.arange(N) + 0.5) / N
    X, Y = np.meshgrid(x, x)
    u = np.sin(2 * np.pi * X) * np.cos(2 * np.pi * Y) * (1 + 0.3 * np.cos(6 * np.pi * Y))
    v = -np.cos(2 * np.pi * X) * np.sin(2 * np.pi * Y) * (1 + 0.2 * np.cos(4 * np.pi * X))
    sim = cup2d_b200.Simulation(L, nu=1e-4)
    dt = 0.25 / N
    sim.upload("vel", u, v)
    sim.rk2(dt)
    a, b = sim.download("vel")
    assert np.abs(a + a[:, ::-1]).max() < 1e-12 and np.abs(b - b[:, ::-1]).max() < 1e-12
    # (c) linearity of the divergence part (chi = 0, pold = 0)
    sim.upload("vel", u, v)
    sim.upload("pres", np.zeros((N, N)))
    sim.upload("tmpV", np.zeros((N, N)), np.zeros((N, N)))
    sim.pressure_rhs(dt)
    r1 = sim.download("tmp")
    sim.upload("vel", 2 * u, 2 * v)
    sim.upload("pres", np.zeros((N, N)))
    sim.pressure_rhs(dt)
    assert np.abs(sim.download("tmp") - 2 * r1).max() < 1e-9 * np.abs(r1).max()
    # (b) residual consistency
    sim.upload("tmp", r1)
    sim.upload("pres", np.zeros((N, N)))
    it, err = sim.poisson_solve(max_iter=30)
    xg = sim.download("pres")
    res = np.abs(r1 - orc.laplacian_neumann(xg)).max()
    assert abs(res - err) < 1e-8 * max(1.0, np.abs(r1).max())
    sim.close()


def test_reference_driver_with_adapter_matches_reference_gpu_solver(golden_dir, tmp_path):
    """The drop-in boundary: the UNMODIFIED reference time loop linked against
    dropin/local_spmat_adapter.cpp + libcup2d_b200.so (oracle/_ref/ref_harness_b200) against the same loop
    with the reference's own cuda.cu (tests/golden/driver_gpu_steps_L3.npz, recorded from oracle/_ref/ref_harness_gpu by
    tests/golden/make_driver_golden.py): 1 step, 1000 iterations."""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "oracle", "_ref", "ref_harness_b200")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/ref_harness_b200 not built (make -C oracle all: needs the reference sources)")
    g = np.load(os.path.join(golden_dir, "driver_gpu_steps_L3.npz"))
    L = int(g["L"])
    N = 8 << L
    u, v, p, *_ = make_fields(N, int(g["seed"]))
    z = np.zeros((N, N))
    fin, fout = tmp_path / "in.bin", tmp_path / "out.bin"
    np.concatenate([a.ravel() for a in (u, v, p, z, z, z)]).tofile(fin)
    subprocess.run([exe, "steps", str(L), "1e-3", "0.5", "1", str(int(g["kiter"])), str(fin), str(fout)], check=True,
                   stderr=subprocess.DEVNULL, env=dict(os.environ, OMP_NUM_THREADS="8"), timeout=420)
    out = np.fromfile(fout).reshape(1, 1 + 5 * N * N)
    assert np.abs(out[:, 0] - g["dt"]).max() < 1e-14          # dt
    f = out[:, 1:].reshape(1, 5, N, N)
    # contract: L-inf(u,v,p) < 1e-6; observed ~1e-12 (u,v) / 1e-10 (p) after 1000 Krylov iterations
    assert max(np.abs(f[:, 0] - g["u"]).max(), np.abs(f[:, 1] - g["v"]).max(), np.abs(f[:, 2] - g["p"]).max()) < 1e-8


@pytest.mark.parametrize("name", ["steps_L2_random_k8", "steps_L3_tg_k15"])
def test_reference_driver_patched_loop_matches_golden(golden_dir, name, tmp_path):
    """The drop-in boundary for the operators: the reference's OWN time loop (unmodified main.cpp with lines 6607-6642 and
    7007-7187 replaced at build time by dropin/patched_loop_*.inc, oracle/_ref/ref_harness_patched) running its hot path on
    libcup2d_b200.so, against the steps the unmodified reference produced."""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "oracle", "_ref", "ref_harness_patched")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/ref_harness_patched not built (make -C oracle all in the build container)")
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    L, K, ns = int(g["L"]), int(g["kiter"]), len(g["dt"])
    N = 8 << L
    z = np.zeros((N, N))
    fin, fout = tmp_path / "in.bin", tmp_path / "out.bin"
    np.concatenate([a.ravel() for a in (g["u0"], g["v0"], g["p0"], z, z, z)]).tofile(fin)
    try:
        subprocess.run([exe, "steps", str(L), repr(float(g["nu"])), repr(float(g["cfl"])), str(ns), str(K), str(fin), str(fout)],
                       check=True, stderr=subprocess.DEVNULL, timeout=300,
                       env=dict(os.environ, OMP_NUM_THREADS="8", CUP2D_B200_MAX_ITER=str(K)))
    except subprocess.TimeoutExpired:
        pytest.skip("the patched reference driver did not finish in 300 s on this box")
    raw = np.fromfile(fout).reshape(ns, 1 + 5 * N * N)
    f = raw[:, 1:].reshape(ns, 5, N, N)
    assert np.abs(raw[:, 0] - g["dt"]).max() < 1e-15
    assert np.abs(f[:, 0] - g["u"]).max() < 1e-12 and np.abs(f[:, 1] - g["v"]).max() < 1e-12
    assert np.abs(f[:, 2] - g["p"]).max() < 1e-10


def test_reference_driver_resident_loop_with_bodies(golden_dir, tmp_path):
    """The device-resident drop-in with bodies (oracle/_ref/ref_harness_resident: dropin/resident_*.inc spliced over
    main.cpp:6607-6642, 6648-6679, 6945-6979, 6981-7187) against the unmodified reference loop with its CPU solver
    (tests/golden/driver_fsteps_L4_k8.npz, recorded from oracle/_ref/ref_harness): two interacting fish, 4 steps, 8 Poisson
    iterations each; u, v, p at the golden's sample of cells, dt and the body states in full."""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "oracle", "_ref", "ref_harness_resident")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/ref_harness_resident not built (make -C oracle all: needs the reference sources)")
    g = np.load(os.path.join(golden_dir, "driver_fsteps_L4_k8.npz"))
    L, K, ns = int(g["L"]), int(g["kiter"]), len(g["dt"])
    env = dict(os.environ, OMP_NUM_THREADS="8", CUP2D_B200_MAX_ITER=str(K),
               CUP2D_REF_SHAPES="angle=0 L=0.8 xpos=0.52 ypos=0.44\n angle=175 L=0.8 xpos=0.47 ypos=0.56")
    out = tmp_path / "resident.bin"
    subprocess.run([exe, "fsteps", str(L), str(ns), str(K), str(out)], check=True, stderr=subprocess.DEVNULL,
                   stdout=subprocess.DEVNULL, env=env, timeout=300)
    N = 8 << L
    b = np.fromfile(out).reshape(-1, 1 + 3 * N * N + 10)
    assert len(b) == ns == 4
    assert np.abs(b[:, 0] - g["dt"]).max() < 1e-14
    assert np.abs(b[:, 1:-10][:, g["fields_idx"]] - g["fields"]).max() < 1e-9    # OpenMP summation order on the reference side
    assert np.abs(b[:, -10:] - g["bodies"]).max() < 1e-9


def test_rectangular_domain_vs_reference_golden(golden_dir):
    """2x1 base blocks, level 2 (64x32 cells): operators and two full steps against the reference."""
    d = np.load(os.path.join(golden_dir, "rect_2x1_L2.npz"))
    nu, dt, K = float(d["nu"]), float(d["dt"]), int(d["kiter"])
    sim = cup2d_b200.Simulation(int(d["L"]), bpdx=2, bpdy=1, nu=nu, cfl=float(d["cfl"]))
    assert abs(sim.h - 1.0 / d["u"].shape[1]) < 1e-18
    sim.upload("vel", d["u"], d["v"])
    sim.advect_diffuse_rhs(dt)
    au, av = sim.download("tmpV")
    assert rel(au, d["adv_u"]) < 1e-12 and rel(av, d["adv_v"]) < 1e-12
    sim.upload("tmpV", d["udef_u"], d["udef_v"])
    sim.upload("chi", d["chi"])
    sim.upload("pres", d["p"])
    sim.pressure_rhs(dt)
    assert rel(sim.download("tmp"), d["rhs1"]) < 1e-13
    sim.upload("vel", d["u"], d["v"])
    sim.upload("pres", d["p"])
    for s in range(len(d["step_dt"])):
        dts, it, err = sim.step(max_iter=K)
        assert abs(dts - d["step_dt"][s]) < 1e-15 and it == K
        u, v = sim.download("vel")
        assert np.abs(u - d["step_u"][s]).max() < 1e-9 and np.abs(v - d["step_v"][s]).max() < 1e-9
        assert np.abs(sim.download("pres") - d["step_p"][s]).max() < 1e-9
    sim.close()


def test_reference_amr_case_through_adapter(golden_dir, tmp_path):
    """SURVEY §8(f) rank 1: the reference's own run.sh case (2 fish, block-AMR) with its pressure solves on
    cup2d_b200 through the LocalSpMatDnVec adapter (coarse-fine rows via the CSR side table) against the same
    driver with the reference's cuda.cu (tests/golden/driver_gpu_amr_lmax8.npz, recorded from oracle/_ref/ref_harness_gpu).
    Same grid every step; solutions within the 1e-6 contract."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "oracle", "_ref", "ref_harness_b200")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/ref_harness_b200 not built (make -C oracle all: needs the reference sources)")
    sys.path.insert(0, os.path.join(root, "tools"))
    from ref_gpu_compare_amr import read_records
    g = np.load(os.path.join(golden_dir, "driver_gpu_amr_lmax8.npz"))
    ns = int(g["nsteps"])
    out = tmp_path / "amr.bin"
    subprocess.run([exe, "amr", str(int(g["level_max"])), str(ns), str(int(g["kiter"])), str(out)], check=True,
                   stderr=subprocess.DEVNULL, env=dict(os.environ, OMP_NUM_THREADS="8"), timeout=420)
    recs = read_records(out)
    assert len(recs) == ns == 2
    for s, r in enumerate(recs):
        lij = g[f"lij_{s}"]
        assert r["lij"].shape == lij.shape and (r["lij"] == lij).all() and len(set(lij[:, 0].tolist())) >= 2  # really multi-level
        assert abs(r["dt"] - g[f"dt_{s}"]) < 1e-7
        assert np.abs(r["b"] - g[f"b_{s}"]).max() < 1e-6 * max(1.0, np.abs(g[f"b_{s}"]).max())
        # mean-free solution (the constant mode of the singular system is free; the driver removes the volume-weighted mean,
        # main.cpp:7126-7148).  With tolerance 0 both solvers run 1000 iterations on a residual that reaches round-off level
        # after a few hundred and return the best iterate of a noisy plateau, picked by different rounding: up to ~1e-6, the
        # size of the difference between cuda.cu and its own CPU restatement (tools/ref_gpu_compare.py)
        w = np.repeat(4.0 ** (-lij[:, 0].astype(np.float64)), 64)
        xa = g[f"x_{s}"] - (w * g[f"x_{s}"]).sum() / w.sum()
        xb = r["x"] - (w * r["x"]).sum() / w.sum()
        assert np.abs(xa - xb).max() < 1e-5 * max(1.0, np.abs(xa).max())


def test_two_ranks_on_two_gpus_match_the_oracle():
    """N>1 path on real GPUs (skipped on a single-GPU box): NVLink peer halo + all-reduce, 2 ranks, vs oracle."""
    import subprocess
    import sys
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29577",
                        os.path.join(root, "tools", "multi_gpu_check.py")], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:]
    for check in ("parity_256", "tags_dump", "adapt_tags_chi", "penalisation"):
        assert f'"check": "{check}"' in r.stdout


def test_general_rows_override_reproduces_stencil_solve():
    """cup2d_poisson_create_general: cut a few block faces out of the neighbour table and hand the affected
    rows over as complete CSR rows instead (what the adapter does with coarse-fine rows).  The matrix is the
    same, so K iterations must give the same iterate as the pure stencil path."""
    import ctypes as C
    from cup2d_b200 import lib as Lb
    lib = cup2d_b200.load_library()
    Lv = 3
    nb1 = 1 << Lv
    order = cup2d_b200.block_order(1, 1, Lv)
    nblk = len(order)
    gid = -np.ones((nb1, nb1), dtype=np.int64)
    gid[order[:, 1], order[:, 0]] = np.arange(nblk)
    nbr = np.empty((nblk, 4), dtype=np.int32)
    for k, (i, j) in enumerate(order):
        nbr[k] = [gid[j, i - 1] if i > 0 else -1, gid[j, i + 1] if i < nb1 - 1 else -1,
                  gid[j - 1, i] if j > 0 else -1, gid[j + 1, i] if j < nb1 - 1 else -1]
    full = nbr.copy()
    rng = np.random.default_rng(3)
    rows = {}

    def stencil_row(k, lr):  # complete row of the 5-point Neumann matrix from the FULL table
        x, y = lr % 8, lr // 8
        cols = []
        for d, (dx, dy) in enumerate([(-1, 0), (1, 0), (0, -1), (0, 1)]):
            xx, yy = x + dx, y + dy
            if 0 <= xx < 8 and 0 <= yy < 8:
                cols.append(k * 64 + yy * 8 + xx)
            elif full[k, d] >= 0:
                cols.append(full[k, d] * 64 + (yy % 8) * 8 + (xx % 8))
        return [(c, 1.0) for c in cols] + [(k * 64 + lr, -float(len(cols)))]

    for k in rng.choice(nblk, 10, replace=False):
        d = int(rng.integers(0, 4))
        n = full[k, d]
        if n < 0:
            continue
        od = d ^ 1
        nbr[k, d] = -1
        nbr[n, od] = -1
        for kk, dd in ((k, d), (n, od)):
            for t in range(8):
                lr = {0: t * 8, 1: t * 8 + 7, 2: t, 3: 56 + t}[dd]
                rows[kk * 64 + lr] = None
    # any row whose block lost a face must be complete in the CSR (corner cells may touch two cut faces)
    irr = sorted(rows)
    rowptr, cols, vals = [0], [], []
    for r in irr:
        for c, v in sorted(stencil_row(r // 64, r % 64)):
            cols.append(c)
            vals.append(v)
        rowptr.append(len(cols))
    irr_a, rp_a = np.array(irr, dtype=np.int32), np.array(rowptr, dtype=np.int32)
    col_a, val_a = np.array(cols, dtype=np.int32), np.array(vals, dtype=np.float64)
    h = C.c_void_p()
    I32 = C.POINTER(C.c_int32)
    Lb.check(lib.cup2d_poisson_create_general(nblk, nbr.ctypes.data_as(I32), len(irr), irr_a.ctypes.data_as(I32),
                                              rp_a.ctypes.data_as(I32), col_a.ctypes.data_as(I32),
                                              val_a.ctypes.data_as(C.POINTER(C.c_double)), 0, C.byref(h)))
    N = 8 << Lv
    bglob = rng.uniform(-1, 1, (N, N))
    bglob -= bglob.mean()
    bb = cup2d_b200.to_blocks(bglob, order, nb1)
    x0 = np.zeros_like(bb)
    Lb.check(lib.cup2d_field_upload(h, 6, bb.ctypes.data))
    Lb.check(lib.cup2d_field_upload(h, 4, x0.ctypes.data))
    it, err = C.c_int(), C.c_double()
    Lb.check(lib.cup2d_poisson_solve(h, 0.0, 0.0, 0, 12, C.byref(it), C.byref(err)))
    xg = np.empty_like(bb)
    Lb.check(lib.cup2d_field_download(h, 4, xg.ctypes.data))
    lib.cup2d_destroy(h)
    sim = cup2d_b200.Simulation(Lv)
    sim.upload("tmp", bglob)
    sim.upload("pres", np.zeros((N, N)))
    it2, err2 = sim.poisson_solve(max_iter=12)
    xs = cup2d_b200.to_blocks(sim.download("pres"), order, nb1)
    sim.close()
    assert it.value == it2 == 12 and len(irr) > 0
    assert np.abs(xg - xs).max() < 1e-10 and abs(err.value - err2) < 1e-10


def test_full_step_1024_vs_oracle():
    """BASELINE config 2 size (1024^2, Taylor-Green, nu = 1e-3 => Re 1000): one full step, 10 BiCGSTAB
    iterations, against the numpy oracle."""
    L = 7
    N = 8 << L
    u, v, p, *_ = make_fields(N, 2024)
    sim = cup2d_b200.Simulation(L, nu=1e-3, cfl=0.5)
    sim.upload("vel", u, v)
    sim.upload("pres", p)
    dt, it, err = sim.step(max_iter=10)
    ref = orc.step(u, v, p, 1e-3, 0.5, kiter=10)
    assert abs(dt - ref["dt"]) < 1e-16 and it == 10
    gu, gv = sim.download("vel")
    assert np.abs(gu - ref["u"]).max() < 1e-9 and np.abs(gv - ref["v"]).max() < 1e-9
    assert np.abs(sim.download("pres") - ref["p"]).max() < 1e-8
    sim.close()


def test_tolerance_driven_steps_vs_oracle():
    """BASELINE config 3's solver setting (Poisson tol 1e-6; main.cpp:7028-7030, stopping rule cuda.cu:535-541) at a size the
    oracle finishes in seconds (256^2): three full steps whose solves stop on the tolerance; tools/bench_c3.py times the same
    mode at 4096^2.  A tolerance-driven solve defines the pressure only up to the tolerance: BiCGSTAB's convergence curve is
    erratic, the two implementations sum their dot products in different orders, and once their histories have drifted
    apart by rounding they may cross the threshold a few iterations apart, at two DIFFERENT points that both satisfy the
    stopping rule (measured on the 128^2 case: 102 vs 100 iterations -> velocities 8e-7, pressure 6e-5 apart; equal
    counts -> 1e-14).  So the statement checked here is: (a) every solve stops with the reported residual below the
    tolerance, and an independent application of A to the returned pressure confirms it; (b) the iteration count is the
    oracle's within 20 %; (c) the fields agree to 1e-9 when the counts agree; when they do not, the pressures — two points
    with residual <= tol — differ by at most 2 tol |A^-1| <= 2 tol (N/pi)^2 (the smallest non-zero eigenvalue of the undivided
    Neumann Laplacian is ~ (pi/N)^2), and the velocities by 1e-4 (100 tol; measured 2e-6)."""
    L = 5
    N = 8 << L
    tol = 1e-6
    u, v, p, *_ = make_fields(N, 77)
    sim = cup2d_b200.Simulation(L, nu=1e-3, cfl=0.5)
    sim.upload("vel", u, v)
    sim.upload("pres", p)
    for _ in range(3):
        dt, it, err = sim.step(tol_abs=tol, tol_rel=0.0, max_restarts=0, max_iter=1000)
        ref = orc.step(u, v, p, 1e-3, 0.5, kiter=1000, tol=tol, tol_rel=0.0, max_restarts=0)
        assert abs(dt - ref["dt"]) < 1e-15 * max(1.0, dt)
        assert 0 < it < 1000 and err <= tol and abs(it - ref["iters"]) <= max(1, 0.2 * ref["iters"]), (it, ref["iters"], err)
        gu, gv = sim.download("vel")
        gp = sim.download("pres")
        # (a) independent residual: b - A x with x = pres - pold up to a constant, which A annihilates
        assert np.abs(ref["b"] - orc.laplacian_neumann(gp - p)).max() <= tol * (1 + 1e-6) + 1e-12
        same = it == ref["iters"]
        du = max(np.abs(gu - ref["u"]).max(), np.abs(gv - ref["v"]).max())
        dp = np.abs(gp - ref["p"]).max()
        assert du < (1e-9 if same else 100 * tol) and dp < (1e-8 if same else 2 * tol * (N / np.pi) ** 2), (same, du, dp)
        u, v, p = ref["u"], ref["v"], ref["p"]
        sim.upload("vel", u, v)   # continue both from the oracle's state so that later steps compare like with like
        sim.upload("pres", p)
    sim.close()


@pytest.mark.parametrize("name", ["vort_L2_random", "vort_L3_tg"])
def test_vorticity_tagging_vs_reference_golden(golden_dir, name):
    """adapt()'s tagging field (KernelVorticity, main.cpp:3343-3366) and its per-block L-inf from device data."""
    d = np.load(os.path.join(golden_dir, name + ".npz"))
    L = int(d["L"])
    sim = cup2d_b200.Simulation(L)
    sim.upload("vel", d["u"], d["v"])
    linf = sim.vorticity_tag()
    assert rel(sim.download("tmp"), d["vort"]) < 1e-14
    ref = orc.block_linf(d["vort"])
    want = ref[sim.local_order[:, 1], sim.local_order[:, 0]]
    assert np.abs(linf - want).max() < 1e-12 * np.abs(want).max()
    sim.close()


@pytest.mark.parametrize("name", ["L3_finest", "L3_coarser"])
def test_adapt_tags_vs_reference_golden(golden_dir, name):
    """adapt()'s whole block criterion (vorticity + body proximity, main.cpp:4631-4689) from device data"""
    d = np.load(os.path.join(golden_dir, f"tags_{name}.npz"))
    L, rtol = int(d["L"]), float(d["rtol"])
    sim = cup2d_b200.Simulation(L)
    sim.upload("vel", d["u"], d["v"])
    sim.upload("chi", d["chi"])
    linf = sim.adapt_tags(rtol, int(d["offset"]))
    got = sim.download("tmp")
    flagged = d["tags"] == 2 * rtol
    assert np.array_equal(got == 2 * rtol, flagged)           # same blocks flagged, same cells overwritten
    assert rel(got, d["tags"]) < 1e-14
    want = orc.block_linf(d["tags"])[sim.local_order[:, 1], sim.local_order[:, 0]]
    assert np.abs(linf - want).max() < 1e-12 * np.abs(want).max()
    sim.close()


def test_dump_files_byte_identical_to_reference(golden_dir, tmp_path):
    """cup2d_dump writes the reference's .xyz.raw / .attr.raw / .xdmf2 byte for byte (main.cpp:3367-3467)"""
    d = np.load(os.path.join(golden_dir, "dump_L2.npz"))
    sim = cup2d_b200.Simulation(int(d["L"]))
    sim.upload("vel", d["u"], d["v"])
    pref = str(tmp_path / "vel.00000007")
    sim.dump(float(d["time"]), pref)
    assert open(pref + ".xyz.raw", "rb").read() == d["xyz"].tobytes()
    assert open(pref + ".attr.raw", "rb").read() == d["attr"].tobytes()
    assert open(pref + ".xdmf2", "rb").read() == d["xdmf"].tobytes()
    sim.close()


def test_dump_large_multi_chunk(tmp_path):
    """more blocks than one staging chunk (16384), rectangular domain: every cell lands at its offset"""
    L = 7  # 2x1 boxes of 128^2 blocks = 32768 blocks = 2 chunks, 92 MB of output
    NX, NY = 2 * (8 << L), 8 << L
    rng = np.random.default_rng(5)
    u, v = rng.uniform(-1, 1, (NY, NX)), rng.uniform(-1, 1, (NY, NX))
    sim = cup2d_b200.Simulation(L, bpdx=2, bpdy=1)
    sim.upload("vel", u, v)
    pref = str(tmp_path / "big")
    sim.dump(0.5, pref)
    attr = np.fromfile(pref + ".attr.raw", dtype=np.float32).reshape(-1, 8, 8, 3)
    xyz = np.fromfile(pref + ".xyz.raw", dtype=np.float32).reshape(-1, 8, 8, 8)
    order = sim.local_order
    assert len(order) == 32768 and len(attr) == 32768
    h = 1.0 / NX  # extent / max(bpdx, bpdy) / 8 / 2^L
    for k in (0, 16383, 16384, 20000, len(order) - 1):
        i, j = order[k]
        assert np.array_equal(attr[k, :, :, 0], u[8 * j:8 * j + 8, 8 * i:8 * i + 8].astype(np.float32))
        assert np.array_equal(attr[k, :, :, 1], v[8 * j:8 * j + 8, 8 * i:8 * i + 8].astype(np.float32))
        assert xyz[k, 0, 0, 0] == np.float32(8 * i * h) and xyz[k, 0, 0, 1] == np.float32(8 * j * h)
    assert not attr[..., 2].any()
    sim.close()


def test_penalisation_phase_vs_reference_golden(penal_golden):
    """shape integrals, penalisation blend and udef assembly on device data against the reference's own
    penalisation phase (two interacting fish; main.cpp:6643-6681, 6944-7002).  Blend and assembly: bit for bit."""
    L, steps = penal_golden
    sim = cup2d_b200.Simulation(L)
    for st in steps:
        sim.upload("vel", st["u0"], st["v0"])
        sim.upload("chi", st["chi"])
        for k, sh in enumerate(st["shapes"]):
            sim.shape_set(k, sh["ids"], sh["X"], sh["udef"])
        for k, sh in enumerate(st["shapes"]):
            Q = sim.shape_integrals(k, st["lam"], st["dt"], sh["cx"], sh["cy"])
            assert np.abs(Q - sh["Q"]).max() <= 1e-12 * np.abs(sh["Q"]).max(), (Q, sh["Q"])
        for k, sh in enumerate(st["shapes"]):
            sim.penalize(k, st["lam"], st["dt"], sh["cx"], sh["cy"], sh["u"], sh["v"], sh["omega"])
        u1, v1 = sim.download("vel")
        assert np.array_equal(u1, st["u1"]) and np.array_equal(v1, st["v1"])
        sim.udef_assemble()
        udu, udv = sim.download("tmpV")
        assert np.array_equal(udu, st["udu"]) and np.array_equal(udv, st["udv"])
    sim.close()


def test_shape_calls_reject_bad_arguments():
    sim = cup2d_b200.Simulation(2)
    with pytest.raises(cup2d_b200.lib.Cup2dError):
        sim.shape_integrals(0, 1e7, 1e-3, 0.5, 0.5)  # shape never set
    with pytest.raises(cup2d_b200.lib.Cup2dError):
        sim.shape_set(0, [16], np.zeros((1, 8, 8)), np.zeros((1, 8, 8, 2)))  # block id outside the grid
    sim.shape_set(0, [], np.zeros((0, 8, 8)), np.zeros((0, 8, 8, 2)))
    assert not sim.shape_integrals(0, 1e7, 1e-3, 0.5, 0.5).any()
    sim.close()


def test_host_pipeline_matches_blocking_calls():
    """cup2d_pipe_*: independent steps with host inputs and results, upload(n+1) || step(n) || download(n-1) on three
    streams with buffer trading — bit-identical to cup2d_field_upload + cup2d_step + cup2d_field_download, for more jobs
    than staging sets (slot reuse), with the context's own fields left alone in between."""
    import torch
    L, jobs = 2, 6
    sim = cup2d_b200.Simulation(L, nu=1e-3, cfl=0.4)
    n = sim.nloc
    rng = np.random.default_rng(5)
    pin = (lambda a: a.pin_memory()) if torch.cuda.is_available() else (lambda a: a)
    vin = [pin(torch.from_numpy(rng.uniform(-1, 1, n * 128))) for _ in range(jobs)]
    pin_ = [pin(torch.from_numpy(rng.uniform(-1, 1, n * 64))) for _ in range(jobs)]
    vout = [pin(torch.empty(n * 128, dtype=torch.float64)) for _ in range(jobs)]
    pout = [pin(torch.empty(n * 64, dtype=torch.float64)) for _ in range(jobs)]
    # blocking reference, job by job
    want = []
    for j in range(jobs):
        sim.upload_blocks("vel", vin[j].numpy())
        sim.upload_blocks("pres", pin_[j].numpy())
        info = sim.step(max_iter=2, max_restarts=0)
        want.append((sim.download_blocks("vel").copy(), sim.download_blocks("pres").copy(), info))
    # the context's own fields must survive a pipelined batch untouched
    sim.upload_blocks("vel", vin[0].numpy())
    sim.upload_blocks("pres", pin_[0].numpy())
    got = sim.pipelined_steps(((vin[j].data_ptr(), pin_[j].data_ptr(), vout[j].data_ptr(), pout[j].data_ptr()) for j in range(jobs)),
                              max_iter=2, max_restarts=0)
    for j in range(jobs):
        assert np.array_equal(vout[j].numpy(), want[j][0]) and np.array_equal(pout[j].numpy(), want[j][1]), j
        assert got[j] == want[j][2]
    assert np.array_equal(sim.download_blocks("vel"), vin[0].numpy()) and np.array_equal(sim.download_blocks("pres"), pin_[0].numpy())
    # slot misuse is refused, not silently accepted
    with pytest.raises(Exception):
        sim.pipe_upload(sim.PIPE_SLOTS, vin[0].data_ptr(), pin_[0].data_ptr())


@pytest.mark.parametrize("case", ["all_zero", "constant_pressure", "uniform_flow", "tiny_values"])
def test_degenerate_inputs_vs_oracle(case):
    """inputs on which the Krylov recurrences divide by (almost) nothing — zero right-hand side, zero residual after the
    first half-step — and the dt rule has umax = 0: the eps = 1e-21 guards of the reference (cuda.cu:315-326) and its
    1e-8 in the CFL rule (main.cpp:6594) must give the same finite results, no NaN"""
    L = 2
    N = 8 << L
    z = np.zeros((N, N))
    rng = np.random.default_rng(9)
    u, v, p = {"all_zero": (z, z, z), "constant_pressure": (z, z, z + 3.0), "uniform_flow": (z + 0.7, z, z),
               "tiny_values": (1e-150 * rng.uniform(-1, 1, (N, N)), 1e-150 * rng.uniform(-1, 1, (N, N)), z)}[case]
    sim = cup2d_b200.Simulation(L, nu=1e-3, cfl=0.5)
    sim.upload("vel", u, v)
    sim.upload("pres", p)
    dt, it, err = sim.step(max_iter=6, max_restarts=0)
    ref = orc.step(u, v, p, 1e-3, 0.5, kiter=6)
    gu, gv = sim.download("vel")
    gp = sim.download("pres")
    assert np.isfinite(gu).all() and np.isfinite(gv).all() and np.isfinite(gp).all() and np.isfinite(err)
    assert abs(dt - ref["dt"]) <= 1e-16 * ref["dt"]
    scale = max(np.abs(ref["u"]).max(), np.abs(ref["v"]).max(), 1e-300)
    assert np.abs(gu - ref["u"]).max() <= 1e-9 * scale and np.abs(gv - ref["v"]).max() <= 1e-9 * scale
    assert np.abs(gp - ref["p"]).max() <= 1e-8 * max(np.abs(ref["p"]).max(), 1e-300)
    sim.close()


def _run_steps(L, nsteps, graph, seed=11, **kw):
    """nsteps time steps through cup2d_step_enqueue (graph replay from the second step on) or, with graph=False, through
    direct launches with the dt rule on the host; returns fields and the per-step (dt, iterations, residual)"""
    N = 8 << L
    u, v, p, *_ = make_fields(N, seed)
    sim = cup2d_b200.Simulation(L, nu=1e-3, cfl=0.4)
    sim.set_graph(graph)
    sim.upload("vel", u, v)
    sim.upload("pres", p)
    info = []
    for _ in range(nsteps):
        if graph:
            sim.step_enqueue(**kw)          # dt <= 0: dt control on the device, inside the graph
            info.append(sim.step_result())
        else:
            _, dt = sim.compute_dt()        # the reference's order: umax -> host -> dt (main.cpp:6579-6595)
            info.append(sim.step(dt=dt, **kw))
    out = (sim.download("vel"), sim.download("pres"), info, sim.launch_count())
    sim.close()
    return out


@pytest.mark.parametrize("L", [2, 5])
def test_graph_replayed_steps_are_bitwise_the_directly_launched_steps(L):
    """cup2d_step_enqueue replays one captured CUDA graph per buffer assignment (dt rule on the device, correction picking
    the best iterate through the device-side Krylov state): five steps must reproduce, bit for bit, five steps launched
    kernel by kernel with dt computed on the host — same dt, same fields"""
    (gu, gv), gp, ginfo, _ = _run_steps(L, 5, True, max_iter=12, max_restarts=0)
    (du, dv), dp, dinfo, _ = _run_steps(L, 5, False, max_iter=12, max_restarts=0)
    assert [i[0] for i in ginfo] == [i[0] for i in dinfo], "dt computed on the device differs from the host rule"
    assert [i[1] for i in ginfo] == [i[1] for i in dinfo] == [12] * 5
    assert np.array_equal(gu, du) and np.array_equal(gv, dv) and np.array_equal(gp, dp)


def test_graph_while_node_stops_where_the_host_polled_solve_stops():
    """tolerance-driven solve inside the step graph: the Krylov loop is a WHILE node whose condition the device sets;
    iteration counts, residuals and fields equal those of the host-polled solve (cuda.cu:535-541 stopping rule)"""
    kw = dict(tol_abs=1e-7, tol_rel=0.0, max_restarts=100, max_iter=400)
    (gu, gv), gp, ginfo, _ = _run_steps(4, 4, True, **kw)
    (du, dv), dp, dinfo, _ = _run_steps(4, 4, False, **kw)
    assert [i[1] for i in ginfo] == [i[1] for i in dinfo]
    assert all(0 < i[1] < 400 and i[2] <= 1e-7 for i in ginfo), ginfo
    assert np.array_equal(gu, du) and np.array_equal(gv, dv) and np.array_equal(gp, dp)


def test_enqueued_steps_need_no_host_round_trip():
    """several steps enqueued back to back, one result read at the end == the same steps read one by one"""
    L, N = 4, 128
    u, v, p, *_ = make_fields(N, 3)
    outs = []
    for batch in (True, False):
        sim = cup2d_b200.Simulation(L, nu=1e-3, cfl=0.4)
        sim.upload("vel", u, v)
        sim.upload("pres", p)
        for k in range(6):
            sim.step_enqueue(max_iter=8, max_restarts=0)
            if not batch:
                sim.step_result()
        last = sim.step_result()
        outs.append((sim.download("vel"), sim.download("pres"), last))
        sim.close()
    assert outs[0][2] == outs[1][2]
    assert np.array_equal(outs[0][0][0], outs[1][0][0]) and np.array_equal(outs[0][1], outs[1][1])
