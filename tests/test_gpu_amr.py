"""GPU tests of the multi-level device path (csrc/amr_ops.cu baseline kernels, csrc/amr_fast.cu, the bodies of csrc/penalize.cu, the
tagging of cup2d_amr_adapt_tags) against the reference's own outputs on its 7-level run.sh mesh (tests/golden/amrlab_lmax8.npz,
amrtags_lmax8.npz), against the reference restatement on a second mesh family, and in situ (the reference's run.sh case
with its hot path spliced onto this path).

They also pass on the CPU against the emulated build of the same sources
(tools/run_emulated_gpu_tests.sh, tests/test_full_emulation.py)."""
import os

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]


@pytest.fixture(scope="module")
def case(golden_dir):
    from cup2d_b200.amr import AmrSimulation
    d = np.load(os.path.join(golden_dir, "amrlab_lmax8.npz"))
    sim = AmrSimulation(d["blocks"], int(d["bpdx"]), int(d["bpdy"]), float(d["h0"]), float(d["nu"]))
    yield d, sim
    sim.close()


def rel(a, b):
    return np.abs(a - b).max() / np.abs(b).max()


def test_amr_advect_diffuse_with_flux_correction(case):
    d, sim = case
    sim.upload("vel", d["vel"])
    sim.advect_diffuse_rhs(float(d["dt"]))
    assert rel(sim.download("tmpV"), d["adv"]) < 1e-12


def test_amr_fast_advect_kernel(case):
    d, sim = case
    sim.upload("vel", d["vel"])
    sim.advect_diffuse_rhs_fast(float(d["dt"]))
    assert rel(sim.download("tmpV"), d["adv"]) < 1e-12


def test_amr_fast_pressure_kernels(case):
    d, sim = case
    sim.upload("vel", d["vel"])
    sim.upload("tmpV", d["udef"])
    sim.upload("chi", d["chi"])
    sim.upload("pold", d["pres"])
    sim.pressure_rhs_fast(float(d["dt"]), with_laplacian=False)
    assert rel(sim.download("tmp"), d["rhs"]) < 1e-12
    sim.pressure_rhs_fast(float(d["dt"]), with_laplacian=True)
    assert rel(sim.download("tmp"), d["rhs1"]) < 1e-12
    sim.upload("pres", d["pres"])
    sim.pressure_gradient_fast(float(d["dt"]))
    assert rel(sim.download("tmpV"), d["gradp"]) < 1e-12


def test_amr_pressure_rhs_and_laplacian(case):
    d, sim = case
    sim.upload("vel", d["vel"])
    sim.upload("tmpV", d["udef"])
    sim.upload("chi", d["chi"])
    sim.upload("pold", d["pres"])
    sim.pressure_rhs(float(d["dt"]), with_laplacian=False)
    assert rel(sim.download("tmp"), d["rhs"]) < 1e-12
    sim.upload("tmpV", d["udef"])
    sim.pressure_rhs(float(d["dt"]), with_laplacian=True)
    assert rel(sim.download("tmp"), d["rhs1"]) < 1e-12


def test_amr_pressure_gradient(case):
    d, sim = case
    sim.upload("pres", d["pres"])
    sim.pressure_gradient(float(d["dt"]))
    assert rel(sim.download("tmpV"), d["gradp"]) < 1e-12


def test_native_amr_poisson_matrix_on_the_device_solver(golden_dir):
    """host-built multi-level Poisson rows (cup2d_amr_plan_poisson, bitwise the reference's) -> the validated general-rows
    solver (cup2d_poisson_create_general): 20 BiCGSTAB iterations against the oracle's BiCGSTAB on the reference's COO"""
    import ctypes as C
    import scipy.sparse as sp
    import cup2d_oracle as orc
    from cup2d_b200 import lib as Lb
    from cup2d_b200.amr import AmrPlan
    d = np.load(os.path.join(golden_dir, "amrlab_lmax8.npz"))
    plan = AmrPlan(d["blocks"], int(d["bpdx"]), int(d["bpdy"]))
    nbr, rows, rowptr, col, val = plan.poisson()
    nb = len(plan.blocks)
    lib = Lb.load_library()
    h = C.c_void_p()
    I32 = C.POINTER(C.c_int32)
    Lb.check(lib.cup2d_poisson_create_general(nb, nbr.ctypes.data_as(I32), len(rows), rows.ctypes.data_as(I32),
                                              rowptr.ctypes.data_as(I32), col.ctypes.data_as(I32),
                                              val.ctypes.data_as(C.POINTER(C.c_double)), 0, C.byref(h)))
    b = np.ascontiguousarray(d["rhs1"].reshape(-1))
    x0 = np.zeros_like(b)
    Lb.check(lib.cup2d_field_upload(h, 6, b.ctypes.data))
    Lb.check(lib.cup2d_field_upload(h, 4, x0.ctypes.data))
    it, err = C.c_int(), C.c_double()
    K = 20
    Lb.check(lib.cup2d_poisson_solve(h, 0.0, 0.0, 0, K, C.byref(it), C.byref(err)))
    x = np.empty_like(b)
    Lb.check(lib.cup2d_field_download(h, 4, x.ctypes.data))
    lib.cup2d_destroy(h)
    plan.close()
    n = 64 * nb
    A = sp.coo_matrix((d["coo_val"], (d["coo_row"], d["coo_col"])), shape=(n, n)).tocsr()
    P = orc.build_P_inv()
    xr, itr, errr = orc.bicgstab(b, x0, max_iter=K, A=lambda v: A @ v, M=lambda v: (v.reshape(nb, 64) @ P.T).reshape(-1))
    assert it.value == itr == K
    assert np.abs(x - xr).max() < 1e-9 * np.abs(xr).max()
    assert abs(err.value - errr) < 1e-9 * errr


@pytest.mark.parametrize("fast", [False, True])
def test_amr_full_step_against_composed_oracle(case, fast):
    """one whole time step without bodies on the 7-level mesh (dt, RK2, rhs, 15 BiCGSTAB iterations on the native Poisson
    rows, correction) against the same step composed from the pinned oracle pieces"""
    import scipy.sparse as sp
    import cup2d_amr_oracle as amr
    import cup2d_oracle as orc
    d, sim = case
    mesh = amr.Mesh(d["blocks"], int(d["bpdx"]), int(d["bpdy"]))
    h0, nu, nb = float(d["h0"]), float(d["nu"]), len(d["blocks"])
    sim.upload("vel", d["vel"])
    sim.upload("pres", d["pres"])
    sim.upload("chi", np.zeros_like(d["chi"]))
    sim.set_fast(fast)
    dt, it, err = sim.step(cfl=0.5, max_iter=15)
    sim.set_fast(False)
    want_dt = amr.amr_compute_dt(mesh, h0, d["vel"], nu, 0.5)
    assert abs(dt - want_dt) < 1e-15 * want_dt and it == 15
    v = amr.amr_rk2(mesh, h0, d["vel"], nu, want_dt)
    zero2, zero1 = np.zeros_like(d["vel"]), np.zeros_like(d["chi"])
    b, pold, p0 = amr.amr_poisson_rhs(mesh, h0, v, zero2, zero1, d["pres"], want_dt)
    n = 64 * nb
    A = sp.coo_matrix((d["coo_val"], (d["coo_row"], d["coo_col"])), shape=(n, n)).tocsr()
    P = orc.build_P_inv()
    x, _, _ = orc.bicgstab(b.reshape(-1), p0.reshape(-1), max_iter=15, A=lambda q: A @ q,
                           M=lambda q: (q.reshape(nb, 64) @ P.T).reshape(-1))
    vel, pres = amr.amr_pressure_correct(mesh, h0, v, x.reshape(nb, 8, 8, 1), pold, want_dt)
    assert rel(sim.download("vel"), vel) < 1e-9 and rel(sim.download("pres"), pres) < 1e-9


@pytest.mark.parametrize("base", [pytest.param(3, id="base3"), pytest.param(4, id="base4")])
def test_synthetic_three_level_mesh_vs_oracle(base):
    """a second family of meshes (tools/bench_amr.py:three_level_mesh — the generator of the C5 bench mesh — here small): two
    nested refined discs, so every orientation of a level interface and its corners occur, walls included; operators on
    baseline and fast kernels against the reference restatement (oracle/cup2d_amr_oracle.py, bit-exact on the reference's own
    meshes)"""
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(root, "tools"))
    import bench_amr
    import cup2d_amr_oracle as ao
    from cup2d_b200.amr import AmrSimulation
    blocks = bench_amr.three_level_mesh(base, r1=0.3, r2=0.15, centre=(0.45, 0.55))
    assert sorted(set(blocks[:, 0].tolist())) == [base, base + 1, base + 2]
    h0, nu, dt = 1 / 8, 1e-3, 1e-3
    rng = np.random.default_rng(3)
    vel, pres = bench_amr.seeded_fields(blocks, h0)
    vel, pres = vel + 0.05 * rng.uniform(-1, 1, vel.shape), pres + 0.05 * rng.uniform(-1, 1, pres.shape)
    chi, udef = rng.uniform(0, 1, pres.shape), rng.uniform(-1, 1, vel.shape)
    out = ao.amr_operators(ao.Mesh(blocks, 1, 1), h0, vel, pres, chi, udef, nu, dt)
    sim = AmrSimulation(blocks, 1, 1, h0, nu)
    for fast in (False, True):
        sim.set_fast(fast)
        sim.upload("vel", vel)
        sim.advect_diffuse_rhs(dt)
        assert rel(sim.download("tmpV"), out["adv"]) < 1e-12
        sim.upload("tmpV", udef)
        sim.upload("chi", chi)
        sim.upload("pold", pres)
        sim.pressure_rhs(dt, True)
        assert rel(sim.download("tmp"), out["rhs1"]) < 1e-12
        sim.upload("pres", pres)
        sim.pressure_gradient(dt)
        assert rel(sim.download("tmpV"), out["gradp"]) < 1e-12
    sim.close()


def test_amr_adapt_tags_vs_reference_golden(golden_dir):
    """cup2d_amr_adapt_tags on the reference's run.sh mesh with its two fish (tests/golden/amrtags_lmax8.npz): the tagging
    field to rounding, the chi rule on exactly the reference's 80 blocks, the same refine / compress sets"""
    from cup2d_b200.amr import AmrSimulation
    d = np.load(os.path.join(golden_dir, "amrtags_lmax8.npz"))
    nb, rtol, ctol = len(d["blocks"]), float(d["rtol"]), float(d["ctol"])
    sim = AmrSimulation(d["blocks"], int(d["bpdx"]), int(d["bpdy"]), float(d["h0"]), 4e-5)
    sim.upload("vel", d["vel"])
    sim.upload("chi", d["chi"])
    for _ in range(2):   # the second call reuses the tables built by the first
        linf = sim.adapt_tags(rtol, int(d["level_max"]))
    field = sim.download("tmp").reshape(nb, 8, 8)
    want = d["tagfield"]
    assert np.abs(field - want).max() < 1e-12 * np.abs(want).max()
    fired = (d["vort"] != want).reshape(nb, -1).any(axis=1)
    assert np.array_equal(field.reshape(nb, 64)[fired][:, [27, 28, 35, 36]], np.full((fired.sum(), 4), 2 * rtol))
    wl = np.abs(want).reshape(nb, -1).max(axis=1)
    assert np.abs(linf - wl).max() < 1e-12 * wl.max()
    assert np.array_equal(linf > rtol, wl > rtol) and np.array_equal(linf < ctol, wl < ctol)
    sim.close()


@pytest.mark.parametrize("fast", [False, True])
def test_multi_level_path_on_a_uniform_mesh_equals_the_uniform_path(fast):
    """the two device paths against each other: a one-level mesh through cup2d_amr (tables, per-block cell size, general-rows
    Poisson context) and through cup2d_sim (the path measured and validated on hardware), two full steps — same dt, same
    iteration count, fields to rounding"""
    import cup2d_b200
    from cup2d_b200.amr import AmrSimulation
    L = 3
    N = 8 << L
    order = cup2d_b200.block_order(1, 1, L)
    nb = len(order)
    blocks = np.concatenate([np.full((nb, 1), L), order], axis=1).astype(np.int32)
    rng = np.random.default_rng(2)
    x = (np.arange(N) + 0.5) / N
    X, Y = np.meshgrid(x, x)
    u = np.sin(2 * np.pi * X) * np.cos(2 * np.pi * Y) + 0.05 * rng.uniform(-1, 1, (N, N))
    v = -np.cos(2 * np.pi * X) * np.sin(2 * np.pi * Y) + 0.05 * rng.uniform(-1, 1, (N, N))
    p = np.cos(2 * np.pi * X) * np.cos(2 * np.pi * Y)
    sim = cup2d_b200.Simulation(L, nu=1e-3, cfl=0.5)
    sim.upload("vel", u, v)
    sim.upload("pres", p)
    a = AmrSimulation(blocks, 1, 1, 1 / 8, 1e-3)
    a.set_fast(fast)
    a.upload("vel", sim.download_blocks("vel").reshape(nb, 8, 8, 2))
    a.upload("pres", sim.download_blocks("pres").reshape(nb, 8, 8, 1))
    for _ in range(2):
        dt1, it1, err1 = sim.step(max_iter=8, max_restarts=0)
        dt2, it2, err2 = a.step(cfl=0.5, max_iter=8)
        assert abs(dt1 - dt2) <= 1e-15 * dt1 and it1 == it2 == 8 and abs(err1 - err2) <= 1e-10 * err1
        assert np.abs(sim.download_blocks("vel").reshape(nb, 8, 8, 2) - a.download("vel")).max() < 1e-12
        assert np.abs(sim.download_blocks("pres").reshape(nb, 8, 8, 1) - a.download("pres")).max() < 1e-11
    a.close()
    sim.close()


def test_amr_dump_files_byte_identical_to_reference(golden_dir, tmp_path):
    """cup2d_amr_dump on the reference's run.sh mesh (7 levels) with its own velocity field: the three files dump() wrote
    there (tests/golden/amrdump_lmax8.npz), byte for byte"""
    from cup2d_b200.amr import AmrSimulation
    d = np.load(os.path.join(golden_dir, "amrdump_lmax8.npz"))
    sim = AmrSimulation(d["blocks"], int(d["bpdx"]), int(d["bpdy"]), float(d["h0"]), 4e-5)
    sim.upload("vel", d["vel"])
    pref = str(tmp_path / "vel.00000003")
    sim.dump(float(d["time"]), pref)
    sim.close()
    assert np.array_equal(np.fromfile(pref + ".xyz.raw", dtype=np.float32), d["xyz"])
    assert np.array_equal(np.fromfile(pref + ".attr.raw", dtype=np.float32), d["attr"])
    assert open(pref + ".xdmf2", "rb").read() == d["xdmf"].tobytes()


def test_amr_bodies_sums_blend_and_udef_assembly(case):
    """cup2d_amr_shape_*: two synthetic shapes whose obstacle blocks span several refinement levels (the field chi is the
    golden's own).  Against a block-wise numpy restatement of main.cpp:6648-6679, 6944-6979, 6980-7002 with the per-block
    cell size and origin (main.cpp:695-696): sums to rounding, blend and assembly bit for bit."""
    d, sim = case
    blocks = np.asarray(d["blocks"])
    nb, h0 = len(blocks), float(d["h0"])
    rng = np.random.default_rng(11)
    h = h0 / (1 << blocks[:, 0]).astype(np.float64)
    levels = sorted(set(blocks[:, 0].tolist()))
    vel = np.asarray(d["vel"]).reshape(nb, 8, 8, 2)
    chi = np.asarray(d["chi"]).reshape(nb, 8, 8)
    lam, dt = 1e7, float(d["dt"])
    shapes = []
    for k in range(2):  # obstacle blocks: some of every level, in increasing block order like obstacleBlocks
        ids = np.sort(np.concatenate([rng.choice(np.flatnonzero(blocks[:, 0] == lv), size=min(3, (blocks[:, 0] == lv).sum()), replace=False)
                                      for lv in levels])).astype(np.int32)
        X = rng.uniform(-0.3, 1.0, (len(ids), 8, 8))
        X[rng.uniform(size=X.shape) < 0.2] = 0.5     # the >= 0.5 / > 0.5 boundary of the two rules
        X[0] = chi[ids[0]]                            # ties with the chi field
        shapes.append(dict(ids=ids, X=X, udef=rng.uniform(-1, 1, (len(ids), 8, 8, 2)), cx=0.9 + 0.3 * k, cy=0.5,
                           u=0.1 * (k + 1), v=-0.2, omega=0.7 - k))
    sim.upload("vel", vel)
    sim.upload("chi", chi)
    ix = np.arange(8, dtype=np.float64)

    def centres(ids, cx, cy):
        hb = h[ids][:, None, None]
        px = (blocks[ids, 1] * 8).astype(np.float64)[:, None, None] * hb + hb * (ix[None, None, :] + 0.5) - cx
        py = (blocks[ids, 2] * 8).astype(np.float64)[:, None, None] * hb + hb * (ix[None, :, None] + 0.5) - cy
        return px + 0 * py, py + 0 * px
    want_v = vel.copy()
    for k, sh in enumerate(shapes):
        sim.shape_set(k, sh["ids"], sh["X"], sh["udef"])
        ids, X, ud = sh["ids"], sh["X"], sh["udef"]
        px, py = centres(ids, sh["cx"], sh["cy"])
        Xl = np.where(X >= 0.5, lam * dt, 0.0)
        F = np.where(X > 0, (h[ids] * h[ids])[:, None, None] * Xl / (1 + Xl), 0.0)
        du, dv = want_v[ids][..., 0] - ud[..., 0], want_v[ids][..., 1] - ud[..., 1]
        want = np.array([t.sum() for t in (F, F * (px * px + py * py), F * px, F * py, F * du, F * dv, F * (px * dv - py * du))])
        got = sim.shape_integrals(k, lam, dt, sh["cx"], sh["cy"])
        assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max(), (k, got, want)
    for k, sh in enumerate(shapes):  # the blend, shape after shape on the same field (a later shape sees the earlier one's result)
        sim.penalize(k, lam, dt, sh["cx"], sh["cy"], sh["u"], sh["v"], sh["omega"])
        ids, X, ud = sh["ids"], sh["X"], sh["udef"]
        px, py = centres(ids, sh["cx"], sh["cy"])
        alpha = np.where(X > 0.5, 1 / (1 + lam * dt), 1.0)
        US, VS = sh["u"] - sh["omega"] * py + ud[..., 0], sh["v"] + sh["omega"] * px + ud[..., 1]
        on = ~(chi[ids] > X) & ~(X <= 0)
        V = want_v[ids]
        V[..., 0] = np.where(on, alpha * V[..., 0] + (1 - alpha) * US, V[..., 0])
        V[..., 1] = np.where(on, alpha * V[..., 1] + (1 - alpha) * VS, V[..., 1])
        want_v[ids] = V
    assert np.array_equal(sim.download("vel").reshape(nb, 8, 8, 2), want_v)
    sim.udef_assemble()
    want_t = np.zeros((nb, 8, 8, 2))
    for sh in shapes:
        on = ~(sh["X"] < chi[sh["ids"]])
        np.add.at(want_t, sh["ids"], np.where(on[..., None], sh["udef"], 0.0))
    assert np.array_equal(sim.download("tmpV").reshape(nb, 8, 8, 2), want_t)
    with pytest.raises(Exception):
        sim.shape_set(0, [nb], np.zeros((1, 8, 8)), np.zeros((1, 8, 8, 2)))   # block id outside the mesh
    with pytest.raises(Exception):
        sim.shape_integrals(5, lam, dt, 0.0, 0.0)                                # shape never set


@pytest.mark.parametrize("form", ["amrloop", "amrresident"])
def test_reference_amr_case_on_the_multi_level_device_path(golden_dir, tmp_path, form):
    """config C1 on the device: the reference's own run.sh case with RK2 and the pressure section on cup2d_amr (fast kernels)
    — oracle/_ref/ref_harness_amrloop; with the penalisation sums, blend and u_def assembly there too: ..._amrresident —
    against the unmodified reference loop (tests/golden/driver_asteps_lmax8_k8.npz, recorded from oracle/_ref/ref_harness),
    6 steps: dt and mesh in full, velocity and pressure at the golden's sample of entries"""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "oracle", "_ref", f"ref_harness_{form}")
    if not os.path.exists(exe):
        pytest.skip(f"oracle/_ref/ref_harness_{form} not built (make -C oracle all: needs the reference sources)")
    sys.path.insert(0, golden_dir)
    from make_driver_golden import parse_asteps
    g = np.load(os.path.join(golden_dir, "driver_asteps_lmax8_k8.npz"))
    ns, K = int(g["nsteps"]), int(g["kiter"])
    env = dict(os.environ, OMP_NUM_THREADS="1", CUP2D_B200_MAX_ITER=str(K), CUP2D_B200_AMR_FAST="1")
    out = tmp_path / "asteps.bin"
    subprocess.run([exe, "asteps", str(int(g["level_max"])), str(ns), str(K), str(out)], check=True, stderr=subprocess.DEVNULL,
                   stdout=subprocess.DEVNULL, env=env, timeout=600)
    steps = parse_asteps(out)
    assert len(steps) == ns == 6
    for s, (dt, mesh, vel, pres) in enumerate(steps):
        assert np.array_equal(mesh, g[f"mesh_{s}"]) and abs(dt - g[f"dt_{s}"]) < 1e-14
        assert np.abs(vel[g[f"vel_idx_{s}"]] - g[f"vel_{s}"]).max() < 1e-10 * g[f"vel_absmax_{s}"]
        assert np.abs(pres[g[f"pres_idx_{s}"]] - g[f"pres_{s}"]).max() < 1e-9 * g[f"pres_absmax_{s}"]


def test_two_ranks_on_two_gpus_multi_level():
    """N>1 on real GPUs (skipped on a single-GPU box): the distributed general-rows Poisson solve and multi-level steps with
    replicated operators and with the mesh distributed (cup2d_poisson_create_general_ranks, cup2d_amr_set_ranks,
    cup2d_amr_create_ranks) against the same work on one GPU"""
    import subprocess
    import sys
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29578", os.path.join(root, "tools", "multi_gpu_check.py")],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=400,
                       env=dict(os.environ))
    assert r.returncode == 0, r.stdout[-2000:]
    for check in ("amr_poisson_ranks", "amr_step_ranks", "amr_distributed_ranks"):
        assert f'"check": "{check}"' in r.stdout
