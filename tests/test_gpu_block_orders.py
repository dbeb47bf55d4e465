"""GPU tests (-m gpu) of the uniform-grid context on domains of any bpdx x bpdy and with any block order.

cup2d_create takes whatever block order the caller passes and derives the neighbour table and the 4x4-block tiles of the
advect stage and of the three-kernel Krylov iteration from it.  The other GPU tests only use the Hilbert order on
domains that are whole multiples of the 4x4 tile (or smaller than one tile).  Here the domains (tests/block_orders.py)
have tiles that stop partway in x or in y next to other tiles, tiles off every wall of a domain with NX != NY, local
block counts that are not a multiple of 4 (a partial last chunk of the row kernels), and orders in which both, one or
neither of a block's W and E neighbours lie in the same chunk of four blocks.

What is checked, and why to that precision:
  * cell-local operators (advect stage in its three modes, pressure rhs, vorticity / adapt tags and their per-block L-inf,
    compute_dt): bitwise the Hilbert run mapped back block by block (the per-cell arithmetic does not depend on the
    order), and the oracle within the tolerances of tests/test_gpu_parity.py;
  * BiCGSTAB with 1, 2, 3, 7 and 12 iterations (odd counts: the (p, nu) buffer pair flips with the iteration's parity):
    the oracle's count and iterate to 1e-9 as in tests/test_gpu_parity.py; the Hilbert run and the five-kernel iteration
    of a Poisson-only context on the same neighbour table to 1e-12 relative.  Only the partition of the dot products
    differs between these three runs.  Measured on an H100 80GB HBM3 (700 W power limit) over all shapes, orders and
    counts: iterates 7.2e-14 relative apart (Hilbert) and 5.9e-14 (five kernels), residuals 6.7e-15 of |b| apart, and
    1.4e-13 from the oracle;
  * full steps, graph replay and the graph WHILE node on odd domains; reference goldens reloaded in other orders; the
    dump's per-block records; one step on 1024 tiles in a random order."""
import functools
import os

import ctypes as C
import numpy as np
import pytest

import cup2d_b200
import cup2d_oracle as orc
from cup2d_b200 import lib as Lb

from block_orders import ORDERS, SHAPES, make_order

pytestmark = pytest.mark.gpu

NU, CFL = 1e-3, 0.5


def rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def make_sim(shape, kind, **kw):
    bpdx, bpdy, level = shape
    return cup2d_b200.Simulation(level, bpdx=bpdx, bpdy=bpdy, order=make_order(bpdx, bpdy, level, kind), **kw)


def make_fields(NX, NY, seed):
    rng = np.random.default_rng(seed)
    X, Y = np.meshgrid((np.arange(NX) + 0.5) / NX, (np.arange(NY) + 0.5) / NY)
    u = np.sin(2 * np.pi * X) * np.cos(2 * np.pi * Y) + 0.05 * rng.uniform(-1, 1, (NY, NX))
    v = -np.cos(2 * np.pi * X) * np.sin(2 * np.pi * Y) + 0.05 * rng.uniform(-1, 1, (NY, NX))
    p = np.cos(2 * np.pi * X) * np.cos(2 * np.pi * Y) + 0.05 * rng.uniform(-1, 1, (NY, NX))
    chi = np.exp(-((X - 0.4) ** 2 + (Y - 0.55) ** 2) / 0.02)
    udu, udv = 0.3 * np.sin(3 * X + Y), 0.2 * np.cos(2 * Y - X)
    return u, v, p, chi, udu, udv


def corner_chi(NX, NY, seed):
    """chi > 0 only on isolated cells within 0..3 cells of block corners, diagonally off the blocks they must tag (the
    corner part of the grown-box mask), plus negative values elsewhere that clamp to 0 and must tag nothing"""
    rng = np.random.default_rng(seed)
    chi = np.zeros((NY, NX))
    for cy in range(0, NY + 1, 8):
        for cx in range(0, NX + 1, 8):
            if rng.uniform() < 0.5:
                continue
            d = int(rng.integers(0, 4))
            sx, sy = (-1 - d, -1 - d) if rng.uniform() < 0.5 else (d, d)
            if rng.uniform() < 0.5:
                sx = -1 - sx
            x, y = cx + sx, cy + sy
            if 0 <= x < NX and 0 <= y < NY:
                chi[y, x] = rng.choice([0.3, 1.0, 1.5])
    neg = rng.uniform(size=(NY, NX)) < 0.05
    chi[neg & (chi == 0)] = -0.5
    return chi


def per_block(sim, vals):
    """per-local-block values -> array [nby, nbx] by the blocks' (i, j)"""
    g = np.full((sim.nby, sim.nbx), np.nan)
    g[sim.local_order[:, 1], sim.local_order[:, 0]] = vals
    return g


def case_ids(shapes=SHAPES, orders=ORDERS):
    return [pytest.param(s, o, id=f"{s[0]}x{s[1]}L{s[2]}-{o}") for s in shapes for o in orders]


# ---- cell-local operators ------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _operators(shape, kind):
    sim = make_sim(shape, kind, nu=NU, cfl=CFL)
    NX, NY = sim.NX, sim.NY
    u, v, p, chi, udu, udv = make_fields(NX, NY, 7)
    dt = 0.3 * sim.h
    out = {}
    sim.upload("vel", u, v)
    out["umax_dt"] = sim.compute_dt()
    sim.advect_diffuse_rhs(dt)                                  # raw K(in)
    out["raw"] = sim.download("tmpV")
    sim.advect_diffuse_stage("vel", "vel", "tmpV", 0.5, dt)     # old == in
    out["same"] = sim.download("tmpV")
    sim.upload("vold", v, u)
    sim.advect_diffuse_stage("vel", "vold", "tmpV", 0.5, dt)    # old is another field
    out["other"] = sim.download("tmpV")
    sim.upload("tmpV", udu, udv)
    sim.upload("chi", chi)
    sim.upload("pres", p)
    sim.pressure_rhs(dt)
    out["rhs"], out["pold"], out["pres"] = sim.download("tmp"), sim.download("pold"), sim.download("pres")
    out["vort_linf"] = per_block(sim, sim.vorticity_tag())
    out["vort"] = sim.download("tmp")
    cchi = corner_chi(NX, NY, 11)
    sim.upload("chi", cchi)
    for off in (2, 4):
        out[f"tags{off}_linf"] = per_block(sim, sim.adapt_tags(0.1, off))
        out[f"tags{off}"] = sim.download("tmp")
    sim.close()
    return dict(out=out, fields=(u, v, p, chi, udu, udv, cchi), h=sim.h, dt=dt)


@pytest.mark.parametrize("shape,kind", case_ids())
def test_cell_local_operators_any_order(shape, kind):
    got, ref = _operators(shape, kind), _operators(shape, "hilbert")
    for key, a in got["out"].items():      # bitwise the Hilbert run, block by block
        b = ref["out"][key]
        for x, y in zip(a if isinstance(a, tuple) else (a,), b if isinstance(b, tuple) else (b,)):
            assert np.array_equal(x, y), key
    u, v, p, chi, udu, udv, cchi = got["fields"]
    h, dt, o = got["h"], got["dt"], got["out"]
    assert o["umax_dt"][0] == max(np.abs(u).max(), np.abs(v).max())
    assert abs(o["umax_dt"][1] - orc.compute_dt(u, v, h, NU, CFL)) < 1e-16
    ru, rv = orc.advect_diffuse(u, v, h, NU, dt)
    assert rel(o["raw"][0], ru) < 1e-12 and rel(o["raw"][1], rv) < 1e-12
    ih2 = 0.5 / (h * h)
    for key, (bu, bv) in (("same", (u, v)), ("other", (v, u))):
        assert np.abs(o[key][0] - (bu + ru * ih2)).max() < 1e-12 * np.abs(ru * ih2).max(), key
        assert np.abs(o[key][1] - (bv + rv * ih2)).max() < 1e-12 * np.abs(rv * ih2).max(), key
    ref_rhs = orc.pressure_rhs1(orc.pressure_rhs(u, v, udu, udv, chi, h, dt), p)
    assert rel(o["rhs"], ref_rhs) < 1e-13
    assert np.array_equal(o["pold"], p) and not np.abs(o["pres"]).any()
    vort = orc.vorticity(u, v, h)
    assert rel(o["vort"], vort) < 1e-14
    assert np.abs(o["vort_linf"] - orc.block_linf(vort)).max() < 1e-12 * np.abs(vort).max()
    for off in (2, 4):
        want = orc.adapt_tags(u, v, cchi, h, 0.1, off)
        flagged = want == 0.2
        assert flagged.any() and np.array_equal(o[f"tags{off}"] == 0.2, flagged)
        assert rel(o[f"tags{off}"], want) < 1e-14
        assert np.abs(o[f"tags{off}_linf"] - orc.block_linf(want)).max() < 1e-12 * np.abs(want).max()


# ---- Krylov: three-kernel iteration vs the oracle, the Hilbert run and the five-kernel iteration -------------------------
KRYLOV_ITERS = (1, 2, 3, 7, 12)


def _rhs(NX, NY):
    rng = np.random.default_rng(100 + NX + NY)
    X, Y = np.meshgrid((np.arange(NX) + 0.5) / NX, (np.arange(NY) + 0.5) / NY)
    xs = np.cos(2 * np.pi * X) * np.cos(np.pi * Y) + 0.1 * rng.uniform(-1, 1, (NY, NX))
    return orc.laplacian_neumann(xs)   # consistent right-hand side of the singular Neumann problem


def neighbour_table(sim):
    """cup2d_plan_table(3) of the context's own configuration: W, E, S, N slots of every local block"""
    lib = cup2d_b200.load_library()
    cfg = Lb.Config(sim.nbx, sim.nby, len(sim.order), sim.order.ctypes.data_as(C.POINTER(C.c_int32)), 0, 1,
                    sim.rank_begin.ctypes.data_as(C.POINTER(C.c_int64)), sim.h, NU, CFL, -1, 0)
    h = C.c_void_p()
    Lb.check(lib.cup2d_plan_create(C.byref(cfg), C.byref(h)))
    nbr = np.empty(4 * sim.nloc, dtype=np.int32)
    assert lib.cup2d_plan_table(h, 3, nbr.ctypes.data_as(C.POINTER(C.c_int32))) == nbr.size
    lib.cup2d_destroy(h)
    return nbr


def five_kernel_solve(nbr, b_blocks, K, x0_blocks=None, tol_abs=0.0, tol_rel=0.0, max_restarts=0):
    """at most K iterations of the five-kernel BiCGSTAB (a Poisson-only context always runs it) from x0 (default 0)"""
    lib = cup2d_b200.load_library()
    h = C.c_void_p()
    nblk = len(nbr) // 4
    Lb.check(lib.cup2d_poisson_create(nblk, nbr.ctypes.data_as(C.POINTER(C.c_int32)), 0, C.byref(h)))
    try:
        x = np.zeros_like(b_blocks) if x0_blocks is None else np.array(x0_blocks, dtype=np.float64)
        Lb.check(lib.cup2d_field_upload(h, Lb.FIELDS["tmp"], b_blocks.ctypes.data))
        Lb.check(lib.cup2d_field_upload(h, Lb.FIELDS["pres"], x.ctypes.data))
        it, err = C.c_int(), C.c_double()
        Lb.check(lib.cup2d_poisson_solve(h, tol_abs, tol_rel, max_restarts, K, C.byref(it), C.byref(err)))
        Lb.check(lib.cup2d_field_download(h, Lb.FIELDS["pres"], x.ctypes.data))
    finally:
        lib.cup2d_destroy(h)
    return it.value, err.value, x


@functools.lru_cache(maxsize=None)
def _krylov(shape, kind):
    sim = make_sim(shape, kind)
    b = _rhs(sim.NX, sim.NY)
    nbr = neighbour_table(sim)
    bb = cup2d_b200.to_blocks(b, sim.local_order, sim.nbx)
    out = {}
    for K in KRYLOV_ITERS:
        sim.upload("tmp", b)
        sim.upload("pres", np.zeros_like(b))
        it, err = sim.poisson_solve(max_iter=K)
        it5, err5, x5 = five_kernel_solve(nbr, bb, K)
        out[K] = (it, err, sim.download("pres"), it5, err5,
                  cup2d_b200.from_blocks(x5, sim.local_order, sim.nbx, sim.nby, 1))
    sim.close()
    return b, out


@functools.lru_cache(maxsize=None)
def _krylov_oracle(shape):
    b = _krylov(shape, "hilbert")[0]
    return {K: orc.bicgstab(b, np.zeros_like(b), max_iter=K) for K in KRYLOV_ITERS}


@pytest.mark.parametrize("shape,kind", case_ids())
def test_krylov_three_kernels_vs_oracle_hilbert_and_five_kernels(shape, kind):
    b, got = _krylov(shape, kind)
    _, hil = _krylov(shape, "hilbert")
    want = _krylov_oracle(shape)
    # the residual r = b - A x is a difference of terms of the size of b (x0 = 0: r0 = b), so its rounding is relative to
    # |b|, not to |r|, which falls by four orders in 12 iterations
    r0 = np.abs(b).max()
    for K in KRYLOV_ITERS:
        it, err, x, it5, err5, x5 = got[K]
        xr, itr, errr = want[K]
        assert it == itr == it5 == hil[K][0] == K
        assert abs(err - errr) < 1e-9 * max(1.0, errr) and np.abs(x - xr).max() < 1e-9, K
        assert rel(x, hil[K][2]) < 1e-12 and abs(err - hil[K][1]) <= 1e-12 * r0, K
        assert rel(x, x5) < 1e-12 and abs(err - err5) <= 1e-12 * r0, K


# ---- full steps -----------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _step(shape, kind):
    sim = make_sim(shape, kind, nu=NU, cfl=CFL)
    u, v, p, *_ = make_fields(sim.NX, sim.NY, 31)
    sim.upload("vel", u, v)
    sim.upload("pres", p)
    dt, it, err = sim.step(max_iter=6)
    out = (dt, it, err, *sim.download("vel"), sim.download("pres"))
    sim.close()
    return (u, v, p), out


@pytest.mark.parametrize("shape,kind", case_ids())
def test_step_any_order_vs_oracle(shape, kind):
    (u, v, p), (dt, it, err, gu, gv, gp) = _step(shape, kind)
    assert dt == _step(shape, "hilbert")[1][0] and it == 6
    ref = orc.step(u, v, p, NU, CFL, kiter=6)
    assert abs(dt - ref["dt"]) <= 1e-16 * ref["dt"]
    scale = max(np.abs(ref["u"]).max(), np.abs(ref["v"]).max())
    assert np.abs(gu - ref["u"]).max() <= 1e-9 * scale and np.abs(gv - ref["v"]).max() <= 1e-9 * scale
    assert np.abs(gp - ref["p"]).max() <= 1e-8 * np.abs(ref["p"]).max()


def _run_steps(shape, kind, nsteps, graph, **kw):
    """as tests/test_gpu_parity.py::_run_steps, on any domain and order"""
    sim = make_sim(shape, kind, nu=NU, cfl=0.4)
    u, v, p, *_ = make_fields(sim.NX, sim.NY, 11)
    sim.set_graph(graph)
    sim.upload("vel", u, v)
    sim.upload("pres", p)
    info = []
    for _ in range(nsteps):
        if graph:
            sim.step_enqueue(**kw)
            info.append(sim.step_result())
        else:
            _, dt = sim.compute_dt()
            info.append(sim.step(dt=dt, **kw))
    out = (sim.download("vel"), sim.download("pres"), info)
    sim.close()
    return out


def test_graph_replayed_steps_on_an_odd_domain_in_random_order():
    """step_enqueue (graph replay from the second step on) bitwise equals directly launched steps on 5x3 blocks in a
    random order: partial tiles next to each other and a partial last chunk"""
    (gu, gv), gp, ginfo = _run_steps((5, 3, 0), "random", 5, True, max_iter=7, max_restarts=0)
    (du, dv), dp, dinfo = _run_steps((5, 3, 0), "random", 5, False, max_iter=7, max_restarts=0)
    assert [i[0] for i in ginfo] == [i[0] for i in dinfo]
    assert [i[1] for i in ginfo] == [i[1] for i in dinfo] == [7] * 5
    assert np.array_equal(gu, du) and np.array_equal(gv, dv) and np.array_equal(gp, dp)


@pytest.mark.parametrize("kind", ["hilbert", "random"])
def test_graph_while_node_stops_where_the_host_polled_solve_stops_on_5x3(kind):
    kw = dict(tol_abs=1e-7, tol_rel=0.0, max_restarts=100, max_iter=400)
    (gu, gv), gp, ginfo = _run_steps((5, 3, 0), kind, 4, True, **kw)
    (du, dv), dp, dinfo = _run_steps((5, 3, 0), kind, 4, False, **kw)
    assert [i[1] for i in ginfo] == [i[1] for i in dinfo]
    assert all(0 < i[1] < 400 and i[2] <= 1e-7 for i in ginfo), ginfo
    assert np.array_equal(gu, du) and np.array_equal(gv, dv) and np.array_equal(gp, dp)


# ---- reference goldens in other orders ------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["steps_L2_random_k8", "steps_L3_tg_k15"])
@pytest.mark.parametrize("kind", ["row", "random"])
def test_time_steps_vs_reference_golden_in_other_orders(golden_dir, name, kind):
    d = np.load(os.path.join(golden_dir, name + ".npz"))
    L, K = int(d["L"]), int(d["kiter"])
    sim = make_sim((1, 1, L), kind, nu=float(d["nu"]), cfl=float(d["cfl"]))
    sim.upload("vel", d["u0"], d["v0"])
    sim.upload("pres", d["p0"])
    for s in range(len(d["dt"])):
        dt, iters, err = sim.step(max_iter=K)
        assert abs(dt - d["dt"][s]) < 1e-15 and iters == K
        u, v = sim.download("vel")
        assert np.abs(u - d["u"][s]).max() < 1e-9 and np.abs(v - d["v"][s]).max() < 1e-9
        assert np.abs(sim.download("pres") - d["p"][s]).max() < 1e-9
    sim.close()


def test_penalisation_phase_vs_reference_golden_in_random_order(penal_golden):
    """the recorded shapes' block ids index the Hilbert order; mapped through the permutation, blend and assembly stay bit
    for bit the reference's"""
    L, steps = penal_golden
    hil = cup2d_b200.block_order(1, 1, L)
    order = make_order(1, 1, L, "random")
    pos = np.empty((1 << L, 1 << L), dtype=np.int32)
    pos[order[:, 1], order[:, 0]] = np.arange(len(order))
    sim = cup2d_b200.Simulation(L, order=order)
    for st in steps:
        sim.upload("vel", st["u0"], st["v0"])
        sim.upload("chi", st["chi"])
        for k, sh in enumerate(st["shapes"]):
            ids = pos[hil[sh["ids"], 1], hil[sh["ids"], 0]]
            assert not np.array_equal(ids, sh["ids"])
            sim.shape_set(k, ids, sh["X"], sh["udef"])
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


# ---- dump -------------------------------------------------------------------------------------------------------------------
def test_dump_records_follow_the_callers_order(tmp_path):
    """each block's .attr.raw / .xyz.raw record equals the Hilbert run's record of the same (i, j) byte for byte"""
    shape = (3, 2, 1)
    recs = {}
    for kind in ("hilbert", "random"):
        sim = make_sim(shape, kind)
        u, v, *_ = make_fields(sim.NX, sim.NY, 5)
        sim.upload("vel", u, v)
        pref = str(tmp_path / kind)
        sim.dump(0.25, pref)
        attr = np.fromfile(pref + ".attr.raw", dtype=np.uint8).reshape(sim.nloc, -1)
        xyz = np.fromfile(pref + ".xyz.raw", dtype=np.uint8).reshape(sim.nloc, -1)
        assert attr.shape[1] == 64 * 3 * 4 and xyz.shape[1] == 64 * 8 * 4
        recs[kind] = {tuple(ij): (attr[k], xyz[k]) for k, ij in enumerate(sim.local_order)}
        ax, aa = orc.dump_arrays(u, v, sim.local_order, 1.0 / max(shape[:2]) / 8, shape[2])
        assert ax.tobytes() == xyz.tobytes() and aa.tobytes() == attr.tobytes()
        sim.close()
    assert recs["hilbert"].keys() == recs["random"].keys()
    for ij, (a, x) in recs["random"].items():
        assert np.array_equal(a, recs["hilbert"][ij][0]) and np.array_equal(x, recs["hilbert"][ij][1]), ij


# ---- one large case ---------------------------------------------------------------------------------------------------------
def test_large_grid_step_in_random_order_matches_hilbert():
    """L = 7 (128^2 blocks, 1024 tiles) in a random order: the tile kernels run one wave of at most 2 CTAs per SM, so the
    tiles in flight are scattered over the whole grid instead of forming one compact region.  One step, 10 iterations:
    dt bitwise, pressure to 1e-10 relative (the dot products are partitioned differently; measured on an H100 80GB HBM3
    at a 700 W power limit: 4.8e-16 relative, residual 3.4e-15 relative).  Too large for the CPU emulation of the device
    code (tools/run_emulated_gpu_tests.sh leaves it out with the other large grids): only the H100 runs it."""
    out = {}
    for kind in ("hilbert", "random"):
        sim = make_sim((1, 1, 7), kind, nu=NU, cfl=CFL)
        u, v, p, *_ = make_fields(sim.NX, sim.NY, 2024)
        sim.upload("vel", u, v)
        sim.upload("pres", p)
        dt, it, err = sim.step(max_iter=10)
        out[kind] = (dt, it, err, sim.download("pres"))
        sim.close()
    (dh, ih, eh, ph), (dr, ir, er, pr) = out["hilbert"], out["random"]
    assert dh == dr and ih == ir == 10
    assert rel(pr, ph) < 1e-10 and abs(er - eh) <= 1e-10 * eh
